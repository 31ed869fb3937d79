/*
 * swim.h — C ABI of swim-b200: an H100-native bulk simulator of the SWIM membership
 * protocol that keeps the Core/Types API surface of jpfuentes2/swim (Haskell).
 *
 * Every entry point names the reference interface it replaces (path:line under the
 * reference checkout, commit 4320f07). The reference has no FFI of its own, so this
 * boundary is what a `foreign import ccall` shim (INTEGRATION.md) binds.
 *
 * Conventions
 *   - plain C, no C++/torch types; caller allocates every buffer; the library copies
 *     in/out and never retains caller pointers; no callbacks.
 *   - every function returns int: SWIM_OK (0) or a negative SWIM_E* code; the String of
 *     the reference's `Either Error a` (Types.hs:33) is swim_last_error().
 *   - `Maybe Message` results (Core.hs:142,189-218) become (out, has_out).
 *   - member names (`String`, Types.hs:70) are u32 ids; ascending id order == the
 *     ascending key order of `Map.elems` (Core.hs:77). Name tables live host-side.
 *   - a handle is externally synchronised (one caller at a time); swim_sim_step blocks
 *     (Haskell: `foreign import ccall safe`).
 *   - the compute path is CUDA sm_90a only. There is no CPU fallback: without a CUDA
 *     device swim_sim_create fails with SWIM_ENODEV.
 */
#ifndef SWIM_H_
#define SWIM_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif
#if defined(__GNUC__)
#pragma GCC visibility push(default) /* the library is built with -fvisibility=hidden */
#endif

#define SWIM_ABI_VERSION 2u

/* Opaque handle: N simulated `Store`s (Types.hs:53-60) resident in HBM. */
typedef struct swim_sim swim_sim_t;

/* ---- error codes (Types.hs:33 `type Error = String`; Core.hs:274 `either error return`) */
enum {
  SWIM_OK = 0,
  SWIM_EINVAL = -1,  /* bad argument / wrong message constructor (Core.hs:191,195,218 `undefined`) */
  SWIM_ENOMEM = -2,
  SWIM_ECUDA = -3,   /* CUDA runtime error; text in swim_last_error */
  SWIM_ERANGE = -4,  /* value does not fit the device width (incarnation > u32, id >= N ...) */
  SWIM_EDECODE = -5, /* wire decode failure (Core.hs:86-87 `fail`) */
  SWIM_ENODEV = -6,  /* no CUDA device: the product path has no CPU fallback */
  SWIM_ENCCL = -7,
  SWIM_ECAP = -8,    /* caller buffer / view row too small */
  SWIM_ESTATE = -9   /* call not valid in this state (e.g. step before set_view) */
};

/* ---- Liveness (Types.hs:76-77, derived Enum order) */
enum { SWIM_ALIVE = 0, SWIM_SUSPECT = 1, SWIM_DEAD = 2, SWIM_VACANT = 3 /* empty view slot */ };

/* ---- MsgType (Types.hs:159-167) / msgIndex (Types.hs:169-178) */
enum {
  SWIM_MSG_PING = 0,
  SWIM_MSG_INDIRECT_PING = 1,
  SWIM_MSG_ACK = 2,
  SWIM_MSG_SUSPECT = 3,
  SWIM_MSG_ALIVE = 4,
  SWIM_MSG_DEAD = 5,
  SWIM_MSG_COMPOUND = 6
};

#define SWIM_NO_MEMBER 0xFFFFFFFFu /* id stored in vacant view slots (sorts last) */
#define SWIM_MAX_K 7u              /* indirect fan-out k <= 7 (1+k draws = two Philox blocks) */
#define SWIM_MAX_PB 32u            /* piggyback buffer records per node (one lane each) */
#define SWIM_MAX_TIMER 63u         /* suspicion rounds fit the 6-bit countdown in vst */
#define SWIM_MAX_TIMER_LIFEGUARD 15u /* with suspicion_max: 4-bit countdown + 2-bit confirmation count */
#define SWIM_MAX_PROBES 4u         /* probes_per_round */
#define SWIM_MAX_VIEW 256u         /* view_cap is 32*W, W in {1,2,4,8} */

/* ---- Config (Types.hs:46-51, Util.hs:44-50) + the simulator's extra knobs -------------
 * numToGossip (Util.hs:48) is used by the reference both as #probes per period and as the
 * indirect fan-out (Core.hs:239,249). Here: one probe per node per round (SWIM; SURVEY Q11)
 * and k_indirect proxies. gossipInterval (Util.hs:49) and the ack timeout (Core.hs:258)
 * are both exactly one round. */
typedef struct swim_config {
  uint32_t abi_version;      /* SWIM_ABI_VERSION */
  uint32_t n_nodes;          /* N simulated nodes == N `Store`s (global, all ranks) */
  uint32_t view_cap;         /* slots per view row: 32, 64, 128 or 256 */
  uint32_t k_indirect;       /* k: `numToGossip` as used at Core.hs:249 */
  uint32_t fanout;           /* piggyback recipients per round, 1..1+k (target, then proxies) */
  uint32_t pb_cap;           /* B: piggyback buffer capacity in records (Core.hs:136 FIXME) */
  uint32_t suspicion_rounds; /* S: Suspect -> Dead after S rounds (Core.hs:141 FIXME) */
  uint32_t retransmit;       /* T: transmissions per record before it leaves the buffer */
  uint32_t loss_ppm;         /* per-leg Bernoulli message loss, parts per million */
  uint32_t flags;            /* SWIM_F_* */
  uint64_t seed;             /* Philox4x32-10 key */
  uint32_t rank;             /* this process's shard (0..world-1) */
  uint32_t world;            /* number of shards == GPUs; 1 = single GPU */
  int32_t device;            /* CUDA device ordinal; -1 = current device */
  uint32_t base_port;        /* port reported in swim_member_t (reference fixture: 4000) */
  /* Seeded churn, generated on the device (BASELINE config C5; no reference counterpart — the reference has no fault
   * injection): at the start of every round, before the events of that round, each live process crashes with probability
   * churn_ppm / 1e6 and comes back after a delay uniform in [rejoin_min, rejoin_max] rounds with incarnation + 1 and an
   * Alive broadcast (exactly what SWIM_EV_CRASH / SWIM_EV_REJOIN do). 0 = off. Draws: Philox purpose 7 (DESIGN.md 2.3). */
  uint32_t churn_ppm;
  uint32_t rejoin_min, rejoin_max; /* 1 <= rejoin_min <= rejoin_max */
  /* Reference-literal probing (SURVEY Q11): `kRandomMembers store numToGossip []` probes numToGossip members per period,
   * one after the other (Core.hs:239-240). 1 = one probe target per node per round (SWIM; the default). */
  uint32_t probes_per_round;
  /* Lifeguard-style dynamic suspicion timeout (SURVEY 8(f)-4): 0 = off (every suspicion lasts suspicion_rounds). Otherwise a
   * suspicion starts with suspicion_max rounds (suspicion_rounds <= suspicion_max <= 15) and every further Suspect message
   * received about the suspected member shortens it logarithmically, down to suspicion_rounds after 3 confirmations:
   * timeout(c) = max - (max - min) * log(c + 1) / log(4). */
  uint32_t suspicion_max;
  uint32_t _reserved;
} swim_config_t;

#define SWIM_F_NONE 0u
/* Protocol variants (SURVEY §8(f)-4). Off = the reference's rules as written / as completed in DESIGN.md §2.
 * SWIM_F_STRICT_OVERRIDE: the SWIM paper's §4.2 override order instead of the guards of suspectOrDeadNode'
 *   (Core.hs:151-152,182-184; SURVEY Q14): Suspect(i) also overrides Suspect(j) for i > j (and re-arms the
 *   countdown); Dead(i) ("Confirm") overrides Alive(j)/Suspect(j) for ANY i, j and keeps max(i, j).
 * SWIM_F_ROUND_ROBIN: the "robust scheme" the reference asks for (`-- FIXME: move from random to robust scheme`,
 *   Core.hs:232; SWIM paper §4.3): ping targets are taken in a per-node, per-epoch pseudo-random ORDER of the view
 *   instead of uniformly at random, so every Alive member is probed at least once per view_cap rounds. */
#define SWIM_F_STRICT_OVERRIDE 1u
#define SWIM_F_ROUND_ROBIN 2u
#define SWIM_F__ALL 3u

/* ---- Member (Types.hs:62-68). name -> id; memberHost/memberHostNew -> (addr, port);
 * memberLastChange (UTCTime) -> the round at which the entry last changed. */
typedef struct swim_member {
  uint32_t id;
  uint32_t addr;        /* HostAddress; the simulator reports addr == id */
  uint16_t port;
  uint8_t liveness;     /* SWIM_ALIVE / SWIM_SUSPECT / SWIM_DEAD */
  uint8_t timer;        /* remaining suspicion rounds (0 unless Suspect) */
  uint32_t incarnation; /* Haskell Int (Types.hs:66) range-checked to u32 */
  uint64_t last_change;
} swim_member_t;

/* ---- Message (Types.hs:122-145), tagged by `kind` = SWIM_MSG_* ------------------------
 *   Ping          { seq_no, node }
 *   IndirectPing  { seq_no, target, port, node }
 *   Ack           { seq_no, payload[payload_len] }
 *   Suspect       { incarnation, node }
 *   Alive         { incarnation, node, target(=addr), port }
 *   Dead          { incarnation, node, dead_from } */
#define SWIM_ACK_PAYLOAD_MAX 16u
typedef struct swim_message {
  uint8_t kind;
  uint8_t payload_len;
  uint16_t port;
  uint32_t seq_no;
  uint32_t node;
  uint32_t target;
  int64_t incarnation;
  uint32_t dead_from;
  uint8_t payload[SWIM_ACK_PAYLOAD_MAX];
  uint32_t _pad;
} swim_message_t;

/* ---- Gossip (Types.hs:42-44): Direct msg addr | Broadcast msg */
typedef struct swim_gossip {
  uint8_t is_direct;  /* 1 = Direct, 0 = Broadcast */
  uint8_t _pad;
  uint16_t dest_port; /* SockAddrInet port of a Direct */
  uint32_t dest_addr; /* SockAddrInet host of a Direct */
  swim_message_t msg;
} swim_gossip_t;

/* ---- piggyback record: the device-side form of a Broadcast Suspect/Alive/Dead -------- */
typedef struct swim_record {
  uint32_t member;      /* Message.node */
  uint32_t incarnation; /* Message.incarnation */
  uint32_t from;        /* Dead.deadFrom (0 for other kinds) */
  uint8_t kind;         /* SWIM_MSG_SUSPECT / _ALIVE / _DEAD */
  uint8_t ttl;          /* remaining transmissions */
  uint16_t _pad;
} swim_record_t;

/* ---- Event: the seeded event trace fed to the simulator (no reference counterpart; the
 * reference's only inputs are UDP datagrams, Core.hs:280). Applied at the start of `round`. */
enum { SWIM_EV_CRASH = 0, SWIM_EV_REJOIN = 1, SWIM_EV_INJECT = 2 };
typedef struct swim_event {
  uint32_t round; /* absolute round number (first executed round is 1) */
  uint32_t node;
  uint8_t kind;   /* SWIM_EV_* */
  uint8_t _pad[7];
  swim_message_t msg; /* SWIM_EV_INJECT: Suspect/Alive/Dead delivered to `node` */
} swim_event_t;

/* ---- bulk state arrays (swim_sim_get_array / swim_sim_set_array) ----------------------
 * n = nodes owned by this rank, cap = view_cap, B = pb_cap.  */
enum {
  SWIM_ARR_ALIVE = 0,    /* u8 [N]      truth: process up (replicated on every rank) */
  SWIM_ARR_SELF_INC = 1, /* u32[n]      storeIncarnation (Types.hs:54) */
  SWIM_ARR_SEQNO = 2,    /* u32[n]      storeSeqNo (Types.hs:53); scalar API only */
  SWIM_ARR_NBR = 3,      /* u32[n*cap]  member ids, ascending, SWIM_NO_MEMBER padded */
  SWIM_ARR_VST = 4,      /* u8 [n*cap]  liveness | timer<<2  (with suspicion_max: liveness | timer<<2 | confirmations<<6) */
  SWIM_ARR_VINC = 5,     /* u32[n*cap]  memberIncarnation */
  SWIM_ARR_VLAST = 6,    /* u32[n*cap]  memberLastChange as a round number */
  SWIM_ARR_PB = 7,       /* swim_record_t[n*B], newest first; entries >= cnt are zero */
  SWIM_ARR_PB_CNT = 8,   /* u8 [n] */
  SWIM_ARR_BACK_AT = 9,  /* u32[N]      churn: round at which a crashed process rejoins, 0 = none (replicated on every rank) */
  SWIM_ARR_LAST_CRASH = 10,  /* u32[N]  round of the process's last crash (up -> down), 0 = never (replicated) */
  SWIM_ARR_LAST_REJOIN = 11, /* u32[N]  round of its last rejoin (down -> up), 0 = never (replicated): what a convergence
                                        study needs to tell a late detection from a false positive */
  SWIM_ARR__COUNT = 12
};

/* ---- per-run counters (swim_sim_counters), cumulative since create ------------------- */
enum {
  SWIM_CTR_PINGS = 0,          /* Ping sent (Core.hs:246) */
  SWIM_CTR_DIRECT_FAIL = 1,    /* no Ack to the direct Ping (Core.hs:247) */
  SWIM_CTR_INDIRECT_PINGS = 2, /* IndirectPing sent (Core.hs:250) */
  SWIM_CTR_SUSPECT_LOCAL = 3,  /* suspectNode raised by a failed probe (Core.hs:253) */
  SWIM_CTR_DEAD_TIMEOUT = 4,   /* Suspect -> Dead by timer (Core.hs:141 FIXME) */
  SWIM_CTR_MSGS = 5,           /* piggyback envelopes sent */
  SWIM_CTR_RECS_SENT = 6,      /* records carried by those envelopes */
  SWIM_CTR_RECS_APPLIED = 7,   /* received records that changed state (re-broadcast) */
  SWIM_CTR_REFUTES = 8,        /* self-refutations (Core.hs:155-166) */
  SWIM_CTR_PB_DROPPED = 9,     /* records pushed out of a full buffer */
  SWIM_CTR_MSGS_RECV = 10,     /* envelopes consumed by live receivers */
  SWIM_CTR__COUNT = 11
};

/* =============================== lifecycle ========================================== */

uint32_t swim_abi_version(void);
const char *swim_strerror(int code);

/* Text of the last error on this handle; sim may be NULL (last error of the calling
 * thread, e.g. from a failed swim_sim_create). Replaces `Left err` (Util.hs:44,103). */
const char *swim_last_error(const swim_sim_t *sim);

/* parseConfig (Util.hs:44-50): fills the defaults used by BASELINE config C1
 * (k=3, fanout=4, B=8, S=5, T=8, view_cap=32, world=1). */
int swim_config_default(swim_config_t *cfg);

/* configure / makeStore (Util.hs:76-107): allocate N stores with seqNo = incarnation = 0
 * (Util.hs:79-80), empty views, every node up. Fails with SWIM_ENODEV without a GPU. */
int swim_sim_create(const swim_config_t *cfg, swim_sim_t **out);
void swim_sim_destroy(swim_sim_t *sim);

/* Number of nodes owned by this rank and the id of the first one (contiguous shards). */
int swim_sim_local_range(const swim_sim_t *sim, uint32_t *first, uint32_t *count);

/* Install the view graph: nbr is the GLOBAL [N*view_cap] id matrix (row i = node i's
 * members, ascending, SWIM_NO_MEMBER padded, never containing i). Every present member
 * starts Alive with incarnation 0 and last_change 0 — the bulk form of the tests'
 * `swapTVar storeMembers` (Spec.hs:101). Each rank keeps its own rows plus the in-edge
 * index of its own nodes. */
int swim_sim_set_view(swim_sim_t *sim, const uint32_t *nbr_global);

/* The same with the matrix already in device memory on the handle's device (read on the handle's stream): no host
 * copy of the N * view_cap ids. Either call builds the in-edge index, the observer lists and the membership filters on
 * the device. SWIM_ESTATE after swim_sim_ipc_connect, as for swim_sim_set_view. */
int swim_sim_set_view_device(swim_sim_t *sim, const uint32_t *nbr_global_dev);

/* Host-side synthetic topologies (BASELINE configs): rows of `degree` distinct ids != i.
 * kind 0 = complete (degree ignored, needs N-1 <= view_cap), 1 = uniform random,
 * 2 = ring lattice (i±1..±degree/2), 3 = symmetric random: the union of degree/2 random
 * Hamiltonian cycles (DESIGN.md §2.3, purpose 11), j in row i exactly when i is in row j,
 * between 2 and degree members per row (fewer than degree where cycles repeat a neighbour);
 * degree must be even and N >= 3 (SWIM_EINVAL otherwise). out is [N*view_cap]. No device needed. */
enum { SWIM_TOPO_COMPLETE = 0, SWIM_TOPO_RANDOM = 1, SWIM_TOPO_RING = 2, SWIM_TOPO_SYMMETRIC = 3 };
int swim_topology_generate(int kind, uint32_t n_nodes, uint32_t view_cap, uint32_t degree,
                           uint64_t seed, uint32_t *out_nbr);

/* The same matrix generated on the device, in temporary device memory on the handle's stream, and installed as
 * swim_sim_set_view_device installs it (same checks, SWIM_ESTATE after swim_sim_ipc_connect, the checkpoint dropped).
 * Bit-identical to swim_topology_generate(kind, N, view_cap, degree, seed, .) for every kind. On a sharded handle every
 * rank generates the whole global matrix itself (no communication). The temporary memory is freed before the call
 * returns. */
int swim_sim_generate_view(swim_sim_t *sim, int kind, uint32_t degree, uint64_t seed);

/* ====================== bulk path: the accelerated protocol loop =====================
 * Replaces the ticker + the three conduits of Core.main (Core.hs:233-241, 279-287). */

/* Run `rounds` protocol periods for every node: events -> tick (timers, target selection,
 * ping / k indirect pings, local suspicion, piggyback send) -> [cross-shard exchange] ->
 * receive (state machine of Core.hs:142-218, re-broadcast). Blocks until done. */
int swim_sim_step(swim_sim_t *sim, uint32_t rounds);

/* Same, but only enqueues the work on the handle's stream; pair with swim_sim_sync. */
int swim_sim_step_async(swim_sim_t *sim, uint32_t rounds);
int swim_sim_sync(swim_sim_t *sim);

/* Run on the caller's cudaStream_t (e.g. torch.cuda.current_stream().cuda_stream) so that
 * the caller's CUDA events bracket the kernels. NULL = the handle's private stream. */
int swim_sim_set_stream(swim_sim_t *sim, void *cuda_stream);

/* Queue events (any order; applied at the start of event.round, same-node events in the
 * order given). Events for rounds already executed are rejected with SWIM_EINVAL. */
int swim_sim_inject(swim_sim_t *sim, const swim_event_t *events, size_t n);

/* Number of rounds executed so far (== the seqNo of the last Ping, Core.hs:238). */
int swim_sim_round(const swim_sim_t *sim, uint32_t *round);

/* Checkpoint / resume: a run is reproduced exactly by the config, the view (SWIM_ARR_NBR rows -> swim_sim_set_view), the
 * other state arrays (swim_sim_set_array), the events still pending, and the round counter — the counter of every
 * Philox draw. swim_sim_set_round puts a fresh handle at `round` (pending events must lie after it). */
int swim_sim_set_round(swim_sim_t *sim, uint32_t round);

/* Device-resident checkpoint, one slot per handle. swim_sim_save copies this rank's mutable state (alive[], incarnations,
 * the rows' liveness / incarnation / lastChange, the piggyback buffers, the counters), the round counter and the pending
 * events into a second set of device arrays: stream-ordered device-to-device copies, no host traffic. swim_sim_load puts
 * the handle back there (and clears every round-stamped scratch array), so the same rounds can be stepped again and
 * give the same result — what a parameter sweep or a repeated timing window needs. A new view (swim_sim_set_view) or
 * a membership change through the scalar or bulk calls drops the checkpoint. Sharded runs: every rank saves / loads its own
 * shard while ALL ranks are between steps (host-side barrier before and after). */
int swim_sim_save(swim_sim_t *sim);
int swim_sim_load(swim_sim_t *sim);

/* Change the protocol scalars of a live handle between steps — suspicion_rounds, suspicion_max, retransmit, loss_ppm,
 * flags, churn_ppm, rejoin_min / rejoin_max and seed are taken from `cfg`; every other field must equal the handle's
 * (SWIM_EINVAL otherwise: sizes and the shard layout are fixed at create). With swim_sim_save / swim_sim_load this is a
 * parameter sweep on ONE handle: the view, its in-edge index and the device arrays are built once. */
int swim_sim_set_params(swim_sim_t *sim, const swim_config_t *cfg);

/* Bulk membership edits between steps, on the device (one warp per affected row, no host copy of the rows). Both mark
 * the view changed: the next step rebuilds the in-edge index, the checkpoint is dropped (swim_sim_load fails until the
 * next swim_sim_save), and swim_sim_export_round returns SWIM_ESTATE until the next step. On a sharded handle (world > 1)
 * they are collectives, like swim_sim_push_pull and swim_sim_load: every rank issues the same calls in the same order
 * (swim_sim_add_members with the same global list; each rank applies its own observers' adds), outputs are this
 * rank's counts, and the next step rebuilds the index on all ranks together; SWIM_ESTATE before swim_sim_ipc_connect /
 * swim_sim_connect. Scalar membership changes on a sharded handle still make its next step return SWIM_ESTATE.
 *
 * removeDeadNodes (Core.hs:65-67) on every local store at once: Dead entries with round - last_change >= min_age leave
 * (round = rounds executed so far; min_age = 0 is the reference's form, swim_remove_dead_nodes on every node). Rows stay
 * ascending with vacancies last. *n_removed (may be NULL) = entries removed. */
int swim_sim_remove_dead_nodes(swim_sim_t *sim, uint32_t min_age, uint64_t *n_removed);

/* addNewMember (Core.hs:206-216) for many stores, applied in the order given: a member the observer does not list is
 * inserted as Alive with `incarnation` and last_change = the current round (what an inserting swim_alive_node does); a
 * member it lists is left untouched; an add to a full row is dropped and counted in *n_full. Every add is checked
 * before anything changes (ids < N, member != observer; SWIM_EINVAL otherwise). Outputs may be NULL. */
typedef struct swim_member_add {
  uint32_t observer, member, incarnation, _pad;
} swim_member_add_t;
int swim_sim_add_members(swim_sim_t *sim, const swim_member_add_t *adds, size_t n, uint64_t *n_added, uint64_t *n_full);

/* Push-pull state exchange between steps (DESIGN.md §2.6): memberlist's anti-entropy, the missing half of the
 * reference's join (Config.joinHosts, Types.hs:47, is parsed and never used); the exchange itself has no reference
 * counterpart. At the current round r (the round counter does not advance) every up node with at least one Alive slot
 * picks one Alive member from the Philox block (r, node, 10, 0); if that partner is up, the two swap their full states
 * (Alive(self), then every occupied slot as Alive / Suspect / Dead(from = sender)), read from a snapshot taken before
 * anything changes. A receiver merges its senders in ascending id, each record through the receive rules; an Alive record
 * about a member it does not list is inserted as swim_alive_node inserts (aliveNode / addNewMember, Core.hs:206-216), and
 * dropped when the row is full. Two calls at the same round pick the same partners. No message is lost. On a sharded
 * handle a collective (every rank calls it; outputs are this rank's, their sums the single-shard ones); SWIM_ESTATE on
 * a sharded handle that is not connected, before a view is installed and on a failed handle. Without inserts only state
 * changes and the checkpoint stays valid; with inserts (on any rank) the view is marked changed as by the bulk edits
 * above.
 * Outputs may be NULL: *n_exchanges = choices whose partner was up, *n_inserted = members inserted, *n_full = inserts
 * dropped on a full row. */
int swim_sim_push_pull(swim_sim_t *sim, uint64_t *n_exchanges, uint64_t *n_inserted, uint64_t *n_full);

/* Seed joins between steps (DESIGN.md §2.7): memberlist's Join(joinHosts), the join the reference names and never
 * performs (Config.joinHosts, Types.hs:47, default udp://127.0.0.1:4000 at Util.hs:46). At the current round (the round
 * counter does not advance) each pair {node j, seed s} is one full-state exchange between j and its join host s, with
 * the push-pull exchange's records and merge rules. A pair is an exchange iff both are up; neither needs to list the
 * other, and either may have an empty row. A receiver merges its distinct senders (the seeds of its exchanges and the
 * joiners that named it) once each, in ascending id. With SWIM_JOIN_FRESH every listed joiner that is up first loses its
 * whole view and piggyback buffer (self_inc is kept): a process that restarts empty, so it sends only Alive(self). Every
 * pair is checked before anything changes (ids < N, node != seed; SWIM_EINVAL otherwise); n = 0 is a no-op. No random
 * draws: the result is a function of the pairs, the state and the round. SWIM_ESTATE as for swim_sim_push_pull. On a
 * sharded handle a collective: every rank is given the same global list; outputs are this rank's (the pairs whose joiner
 * it owns, its receivers' inserts and drops), their sums the single-shard ones. The view is marked changed as by the
 * bulk edits when some rank inserted a member or a fresh reset emptied an occupied slot; otherwise only state changes
 * and the checkpoint stays valid.
 * Outputs may be NULL: *n_exchanges = pairs that were exchanges (duplicates included), *n_inserted = members inserted,
 * *n_full = inserts dropped on a full row. */
typedef struct swim_join {
  uint32_t node, seed;
} swim_join_t;
enum { SWIM_JOIN_FRESH = 1u << 0 };
int swim_sim_join(swim_sim_t *sim, const swim_join_t *joins, size_t n, uint32_t flags, uint64_t *n_exchanges,
                  uint64_t *n_inserted, uint64_t *n_full);

/* Graceful leaves between steps (DESIGN.md §2.8): memberlist's Leave, a dead message about the departing process whose
 * From is the process itself, broadcast before it stops. The reference has no leave: every departure is a failure that
 * the others must detect. At the current round (the round counter does not advance; no random draws) the leavers are the
 * distinct listed ids that are up (a repeated id leaves once, a down id is ignored). Every leaver goes down as by a
 * SWIM_EV_CRASH at this round (alive = 0, last_crash = round) and back_at = 0, so the seeded churn never brings it back
 * (a SWIM_EV_REJOIN does, with self_inc + 1). Its row, buffer and self_inc are kept. Then each member m that leaver L
 * holds Alive or Suspect and that is up receives Dead(self_inc_L, L, from = L), handled exactly as a SWIM_EV_INJECT
 * datagram at this round; a recipient applies its leavers' records in ascending leaver id. The gossip memberlist's Leave
 * waits for is condensed into the call: a "flushed" leave. No membership changes: the mail graph and the checkpoint stay
 * valid. Every id is checked before anything changes (id < N, at most 2^31 - 1 ids; SWIM_EINVAL otherwise); n = 0 is a
 * no-op. SWIM_ESTATE as for swim_sim_join. On a sharded handle a collective: every rank is given the same global list;
 * outputs are this rank's (the leavers it owns, its recipients' records), their sums the single-shard ones.
 * Outputs may be NULL: *n_left = leavers, *n_delivered = (recipient, leaver) records applied or rejected. */
int swim_sim_leave(swim_sim_t *sim, const uint32_t *nodes, size_t n, uint64_t *n_left, uint64_t *n_delivered);

/* Bulk copies of one state array (SWIM_ARR_*) between device and a host buffer of exactly
 * `bytes` bytes. set_array(SWIM_ARR_NBR) is rejected: use swim_sim_set_view. */
int swim_sim_get_array(swim_sim_t *sim, int arr, void *host_buf, size_t bytes);
int swim_sim_set_array(swim_sim_t *sim, int arr, const void *host_buf, size_t bytes);
int swim_sim_array_bytes(const swim_sim_t *sim, int arr, size_t *bytes);

/* Order-independent 64-bit digest of this rank's state (sum mod 2^64 of a mixed hash per node, per view
 * slot and per buffered record, keyed by global indices: DESIGN.md 2.4); the digests of all ranks add up
 * to the single-GPU digest. dumpStore's content (Util.hs:64-74) in checkable form. */
int swim_sim_digest(swim_sim_t *sim, uint64_t *digest);

/* Copy min(n, SWIM_CTR__COUNT) cumulative counters of this rank. */
int swim_sim_counters(swim_sim_t *sim, uint64_t *out, size_t n);

/* counters + digest + convergence count in one call and ONE synchronisation (any output may be NULL): the
 * per-round read-back of a convergence-study loop. */
int swim_sim_observe(swim_sim_t *sim, uint64_t *counters, size_t n_counters, uint64_t *digest, uint64_t *mismatches);

/* swim_sim_step + the read-back of a study loop in one call: run `rounds` rounds, then deliver the cumulative counters
 * and the convergence count. A kernel chained behind the rounds writes them into pinned host memory mapped into the
 * device and the call polls a sequence number there: no memset, no copy-engine operation and no stream synchronisation
 * on the path (what swim_sim_step_async + swim_sim_observe cost per round at one round per call). */
int swim_sim_step_observe(swim_sim_t *sim, uint32_t rounds, uint64_t *counters, size_t n_counters, uint64_t *mismatches);

/* Convergence detector: number of (live observer, member) view entries on this rank that
 * disagree with the truth (crashed member not Dead, or live member not Alive). */
int swim_sim_mismatches(swim_sim_t *sim, uint64_t *count);

/* Device time in ms of the last swim_sim_step / step_async+sync on this handle, measured
 * with CUDA events on the handle's stream. (swim_sim_step_observe records no events: SWIM_ESTATE after it.) */
int swim_sim_last_step_ms(const swim_sim_t *sim, float *ms);

/* Number of kernels this handle has launched since create (bench.py's `gpu_launches`). */
int swim_sim_launch_count(const swim_sim_t *sim, uint64_t *count);

/* Per-kernel device timing: when enabled, every kernel of swim_sim_step is bracketed by CUDA
 * events on the handle's stream; swim_sim_profile_ms returns the cumulative milliseconds per
 * phase since it was enabled: out[0]=events, out[1]=tick scan (K1a), out[2]=exchange,
 * out[3]=receive (K2), out[4]=tick work (K1b), and the number of rounds profiled in out[5].
 * Costs two event records per kernel. */
#define SWIM_PROFILE_SLOTS 6
int swim_sim_set_profile(swim_sim_t *sim, int enable);
int swim_sim_profile_ms(swim_sim_t *sim, double *out, size_t n);

/* Phase timeline of the fused per-round kernel (profiling aid): after swim_sim_set_timeline(sim, R) the next R rounds
 * record the device's nanosecond timer at their phase boundaries, 8 words per round — [0] round start, [1] scan done
 * (CTA 0), [2] first grid barrier passed, [3] tick work done (CTA 0), [4] second barrier passed, [5] / [6] arrival of the
 * LAST CTA at the first / second barrier (so [5]-[0] is what the slowest CTA's scan phase took and [2]-[5] the release
 * latency of the barrier), [7] rounds committed by a batched quiet scan; words of phases a round skipped stay 0.
 * R = 0 switches it off. Single-kernel launch path only. */
int swim_sim_set_timeline(swim_sim_t *sim, uint32_t rounds);
int swim_sim_get_timeline(swim_sim_t *sim, uint64_t *out /* [rounds][8] */, size_t rounds);

/* Latency calibration of this GPU, in nanoseconds: out[0] = one grid barrier of the fused kernel's resident wave,
 * out[1] = one dependent global load missing L2 (pointer chase over 512 MB), out[2] = the same hitting L2 (1 MB),
 * out[3] = resident warps of the fused kernel. n >= 4. What bench.py's roofline.latency_floor is built from. */
int swim_sim_calibrate(swim_sim_t *sim, double *out, size_t n);

/* ---- multi-GPU plumbing (one process per GPU; ranks own contiguous node ranges) ------
 * The per-round exchange is one all-to-all of cross-shard piggyback envelopes (the UDP
 * hop of Core.hs:280,286). Rank 0 obtains an id, the host side broadcasts the bytes
 * (torch.distributed / MPI / files), every rank calls swim_sim_connect. */
#define SWIM_NCCL_ID_BYTES 128
int swim_nccl_unique_id(uint8_t id[SWIM_NCCL_ID_BYTES]);
int swim_sim_connect(swim_sim_t *sim, const uint8_t id[SWIM_NCCL_ID_BYTES]);

/* Fused exchange over peer memory (preferred when all ranks share one NVLink/NVSwitch box):
 * instead of staging envelopes for NCCL, K1b raises the in-edge flag and appends the receiver
 * directly in the owner GPU's memory, and K2 pulls the sender's snapshot from the sender GPU's
 * memory (plain NVLink stores and loads, nothing staged); one device-side cross-GPU barrier per round
 * replaces the collective (everything senders write is double-buffered by round parity). Call after
 * swim_sim_set_view: every rank exports a blob (CUDA IPC handles of its mail arrays), the host
 * side all-gathers the blobs in rank order, every rank connects. Without this call (only
 * swim_sim_connect) the staged NCCL all-to-all is used. */
#define SWIM_IPC_BLOB_BYTES 1024
int swim_sim_ipc_export(swim_sim_t *sim, uint8_t blob[SWIM_IPC_BLOB_BYTES]);
int swim_sim_ipc_connect(swim_sim_t *sim, const uint8_t *blobs /* world x SWIM_IPC_BLOB_BYTES */);

/* ====================== scalar API: Core.hs function parity ==========================
 * Each call acts on ONE simulated node's store, executing the same device code as the
 * bulk path (a one-warp launch), so the reference's unit tests (test/Spec.hs) can be
 * restated against the accelerated implementation. */

/* members (Core.hs:76-77): the view of `node` in ascending id order. */
int swim_get_members(swim_sim_t *sim, uint32_t node, swim_member_t *out, size_t cap,
                     size_t *n_out);
/* `swapTVar storeMembers` (Spec.hs:101,112,118,125,134): replace the view of `node`.
 * Members are sorted by id; n <= view_cap. */
int swim_set_members(swim_sim_t *sim, uint32_t node, const swim_member_t *members, size_t n);

/* kRandomMembers (Core.hs:69-74) + shuffle (Util.hs:36-42): alive members not in
 * `excludes` (full structural equality, Types.hs:68), order-preserving pick-and-remove
 * shuffle, take n. Returns min(n, L) members. */
int swim_k_random_members(swim_sim_t *sim, uint32_t node, uint32_t n,
                          const swim_member_t *excludes, size_t n_excludes,
                          swim_member_t *out, size_t cap, size_t *n_out);

/* removeDeadNodes (Core.hs:65-67). */
int swim_remove_dead_nodes(swim_sim_t *sim, uint32_t node);

/* nextSeqNo (Core.hs:49-50) / nextIncarnation (Core.hs:52-53): increment, return new. */
int swim_next_seqno(swim_sim_t *sim, uint32_t node, uint32_t *out);
int swim_next_incarnation(swim_sim_t *sim, uint32_t node, uint32_t *out);

/* suspectNode / deadNode / aliveNode (Core.hs:189-218): apply one message to the node's
 * view. *has_out = 1 and *out = the message to re-broadcast (`Just`), else 0 (`Nothing`).
 * A message of the wrong constructor returns SWIM_EINVAL (reference: `undefined`). */
int swim_suspect_node(swim_sim_t *sim, uint32_t node, const swim_message_t *msg,
                      swim_message_t *out, int *has_out);
int swim_dead_node(swim_sim_t *sim, uint32_t node, const swim_message_t *msg,
                   swim_message_t *out, int *has_out);
int swim_alive_node(swim_sim_t *sim, uint32_t node, const swim_message_t *msg,
                    swim_message_t *out, int *has_out);

/* `process` of handleUDPMessage (Core.hs:89-117) for one decoded message from
 * (sender_addr, sender_port): writes the resulting Gossip values. */
int swim_handle_message(swim_sim_t *sim, uint32_t node, uint32_t sender_addr,
                        uint16_t sender_port, const swim_message_t *msg,
                        swim_gossip_t *out, size_t cap, size_t *n_out);

/* disseminate's `Broadcast msg -> enqueue msg` branch (Core.hs:131,136-138; a FIXME no-op in the reference):
 * put a Suspect/Alive/Dead message into the node's piggyback buffer, from where the bulk rounds send
 * it `retransmit` times. swim_get_broadcasts reads the buffer back, newest first (what the next
 * compound Envelope to a ping target would carry). */
int swim_broadcast(swim_sim_t *sim, uint32_t node, const swim_message_t *msg);
int swim_get_broadcasts(swim_sim_t *sim, uint32_t node, swim_message_t *out, size_t cap, size_t *n_out);

/* The two per-period steps a real-time node runs besides the probe (`failureDetector`, Core.hs:233-241), for ONE store:
 * swim_tick_timers — the suspicion countdown the reference leaves as a FIXME (`need a timer to mark this node as dead
 *   after suspect timeout`, Core.hs:141): every Suspect entry's timer - 1; an entry reaching 0 becomes Dead and
 *   Dead(incarnation, member, from = node) is enqueued for dissemination. *n_expired (may be NULL) = entries that died.
 * swim_take_broadcasts — the piggyback payload of the next outgoing message (the compound Envelope of Types.hs:96-119
 *   that `disseminate`'s FIXME, Core.hs:136, never builds): the buffer as swim_get_broadcasts returns it, after which
 *   one of each record's `retransmit` transmissions is spent; records at 0 leave the buffer.
 * Both run the same device code as phases T1 / T4 of the bulk rounds (DESIGN.md 2.2). */
int swim_tick_timers(swim_sim_t *sim, uint32_t node, uint32_t *n_expired);
int swim_take_broadcasts(swim_sim_t *sim, uint32_t node, swim_message_t *out, size_t cap, size_t *n_out);

/* ====================== wire codec: Types.hs parity ==================================
 * Envelope framing (Types.hs:96-119) around msgpack-of-aeson-generic bodies
 * (Types.hs:147-155). Names travel as strings on the wire. */
#define SWIM_NAME_MAX 255u
typedef struct swim_wire_message {
  uint8_t kind; /* SWIM_MSG_PING .. SWIM_MSG_DEAD */
  uint8_t payload_len;
  uint16_t port;
  uint32_t seq_no;
  uint32_t target; /* IndirectPing.target / Alive.addr */
  int64_t incarnation;
  uint8_t payload[SWIM_ACK_PAYLOAD_MAX];
  char node[SWIM_NAME_MAX + 1];      /* NUL-terminated */
  char dead_from[SWIM_NAME_MAX + 1]; /* NUL-terminated */
} swim_wire_message_t;

/* `encode (Envelope msgs)`: n == 1 -> type byte + body; n >= 2 -> compound. */
int swim_envelope_encode(const swim_wire_message_t *msgs, size_t n, uint8_t *buf, size_t cap,
                         size_t *len);
/* `decode :: Either String Envelope`; on failure returns SWIM_EDECODE and
 * swim_last_error(NULL) carries the reference's message (Types.hs:115,118). */
int swim_envelope_decode(const uint8_t *buf, size_t len, swim_wire_message_t *msgs,
                         size_t cap, size_t *n_out);

/* ====================== simulated traffic as real datagrams (SURVEY 8(f)-2) ===========
 * The piggyback envelopes of the LAST executed round, encoded exactly as the reference would put them
 * on the wire (Types.hs:96-119,151-155): one datagram per (sender, receiver), a single message or a
 * compound Envelope of the sender's buffered Suspect/Alive/Dead records. Simulated nodes have no
 * names; on the wire node i is called "n<i>" (decimal), Alive carries addr = i and port = base_port.
 * Host-side encoder (the codec above, one sender per OpenMP thread) over device snapshots; single
 * shard only. Datagram k occupies buf[index[k].offset .. +index[k].length). */
typedef struct swim_datagram {
  uint32_t src, dst;   /* simulated sender and receiver */
  uint32_t length;     /* bytes */
  uint32_t n_messages; /* records in the envelope */
  uint64_t offset;     /* into buf */
} swim_datagram_t;
int swim_sim_export_round(swim_sim_t *sim, uint8_t *buf, size_t cap, swim_datagram_t *index, size_t index_cap,
                          size_t *n_datagrams, size_t *n_bytes);

/* The reverse direction: decode one captured datagram (names "n<i>") addressed to `node` and queue its
 * Suspect/Alive/Dead messages as SWIM_EV_INJECT events for `round` (Ping/IndirectPing/Ack carry no state
 * and are skipped). A decode failure returns SWIM_EDECODE (Core.hs:86-87). */
int swim_sim_inject_datagram(swim_sim_t *sim, uint32_t round, uint32_t node, const uint8_t *data, size_t len);

#if defined(__GNUC__)
#pragma GCC visibility pop
#endif
#ifdef __cplusplus
}
#endif
#endif /* SWIM_H_ */
