// swim_device.cuh — sm_90a device code of the SWIM bulk simulator.
//
// One simulated node == one `Store` (reference Types.hs:53-60). Per round every node runs
//   K1a scan : kRandomMembers/shuffle target selection (Core.hs:69-74, Util.hs:36-42) and the direct
//              Ping/Ack of probeNode' (Core.hs:243-247)
//   K1b work : suspicion countdown (Core.hs:141 FIXME), k IndirectPings, local suspicion
//              (Core.hs:247-254), piggyback send (Core.hs:127-138)
//   K2  recv : process / suspectOrDeadNode' / aliveNode (Core.hs:89-121,142-218)
//
// Mapping to the hardware (integer / indexing work, no tensor cores by design):
//   * K1a streams ONE 4-byte summary word per node (up, piggyback count, min(L, 4), suspect, exposed); a lane handles 8
//     nodes (2 independent 128-bit loads); only exposed nodes (a crashed process in an Alive slot) gather their 16-byte
//     `meta` record (alive / suspect / crashed-member bitmaps) and spend Philox4x32-10 blocks — four nodes share a
//     block — and r-th-set-bit picks; a warp covers 1 KB contiguous.
//   * nodes that need more than the read-only probe (a countdown to run, a failed probe, a non-empty
//     piggyback buffer) go to a work list (warp-aggregated append) and are handled warp-per-node:
//     lane s owns view slot s, the piggyback buffer is staged in shared memory, membership lookups
//     are a ballot over the id row.
//   * mail is delivered without sorting or contended atomics: the sender raises a byte flag on the
//     static in-edge (i -> j) of the receiver's sorted in-list and records j in its own candidate
//     slot; a receiver is claimed once (per-receiver stamp), walks its flags in ascending sender
//     order and pulls the sender's snapshot — from local HBM or, across shards, from the peer GPU's
//     HBM over NVLink.
//   * default launch: one resident wave per event-free stretch of rounds. round_kernel: per round (receive of the round
//     before || K1a) | grid barrier | K1b | grid barrier; round_kernel_x (long single-shard stretches): per round ONE
//     interval (mail of the round before + K1b + K1a of the next round) and one grid barrier. The same passes exist as
//     separate kernels for profiling and the staged NCCL exchange.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/swim.h"

// Kernel launches and CTA-shared arrays go through two macros so that tests/emu (a SIMT emulator + CUDA runtime stubs,
// test infrastructure) can compile these very sources for the CPU. In a CUDA build they expand to the plain syntax.
#ifdef SWIM_EMU
#define SWIM_LAUNCH(kernel, grid, block, stream, ...) swim_emu::launch((grid), (block), [=] { kernel(__VA_ARGS__); })
#define SWIM_SHARED_1D(T, name, n) static char name##_tag; T *name = (T *)swim_emu::shared(&name##_tag, sizeof(T) * (n))
#define SWIM_SHARED_2D(T, name, n0, n1) static char name##_tag; T (*name)[n1] = (T (*)[n1])swim_emu::shared(&name##_tag, sizeof(T) * (n0) * (n1))
#else
#define SWIM_LAUNCH(kernel, grid, block, stream, ...) kernel<<<(grid), (block), 0, (stream)>>>(__VA_ARGS__)
#define SWIM_SHARED_1D(T, name, n) __shared__ T name[n]
#define SWIM_SHARED_2D(T, name, n0, n1) __shared__ T name[n0][n1]
#endif

namespace swim {

struct DevEvent;

// CTA shape of the per-round kernels: 8 warps x 4 CTAs per SM by default. -DSWIM_WARPS_PER_BLOCK=16|32 (build.py: env
// SWIM_WPB) keeps 32 resident warps per SM at 64 registers with fewer, larger CTAs: fewer arrivals on the grid barrier.
#ifndef SWIM_WARPS_PER_BLOCK
#define SWIM_WARPS_PER_BLOCK 8
#endif
constexpr int kWarpsPerBlock = SWIM_WARPS_PER_BLOCK;
constexpr int kMinBlocks = 32 / kWarpsPerBlock;
static_assert(kWarpsPerBlock == 8 || kWarpsPerBlock == 16 || kWarpsPerBlock == 32, "SWIM_WARPS_PER_BLOCK");
constexpr int kThreads = kWarpsPerBlock * 32;
constexpr unsigned kFull = 0xFFFFFFFFu;
// Ranks drift (host-side setup, first-launch module loads): a peer may legitimately be seconds late.
constexpr long long kPeerWaitCycles = 120000000000ll; // ~60 s at 2 GHz, then the wait gives up and reports
#define SWIM_MAX_WORLD 8

// Philox counter purposes (DESIGN.md §2.3). TARGET and LOSS0 blocks are shared by the four nodes
// 4g..4g+3 (counter word 1 = node >> 2, draw = word node & 3): one Philox call serves four probes.
enum : uint32_t { P_TARGET = 0, P_LOSS0 = 1, P_SCALAR = 2, P_TOPO = 3, P_PROXY = 4, P_LOSS = 5, P_RR = 6, P_CHURN = 7, P_TARGETS = 8, P_LOSSD = 9,
                   P_PUSHPULL = 10, P_TOPOSYM = 11 };

struct SimDev {
  uint32_t N, first, n, cap;
  uint32_t k, fanout, B, S, T, loss_ppm;
  uint32_t P;                // probes per node per round (cfg.probes_per_round; 1 = SWIM)
  uint32_t flags;            // SWIM_F_* protocol variants
  // suspicion countdown in the state byte: liveness | timer << 2 (6 bits); with cfg.suspicion_max (Lifeguard-style dynamic
  // timeout) liveness | timer << 2 (4 bits) | confirmations << 6
  uint32_t S_arm, tmask, lg; // rounds a new suspicion starts with; timer mask (63 / 15); dynamic timeout on
  uint32_t lg_delta[4];      // lg_delta[c]: what the c-th confirmation takes off the countdown
  uint32_t key0, key1;
  uint32_t round;
  uint32_t nrounds;          // round_kernel: consecutive rounds in this launch (>= 1)
  uint32_t world, rank, per; // per = nodes per shard
  uint8_t *alive;            // [N]
  uint32_t *back_at;         // [N] churn: round at which a crashed process rejoins (0 = none)
  uint32_t *last_crash, *last_rejoin; // [N] round of the last up -> down / down -> up transition (0 = never)
  uint32_t churn_ppm, rejoin_min, rejoin_span; // seeded churn (phase C); rejoin delay = rejoin_min + U[0, span)
  struct DevEvent *churn_ev; // [churn_cap] crash / rejoin events of the round, generated on the device
  uint32_t *churn_cnt;       // [0] their number (the host clears it on the stream ahead of every round)
  uint32_t churn_cap;
  uint32_t *self_inc;        // [n]
  uint32_t *seqno;           // [n]
  uint32_t *nbr;             // [n*cap]
  uint8_t *vst;              // [n*cap] liveness | timer<<2
  uint32_t *vinc;            // [n*cap]
  uint32_t *vlast;           // [n*cap]
  uint4 *pb;                 // [n*B] {member, inc, from, kind | ttl<<8}
  uint8_t *pb_cnt;           // [n]
  uint4 *out;                // [2][per*B] snapshot sent this round (round parity)
  uint8_t *out_cnt;          // [2][per]
  uint32_t *ridx;            // [n*cap] index of edge (i,s) in the receiver's in-list
  uint32_t *in_off;          // [n+1]
  uint32_t *in_src;          // [E] sender ids, ascending per receiver
  uint8_t *eflag;            // [E] 1 = sender mailed this round
  uint4 *meta;               // [n*W] per 32 slots: {alive bitmap, suspect bitmap, crashed-member bitmap, unused}
  // [n] per node, what the scan reads (a lane's Philox group of four nodes is one 16-byte load): byte 0 = process up,
  // byte 1 = piggyback count, byte 2 = min(L, 4) (L = Alive slots; P <= SWIM_MAX_PROBES = 4) | some slot Suspect << 3 |
  // exposed << 4. Exposed: a crashed process may sit in an Alive slot (am & td != 0). Every other field is exact; the
  // exposed bit may be set spuriously (that costs the scan one meta gather) but is never clear for an exposed node.
  uint32_t *nsum;
  uint32_t *obs_off;         // [N+1] observers of member m among this shard's rows ...
  uint32_t *obs_slot;        // [n*cap] ... as linear slot indices l*cap + s
  uint32_t *wl, *wl_cnt;     // work lists of K1b [2][n] (round parity); counters indexed by round % 3
  // one-barrier round kernel (round_kernel_x): a round's work list is still being extended (by the nodes whose mail
  // made them need K1b after all) while its items are walked, so the barrier that completes the list freezes its length in
  // wl_n[round % 3]; workbits: bit l of slot r % 3 = local node l is on the work list of round r
  uint32_t *wl_n;            // [3]
  uint32_t *workbits;        // [3][mbw]
  uint2 *rl;                 // [2][n*fanout] recipient slots (round parity), slot = item*fanout + f:
                             //   .x = local receiver (bit 31 set: sent, but not delivered — see `bloom`), .y = the sender
  // Mail bitmap (fused kernel only, `fused` != 0): bit l of slot (r % 3) = local node l was delivered mail in round r.
  // The scan of round r + 1 leaves such nodes alone — their views are being updated by the warps that apply the mail in
  // the same phase, and those warps take the node's tick decision themselves afterwards. THREE slots, not two: slot r % 3
  // is cleared after the scan barrier of round r + 1, and that barrier may already contain the cross-GPU handshake of
  // round r + 1 (a rank without work), after which a peer is free to mark receivers of round r + 2 — in slot (r + 2) % 3,
  // never in the one being cleared. (With two slots a 2-GPU parity test lost marks exactly this way.)
  uint32_t *mailbits;        // [3][mbw]
  uint32_t *mailbits_p[SWIM_MAX_WORLD];
  uint32_t mbw;              // words per parity = ceil(per / 32), the same on every rank
  uint32_t fused;            // this launch is round_kernel or round_kernel_x (senders mark their receivers in the mail bitmap)
  uint2 *cl;                 // [2][n*fanout] the delivered slots of a round, compact (what K2 walks): {receiver, sender}
  uint32_t *ncand;           // [3] (round % 3) length of this round's compact list
  // Static membership filter of every node's view row (all N nodes, replicated on every rank): 512 W bits per node, two
  // hash positions per member id (2 % false positives on a full row). A sender tests its records against the recipient's filter: an envelope none of whose
  // records is about the recipient or about a member the recipient may know cannot change the recipient's state
  // (Core.hs:147-148 `we don't know this node. ignore`), so it is counted and dropped at the sender instead of being
  // flagged, listed and walked by K2. False positives are delivered and ignored there; there are no false negatives.
  const uint32_t *bloom;     // [N * 16 W]
  // Round-parity double buffering: everything a round's senders write for its receivers exists twice
  // (index = round & 1), so round r+1's senders never touch what round r's receivers still read and ONE
  // cross-GPU barrier per round (between K1b and K2) is enough.
  uint32_t estride;          // eflag parity stride of this rank (>= E)
  uint32_t *claim;           // [n] round stamp: a receiver is processed by exactly one warp per round
  // cross-shard delivery over peer memory (NVLink): the same arrays of every rank, mapped here with CUDA
  // IPC; entry [rank] is this rank's own array. Remote traffic is fire-and-forget stores only.
  uint8_t *eflag_p[SWIM_MAX_WORLD];      // [2][estride_p[r]] in-edge mail flags
  uint32_t estride_p[SWIM_MAX_WORLD];
  const uint4 *out_p[SWIM_MAX_WORLD];    // [2][per*B] sender snapshots
  const uint8_t *out_cnt_p[SWIM_MAX_WORLD]; // [2][per]
  uint32_t *bar_err;                     // set by a cross-GPU / grid wait that timed out
  uint32_t *gbar;                        // [2] grid barrier of round_kernel: arrival count, generation
  uint32_t *qm;                          // [3] busy masks of round_kernel's batched quiet scans (batch number % 3)
  uint32_t qbatch;                       // rounds per batched quiet scan (<= 8); 0 or 1 = off
  uint32_t *rlr_p[SWIM_MAX_WORLD];       // [2][world][rcap] receiver ids appended by each source rank
  uint32_t *rcnt_p[SWIM_MAX_WORLD];      // [2][world] their counts, published by the barrier kernel
  uint32_t *bar_p[SWIM_MAX_WORLD];       // [world] cross-GPU barrier words
  uint32_t *rlr, *rcnt;                  // this rank's own receive-side arrays
  uint32_t *xcnt;                        // [world] envelopes sent to each rank this round (sender side)
  uint32_t rcap;                         // capacity of one (parity, source) remote list
  uint32_t p2p;                          // 1 = fused peer-memory exchange, 0 = staged NCCL all-to-all
  // staged exchange through NCCL (baseline path)
  uint4 *xsend;              // [world][xcap] envelopes {ridx, cnt, src, -} + B records, bucketed by rank
  uint32_t *xsend_cnt;       // [world + 1]; the last word is the bucket-overflow flag
  uint4 *xrecv;              // received envelopes, all source ranks back to back
  uint32_t *eslot;           // [E] exchange-buffer slot of the envelope raised on in-edge e
  uint32_t xcap;             // envelopes per destination bucket
  unsigned long long *ctr;   // [SWIM_CTR__COUNT]
  // in-kernel phase timeline (swim_sim_set_timeline; null = off): %globaltimer of CTA 0 at the phase boundaries of
  // round_kernel, 8 words per round starting at round tl_round0
  unsigned long long *tl;
  uint32_t tl_cap, tl_round0;
};


// ------------------------------------------------------------------ programmatic dependent launch
// The per-round kernels are launched with cudaLaunchAttributeProgrammaticStreamSerialization: the
// next kernel's CTAs may be scheduled while this one drains; pdl_wait() blocks until the previous
// grid has completed and its writes are visible, pdl_launch() lets the following grid start early.
#ifdef SWIM_EMU
__device__ __forceinline__ void pdl_wait() {}
__device__ __forceinline__ void pdl_launch() {}
#else
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
#endif

// System-scope release / acquire on one word: what the cross-GPU handshake of the fused exchange needs (a rank's round
// word is stored with release semantics after its mail — plain stores into peer memory, ordered before it by the CTA
// barrier and a fence.sys of the arriving threads —, and polled with acquire semantics by the owner). sm_70+ PTX.
__device__ __forceinline__ void st_release_sys(uint32_t *p, uint32_t v) {
#ifdef SWIM_EMU
  __atomic_store_n(p, v, __ATOMIC_RELEASE);
#else
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#endif
}
// relaxed system-scope loads (never served from a stale L1 line): peer-GPU memory that changes from round to round
__device__ __forceinline__ uint4 ld_sys_u4(const uint4 *p) {
#ifdef SWIM_EMU
  return *p;
#else
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ uint32_t ld_sys_u8(const uint8_t *p) {
#ifdef SWIM_EMU
  return *p;
#else
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u8 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t *p) {
#ifdef SWIM_EMU
  return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#else
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
#endif
}

// Bounded waits: a wait that runs out of time sets *bar_err and gives up; every later wait of the launch then gives up
// quickly (it looks at the word every 4096 polls), so a lost peer or a grid that is not co-resident costs ONE time-out and
// swim_sim_sync reports it — not one time-out per barrier of every remaining round.
__device__ __forceinline__ bool wait_expired(const SimDev &d, long long t0, long long limit, uint32_t &polls, uint32_t code) {
  if ((++polls & 255u) != 0) return false;
  if (clock64() - t0 > limit) { *d.bar_err = code; return true; }
  return (polls & 4095u) == 0 && *(volatile uint32_t *)d.bar_err != 0; // (the word lives in mapped host memory: look rarely)
}

// Phase timeline of round_kernel: one thread of CTA 0 stores %globaltimer (ns) at each phase boundary. Slots per round:
// 0 start, 1 scan done (CTA 0), 2 barrier 1 passed (every CTA's scan done), 3 work done (CTA 0), 4 barrier 2 passed,
// 5 / 6 the LAST CTA's arrival at the first / second barrier (tl_mark_last), 7 = number of rounds a batched quiet scan
// committed at this round.
__device__ __forceinline__ void tl_mark(const SimDev &d, uint32_t round, int slot, unsigned long long val = ~0ull) {
#ifndef SWIM_EMU
  if (d.tl && blockIdx.x == 0 && threadIdx.x == 0 && round - d.tl_round0 < d.tl_cap) {
    if (val == ~0ull) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(val));
    d.tl[(size_t)(round - d.tl_round0) * 8 + slot] = val;
  }
#endif
}

// the same stamp from thread 0 of ANY CTA: slots 5 / 6 = when the LAST CTA arrived at the round's first / second grid
// barrier (what a phase really took; the difference to slot 2 / 4 is the release latency of the barrier itself)
__device__ __forceinline__ void tl_mark_last(const SimDev &d, uint32_t round, int slot) {
#ifndef SWIM_EMU
  if (d.tl && slot >= 0 && round - d.tl_round0 < d.tl_cap) {
    unsigned long long val;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(val));
    d.tl[(size_t)(round - d.tl_round0) * 8 + slot] = val;
  }
#endif
}

// ------------------------------------------------------------------ pure integer helpers
// Philox and the slot-selection arithmetic are host+device so that tests/device_helpers_harness.cu can run the very
// same functions on the CPU (no GPU in the build container) against the oracle's independent statements.
#ifdef __CUDA_ARCH__
#define SWIM_UMULHI(a, b) __umulhi((a), (b))
#define SWIM_POPC(x) __popc(x)
#define SWIM_FFS(x) __ffs(x)
#define SWIM_ROTR(x, n) __funnelshift_r((x), (x), (n))
#else
#define SWIM_UMULHI(a, b) ((uint32_t)(((uint64_t)(a) * (uint64_t)(b)) >> 32))
#define SWIM_POPC(x) __builtin_popcount(x)
#define SWIM_FFS(x) __builtin_ffs((int)(x))
#define SWIM_ROTR(x, n) (((n) & 31u) ? (((x) >> ((n) & 31u)) | ((x) << (32u - ((n) & 31u)))) : (x))
#endif
#define SWIM_HD __host__ __device__ __forceinline__

// ------------------------------------------------------------------ Philox4x32-10
SWIM_HD uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = SWIM_UMULHI(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    uint32_t hi1 = SWIM_UMULHI(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}
SWIM_HD uint32_t word_of(uint4 v, int i) {
  return i == 0 ? v.x : i == 1 ? v.y : i == 2 ? v.z : v.w;
}
// randomR (0, L-1) (Util.hs:40) on the Philox stream
SWIM_HD uint32_t bounded(uint32_t x, uint32_t L) { return SWIM_UMULHI(x, L); }

// position of the r-th (0-based) set bit of m; requires r < popc(m)
SWIM_HD uint32_t nth_set(uint32_t m, uint32_t r) {
  uint32_t pos = 0, c;
  c = SWIM_POPC(m & 0xFFFFu); if (r >= c) { r -= c; pos += 16; m >>= 16; }
  c = SWIM_POPC(m & 0xFFu);   if (r >= c) { r -= c; pos += 8;  m >>= 8; }
  c = SWIM_POPC(m & 0xFu);    if (r >= c) { r -= c; pos += 4;  m >>= 4; }
  c = SWIM_POPC(m & 0x3u);    if (r >= c) { r -= c; pos += 2;  m >>= 2; }
  if (r >= (m & 1u)) pos += 1;
  return pos;
}

// `shuffle` (Util.hs:36-42) on a W-word bitmask of candidate slots: pick the r-th remaining
// candidate in ascending slot order and remove it (order preserved by construction).
template <int W>
SWIM_HD uint32_t pick_remove(uint32_t (&m)[W], uint32_t r) {
#pragma unroll
  for (int w = 0; w < W; ++w) {
    uint32_t c = SWIM_POPC(m[w]);
    if (r < c) {
      uint32_t b = nth_set(m[w], r);
      m[w] &= ~(1u << b);
      return w * 32 + b;
    }
    r -= c;
  }
  return 0; // unreachable when r < total
}

// The same pick by a whole warp (K1b: warp per node, every lane holds the same mask and rank): lane s answers for bit s —
// "am I set, with exactly r set bits below me?" — and a ballot names the winner: ~10 instructions instead of the ~60 of the
// scalar five-step search. Must be called by all 32 lanes with warp-uniform arguments.
template <int W>
__device__ __forceinline__ uint32_t pick_remove_warp(uint32_t (&m)[W], uint32_t r, int lane) {
#pragma unroll
  for (int w = 0; w < W; ++w) {
    const uint32_t c = SWIM_POPC(m[w]);
    if (r < c) {
      const bool mine = (m[w] >> lane & 1u) && (uint32_t)SWIM_POPC(m[w] & ((1u << lane) - 1u)) == r;
      const uint32_t b = (uint32_t)__ffs(__ballot_sync(0xFFFFFFFFu, mine)) - 1u;
      m[w] &= ~(1u << b);
      return w * 32 + b;
    }
    r -= c;
  }
  return 0; // unreachable when r < total
}

template <int W>
SWIM_HD void clear_slot(uint32_t (&m)[W], uint32_t slot) {
#pragma unroll
  for (int w = 0; w < W; ++w)
    if ((uint32_t)w == (slot >> 5)) m[w] &= ~(1u << (slot & 31));
}

// ---- SWIM_F_ROUND_ROBIN (`-- FIXME: move from random to robust scheme`, Core.hs:232; SWIM paper 4.3) ----------------
// Rounds are grouped in epochs of cap = 32 W rounds; in epoch e a node walks its view in the order slot(p) = p xor b,
// p = (round + r) mod cap, with (b, r) drawn once per (epoch, node); the target is the first Alive slot at or after p in
// that order (cyclic). Stateless — nothing to store or write back — and every position comes up once per epoch.
// bit i of the result = bit (i xor b) of m (b < 32): five conditional butterfly stages
SWIM_HD uint32_t xor_permute(uint32_t m, uint32_t b) {
  if (b & 1u)  m = ((m & 0x55555555u) << 1) | ((m >> 1) & 0x55555555u);
  if (b & 2u)  m = ((m & 0x33333333u) << 2) | ((m >> 2) & 0x33333333u);
  if (b & 4u)  m = ((m & 0x0F0F0F0Fu) << 4) | ((m >> 4) & 0x0F0F0F0Fu);
  if (b & 8u)  m = ((m & 0x00FF00FFu) << 8) | ((m >> 8) & 0x00FF00FFu);
  if (b & 16u) m = (m << 16) | (m >> 16);
  return m;
}

// requires at least one bit set in am[]
template <int W>
SWIM_HD uint32_t rr_pick(const uint32_t (&am)[W], uint32_t word, uint32_t round) {
  constexpr uint32_t capm = 32u * W - 1u;
  const uint32_t b = word & capm, r = (word >> 16) & capm, p = (round + r) & capm;
  if constexpr (W == 1) {
    const uint32_t pm = xor_permute(am[0], b);
    const uint32_t x = SWIM_ROTR(pm, p); // rotate position p to bit 0
    return ((p + (uint32_t)SWIM_FFS(x) - 1u) & 31u) ^ b;
  } else {
    uint32_t pm[W];
#pragma unroll
    for (int w = 0; w < W; ++w) {
      uint32_t src = 0;
#pragma unroll
      for (int v = 0; v < W; ++v)
        if ((uint32_t)v == ((uint32_t)w ^ (b >> 5))) src = am[v];
      pm[w] = xor_permute(src, b & 31u);
    }
    const uint32_t pw = p >> 5, po = p & 31u;
#pragma unroll
    for (int t = 0; t <= W; ++t) {
      const uint32_t w = (pw + t) & (W - 1);
      uint32_t m = 0;
#pragma unroll
      for (int v = 0; v < W; ++v)
        if ((uint32_t)v == w) m = pm[v];
      if (t == 0) m &= ~0u << po;
      if (t == W) m &= (1u << po) - 1u;
      if (m) return (w * 32u + (uint32_t)SWIM_FFS(m) - 1u) ^ b;
    }
    return 0; // unreachable when a bit is set
  }
}

// ------------------------------------------------------------------ records
__device__ __forceinline__ uint4 make_rec(uint32_t member, uint32_t inc, uint32_t from, uint32_t kind) {
  return make_uint4(member, inc, from, kind);
}
__device__ __forceinline__ uint32_t rec_kind(uint4 r) { return r.w & 0xFFu; }
__device__ __forceinline__ uint32_t rec_ttl(uint4 r) { return (r.w >> 8) & 0xFFu; }

// Warp-cooperative piggyback buffer in shared memory: lane q < cnt owns record q, newest
// first. This is the `Broadcast` branch of disseminate (Core.hs:131) that the reference
// leaves as `enqueue _msg = return ()` (Core.hs:136-138).
struct PbStage {
  uint4 *s;     // shared memory, 32 entries for this warp
  uint32_t cnt; // uniform across the warp
  bool dirty;
};

__device__ __forceinline__ void pb_load(PbStage &p, const SimDev &d, uint32_t l, int lane) {
  // count and records are fetched together (records speculatively: B lanes, whatever the count)
  uint4 mine = make_uint4(0, 0, 0, 0);
  if ((uint32_t)lane < d.B) mine = d.pb[(size_t)l * d.B + lane];
  p.cnt = d.pb_cnt[l];
  p.dirty = false;
  __syncwarp();
  if ((uint32_t)lane < p.cnt) p.s[lane] = mine;
  __syncwarp();
}

// Fields of the summary word SimDev::nsum.
constexpr uint32_t kNsPb = 0xFF00u, kNsSus = 1u << 19, kNsExposed = 1u << 20;
constexpr uint32_t kNsBusy = kNsPb | kNsSus; // the word alone sends a live node to K1b
__device__ __forceinline__ uint32_t ns_up(uint32_t s) { return s & 0xFFu; }
__device__ __forceinline__ uint32_t ns_alive(uint32_t s) { return s >> 16 & 7u; } // min(L, 4)

// atomic_ns: the caller is event_kernel, where another warp's crash event may set the exposed bit of the same summary
// word at the same time; there every update of the word is an atomic on all 32 bits.
__device__ __forceinline__ void pb_store(PbStage &p, const SimDev &d, uint32_t l, int lane, bool atomic_ns = false) {
  if (!p.dirty) return;
  __syncwarp();
  if ((uint32_t)lane < p.cnt) d.pb[(size_t)l * d.B + lane] = p.s[lane];
  if (lane == 0) {
    d.pb_cnt[l] = (uint8_t)p.cnt;
    if (atomic_ns) { atomicAnd(&d.nsum[l], ~kNsPb); atomicOr(&d.nsum[l], p.cnt << 8); }
    else reinterpret_cast<uint8_t *>(d.nsum + l)[1] = (uint8_t)p.cnt;
  }
}

__device__ __forceinline__ void pb_enqueue(PbStage &p, const SimDev &d, uint4 rec, int lane,
                                           uint32_t &dropped) {
  rec.w = (rec.w & 0xFFu) | (d.T << 8);
  uint4 mine = make_uint4(0, 0, 0, 0);
  bool have = (uint32_t)lane < p.cnt;
  if (have) mine = p.s[lane];
  unsigned same = __ballot_sync(kFull, have && mine.x == rec.x);
  uint32_t pos = same ? (uint32_t)(__ffs(same) - 1) : p.cnt; // slot that disappears
  uint32_t ncnt = same ? p.cnt : p.cnt + 1;
  if (!same && p.cnt == d.B) { pos = d.B - 1; ncnt = d.B; if (lane == 0) ++dropped; }
  __syncwarp();
  if (have && (uint32_t)lane < pos) p.s[lane + 1] = mine; // shift older records down
  if (lane == 0) p.s[0] = rec;                           // newest first
  p.cnt = ncnt;
  p.dirty = true;
  __syncwarp();
}

// ------------------------------------------------------------------ view row, warp-per-node
// lane owns slots {w*32 + lane}.
template <int W>
struct Row {
  uint32_t nb[W];
  uint32_t inc[W];
  uint32_t st[W];     // packed liveness | timer<<2
  uint32_t touched;   // bit w: slot (w, lane) changed liveness/incarnation -> write st, inc, last
  uint32_t ticked;    // bit w: only the countdown of slot (w, lane) changed -> write st
};

template <int W>
__device__ __forceinline__ void row_load(Row<W> &r, const SimDev &d, uint32_t l, int lane) {
  size_t base = (size_t)l * d.cap + lane;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    r.nb[w] = d.nbr[base + w * 32];
    r.st[w] = d.vst[base + w * 32];
    r.inc[w] = d.vinc[base + w * 32];
  }
  r.touched = 0;
  r.ticked = 0;
}

// td: the row's crashed-member bits, for the exposed bit of the summary word. In the round kernels they cannot change, so
// the byte is stored exactly; in event_kernel (atomic_ns) a crash event of another warp may be setting them, so the
// exposed bit is only ever set there (mark_observers sets it on every crash).
template <int W>
__device__ __forceinline__ void row_store(const Row<W> &r, const SimDev &d, uint32_t l, int lane, uint32_t round,
                                          const uint32_t (&td)[W], bool atomic_ns = false) {
  size_t base = (size_t)l * d.cap + lane;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    if (r.touched & (1u << w)) {
      d.vst[base + w * 32] = (uint8_t)r.st[w];
      d.vinc[base + w * 32] = r.inc[w];
      d.vlast[base + w * 32] = round;
    } else if (r.ticked & (1u << w)) {
      d.vst[base + w * 32] = (uint8_t)r.st[w];
    }
  }
  if (__any_sync(kFull, r.touched != 0)) { // liveness changed somewhere: refresh the row's bitmaps and its summary byte
    uint32_t acc = 0; // L in bits 0-8, some slot Suspect: bit 16, exposed: bit 17 (one register across the loop)
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const unsigned am = __ballot_sync(kFull, (r.st[w] & 3u) == SWIM_ALIVE);
      const unsigned sm = __ballot_sync(kFull, (r.st[w] & 3u) == SWIM_SUSPECT);
      if (lane == 0) {
        uint32_t *m = reinterpret_cast<uint32_t *>(d.meta + (size_t)l * W + w);
        m[0] = am;
        m[1] = sm;
        if constexpr (W >= 8) { // wide rows: the crashed-member word is read back, which keeps td out of this loop's registers
          acc += __popc(am);
          acc |= (sm ? 1u << 16 : 0u) | ((am & m[2]) ? 1u << 17 : 0u);
        }
      }
      if constexpr (W < 8) {
        acc += __popc(am);
        acc |= (sm ? 1u << 16 : 0u) | ((am & td[w]) ? 1u << 17 : 0u);
      }
    }
    if (lane == 0) {
      const uint32_t L = acc & 0x1FFu, b2 = (L < 4u ? L : 4u) | (acc >> 16 & 1u) << 3 | (acc >> 17 & 1u) << 4;
      if (atomic_ns) { atomicAnd(&d.nsum[l], ~(0xFu << 16)); atomicOr(&d.nsum[l], b2 << 16); }
      else reinterpret_cast<uint8_t *>(d.nsum + l)[2] = (uint8_t)b2;
    }
  }
}

// suspectOrDeadNode' (Core.hs:142-187) + aliveNode's known-member completion [Q7], for one
// record delivered to node `self`. Every lane returns the same verdict:
//   0 = `Nothing`; 1 = `Just` *rb (re-broadcast); 2 = unknown member + Alive (Core.hs:206-216
//   would insert; bulk rounds ignore, the scalar call inserts).
template <int W>
__device__ __forceinline__ int row_apply(Row<W> &r, const SimDev &d, uint32_t self, uint32_t &self_inc,
                                         uint4 rec, uint4 &rb, int lane, uint32_t &refutes, bool net = true) {
  const uint32_t kind = rec_kind(rec);
  if (rec.x == self) {
    // own entry is virtual: (Alive, storeIncarnation)
    if (kind == SWIM_MSG_ALIVE) return 0;
    // Core.hs:151 stale incarnation; STRICT_OVERRIDE: a Confirm overrides whatever the others hold -> always refuted
    if (rec.y < self_inc && !((d.flags & SWIM_F_STRICT_OVERRIDE) && kind == SWIM_MSG_DEAD)) return 0;
    uint32_t base = self_inc > rec.y ? self_inc : rec.y;
    self_inc = base + 1;                            // Core.hs:155-166; [Q9] terminating bump
    if (lane == 0) ++refutes;
    rb = make_rec(self, base + 1, 0, SWIM_MSG_ALIVE);
    return 1;
  }
  // Core.hs:144-145 `find ((== name) . memberName) ms` as a ballot over the id row
  int hw = -1, hl = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    unsigned hit = __ballot_sync(kFull, r.nb[w] == rec.x && (r.st[w] & 3u) != SWIM_VACANT);
    if (hit && hw < 0) { hw = w; hl = __ffs(hit) - 1; }
  }
  if (hw < 0) return kind == SWIM_MSG_ALIVE ? 2 : 0; // Core.hs:147-148 unknown: ignore
  uint32_t st_s = 0, inc_s = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    uint32_t a = __shfl_sync(kFull, r.st[w], hl), b = __shfl_sync(kFull, r.inc[w], hl);
    if (w == hw) { st_s = a; inc_s = b; }
  }
  const uint32_t live = st_s & 3u;
  uint32_t nst, ninc = rec.y;
  // [Lifeguard] a Suspect received (net: in a datagram, not raised by this node's own probe) about a member that is
  // already Suspect is `Nothing` for the reference (Core.hs:151,183) and stays so, but with cfg.suspicion_max it counts as
  // a confirmation: the countdown loses lg_delta[c], never below 1 (timeout(c) = max - (max - min) log(c+1) / log 4).
  bool confirm = false;
  if (d.flags & SWIM_F_STRICT_OVERRIDE) { // SWIM paper 4.2 instead of the reference's guards (include/swim.h)
    if (kind == SWIM_MSG_SUSPECT) {
      if (live == SWIM_DEAD || (live == SWIM_ALIVE ? rec.y < inc_s : rec.y <= inc_s)) {
        confirm = live == SWIM_SUSPECT && rec.y == inc_s;
        if (!(confirm && d.lg && net)) return 0;
      }
      nst = SWIM_SUSPECT | (d.S_arm << 2);
    } else if (kind == SWIM_MSG_DEAD) {
      if (live == SWIM_DEAD) return 0;
      ninc = rec.y > inc_s ? rec.y : inc_s;
      nst = SWIM_DEAD;
    } else {
      if (rec.y <= inc_s) return 0;
      nst = SWIM_ALIVE;
    }
  } else if (kind == SWIM_MSG_SUSPECT) {
    if (rec.y < inc_s || live != SWIM_ALIVE) {           // Core.hs:151,183
      confirm = live == SWIM_SUSPECT && rec.y >= inc_s;
      if (!(confirm && d.lg && net)) return 0;
    }
    nst = SWIM_SUSPECT | (d.S_arm << 2);               // [Q8] arm the countdown
  } else if (kind == SWIM_MSG_DEAD) {
    if (rec.y < inc_s || live == SWIM_DEAD) return 0;  // Core.hs:151,184
    nst = SWIM_DEAD;
  } else {
    if (rec.y <= inc_s) return 0;                      // [Q7] Alive(i) applies iff i > j
    nst = SWIM_ALIVE;
  }
  if (confirm) { // only the state byte changes; nothing is re-broadcast
    const uint32_t c = st_s >> 6;
    if (c < 3u && lane == hl) {
      const uint32_t t = (st_s >> 2) & 15u, dl = d.lg_delta[c + 1];
      const uint32_t nt = t > dl ? t - dl : 1u;
#pragma unroll
      for (int w = 0; w < W; ++w)
        if (w == hw) { r.st[w] = SWIM_SUSPECT | (nt << 2) | ((c + 1u) << 6); r.ticked |= 1u << w; }
    }
    return 0;
  }
  if (lane == hl) {
#pragma unroll
    for (int w = 0; w < W; ++w)
      if (w == hw) { r.st[w] = nst; r.inc[w] = ninc; r.touched |= 1u << w; } // Core.hs:171-177
  }
  rb = rec; // Core.hs:179 `return $ Just msg`: the identical message (deadFrom intact)
  return 1;
}

// ------------------------------------------------------------------ counters
// A thread's counters live in shared memory, not in registers: the round kernels keep them for the whole launch, and
// eleven registers held across every pass pushed the passes' own values out to local memory. Thread t owns words
// t * SWIM_CTR__COUNT ..; the stride is odd, so the 32 lanes of a warp hit 32 different banks.
static_assert(SWIM_CTR__COUNT % 2 == 1, "per-thread counter slots must have an odd stride");
struct Ctr {
  uint32_t *v;
  // binds this thread's slot and zeroes it; every kernel that uses Ctr runs CTAs of kThreads threads
  __device__ __forceinline__ void clear() {
    SWIM_SHARED_1D(uint32_t, s_slots, kThreads * SWIM_CTR__COUNT);
    v = s_slots + threadIdx.x * SWIM_CTR__COUNT;
#pragma unroll
    for (int i = 0; i < SWIM_CTR__COUNT; ++i) v[i] = 0;
  }
  // block-level flush: warps add into shared memory, then one global atomic per counter per CTA.
  // Every thread of the CTA must call it (it contains __syncthreads).
  __device__ __forceinline__ void flush(unsigned long long *g, int lane) {
    SWIM_SHARED_1D(uint32_t, s_ctr, SWIM_CTR__COUNT);
    if (threadIdx.x < SWIM_CTR__COUNT) s_ctr[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll
    for (int i = 0; i < SWIM_CTR__COUNT; ++i) {
      uint32_t x = __reduce_add_sync(kFull, v[i]);
      if (lane == 0 && x) atomicAdd(&s_ctr[i], x);
    }
    __syncthreads();
    // (the Ping count takes corrections of either sign — round_kernel_x — and is carried modulo 2^32 up to here: extend its sign)
    if (threadIdx.x < SWIM_CTR__COUNT && s_ctr[threadIdx.x])
      atomicAdd(&g[threadIdx.x], threadIdx.x == SWIM_CTR_PINGS ? (unsigned long long)(long long)(int32_t)s_ctr[threadIdx.x]
                                                                : (unsigned long long)s_ctr[threadIdx.x]);
  }
};

// =================================================================== K1: tick
// seeded Bernoulli loss of one probe leg: leg 0 = the direct Ping/Ack round trip (group stream),
// leg 1+j = the round trip through proxy j (per-node stream)
__device__ __forceinline__ bool leg_lost(const SimDev &d, uint32_t round, uint32_t self, uint32_t leg) {
  if (!d.loss_ppm) return false;
  uint4 y;
  uint32_t w;
  if (leg == 0) { y = philox4x32_10(make_uint4(round, self >> 2, P_LOSS0, 0), d.key0, d.key1); w = self & 3; }
  else { y = philox4x32_10(make_uint4(round, self, P_LOSS, (leg - 1) >> 2), d.key0, d.key1); w = (leg - 1) & 3; }
  return bounded(word_of(y, w), 1000000u) < d.loss_ppm;
}
// the direct leg of probe j >= 1 of a period (cfg.probes_per_round > 1): a per-node stream
__device__ __forceinline__ bool direct_leg_lost(const SimDev &d, uint32_t round, uint32_t self, uint32_t j) {
  if (j == 0) return leg_lost(d, round, self, 0);
  if (!d.loss_ppm) return false;
  const uint4 y = philox4x32_10(make_uint4(round, self, P_LOSSD, (j - 1) >> 2), d.key0, d.key1);
  return bounded(word_of(y, (j - 1) & 3), 1000000u) < d.loss_ppm;
}

constexpr int kScanGroups = 2; // Philox groups (of 4 nodes) per lane per iteration: 8 nodes, 8 loads in flight

__device__ __forceinline__ uint32_t ci(uint32_t round) { return round % 3u; } // slot of the per-round list counters
__device__ __forceinline__ uint32_t *wl_of(const SimDev &d, uint32_t round) { return d.wl + (size_t)(round & 1u) * d.n; } // that round's work list

// The two filter positions of member id x in a node's 512 W-bit membership filter (SimDev::bloom); bloom_kernel
// (swim_graph.cuh) builds the filters with the same two lines.
SWIM_HD uint32_t bloom_pos(uint32_t x, int which, uint32_t bits) {
  return SWIM_UMULHI(x * (which ? 0x85EBCA77u : 0x9E3779B1u), bits);
}

// The Philox block holding the target draws of the four nodes 4g..4g+3, and the pick itself (random: kRandomMembers
// store 1 [], Core.hs:239 over shuffle, Util.hs:36-42; round-robin: see rr_pick). `am` is consumed.
template <int W>
__device__ __forceinline__ uint4 target_block(const SimDev &d, uint32_t round, uint32_t g) {
  const bool rr = (d.flags & SWIM_F_ROUND_ROBIN) != 0; // one Philox call either way: only the counter words differ
  return philox4x32_10(make_uint4(rr ? round / (32u * W) : round, g, rr ? P_RR : P_TARGET, 0), d.key0, d.key1);
}
// K1b's draws of one node and round, computed by the warp in ONE Philox pass: lane 0 holds the group's TARGET block (or the
// round-robin block), lanes 1..7 the node's PROXY blocks 0..6 (draw j k + x <= 27), lanes 8.. its TARGETS block 0 (draws
// 0..2 of probes 1..3). tab_draw(tab, b, w) = word w of the block held by lane b (b, w warp-uniform).
template <int W>
__device__ __forceinline__ uint4 item_draws(const SimDev &d, uint32_t round, uint32_t self, int lane) {
  const bool rr = (d.flags & SWIM_F_ROUND_ROBIN) != 0;
  uint4 c;
  if (lane == 0) c = make_uint4(rr ? round / (32u * W) : round, self >> 2, rr ? P_RR : P_TARGET, 0);
  else if (lane < 8) c = make_uint4(round, self, P_PROXY, (uint32_t)lane - 1u);
  else c = make_uint4(round, self, P_TARGETS, 0);
  return philox4x32_10(c, d.key0, d.key1);
}
__device__ __forceinline__ uint32_t tab_draw(uint4 tab, uint32_t b, uint32_t w) {
  return __shfl_sync(kFull, word_of(tab, (int)w), (int)b);
}

template <int W>
__device__ __forceinline__ uint32_t pick_target(const SimDev &d, uint32_t (&am)[W], uint32_t word, uint32_t L, uint32_t round) {
  if (d.flags & SWIM_F_ROUND_ROBIN) return rr_pick<W>(am, word, round);
  return pick_remove<W>(am, bounded(word, L));
}
template <int W> // by a whole warp with warp-uniform arguments (K1b)
__device__ __forceinline__ uint32_t pick_target_warp(const SimDev &d, uint32_t (&am)[W], uint32_t word, uint32_t L, uint32_t round, int lane) {
  if (d.flags & SWIM_F_ROUND_ROBIN) return rr_pick<W>(am, word, round);
  return pick_remove_warp<W>(am, bounded(word, L), lane);
}

// The period's direct probes of one node (kRandomMembers store P [] — ONE shuffle, take P, Core.hs:239 — each target
// pinged once): true if some target's Ack will not come back (the target process is down, or the leg is lost), i.e. the
// node must go through K1b. `am` is consumed; L = popc(am) > 0.
template <int W>
__device__ __forceinline__ bool probe_fails(const SimDev &d, uint32_t (&am)[W], const uint32_t (&td)[W], uint32_t L,
                                            uint32_t tdraw, uint32_t ldraw, uint32_t round, uint32_t self) {
  const uint32_t nt = d.P < L ? d.P : L;
  bool fails = false;
  uint4 tb = make_uint4(0, 0, 0, 0);
  for (uint32_t j = 0; j < nt; ++j) {
    uint32_t draw = tdraw; // round-robin order: one walk (one word) for all probes of the period
    if (j && !(d.flags & SWIM_F_ROUND_ROBIN)) {
      if (((j - 1) & 3) == 0) tb = philox4x32_10(make_uint4(round, self, P_TARGETS, (j - 1) >> 2), d.key0, d.key1);
      draw = word_of(tb, (j - 1) & 3);
    }
    const uint32_t tslot = pick_target<W>(d, am, draw, L - j, round);
    clear_slot<W>(am, tslot);                                      // (round-robin order: the walk goes on behind it)
    bool acked = (td[tslot >> 5] >> (tslot & 31) & 1u) == 0;       // Ack iff the target process is up
    if (acked && d.loss_ppm) acked = j ? !direct_leg_lost(d, round, self, j) : !(bounded(ldraw, 1000000u) < d.loss_ppm);
    fails |= !acked;
  }
  return fails;
}
// probe_fails of a node that is not exposed (am & td == 0): every pick lands on a live target, in random and round-robin
// order alike, so the period fails iff the direct leg of one of its nt = min(P, L) probes is lost. Needs no bitmaps.
__device__ __forceinline__ bool probe_lost(const SimDev &d, uint32_t nt, uint32_t ldraw, uint32_t round, uint32_t self) {
  bool lost = bounded(ldraw, 1000000u) < d.loss_ppm;
  for (uint32_t j = 1; j < nt; ++j) lost |= direct_leg_lost(d, round, self, j);
  return lost;
}

// A node's tick decision — does it need K1b in this round? A crashed process does nothing. A buffered record to send or
// a countdown to run [Q8] means work. Otherwise only a failed probe can, and only if a crashed process sits in an Alive
// slot or messages can be lost: then the probe decides (probe_fails, on the node's draws). Without either, whichever slot
// a draw selects, the Ack comes back, so the picks and the Philox blocks behind them are not needed — the common case.
// The rule is stated from a node's summary word by the scans (scan_pass, quiet_scan: bitmaps only for exposed nodes), from
// bitmaps by node_needs_work (the receive pass, with the draws made early) and from a view row a warp has loaded by
// tick_decide and x_node. Each form is written for the register budget of the kernels it sits in: one shared row form, used by
// recv_one and x_node too, made ptxas spill more in several round-kernel instances (DESIGN.md §5).

// From the meta words; counts the node's Pings as well.
template <int W>
__device__ __forceinline__ bool node_needs_work(const SimDev &d, uint32_t flags, uint32_t (&am)[W], const uint32_t (&td)[W],
                                                uint32_t sus, uint32_t tdraw, uint32_t ldraw, uint32_t round, uint32_t &pings,
                                                uint32_t self) {
  if ((flags & 0xFFu) == 0) return false;
  bool need = (flags & 0xFF00u) != 0 || sus != 0;
  uint32_t L = 0, risk = d.loss_ppm;
#pragma unroll
  for (int w = 0; w < W; ++w) { L += __popc(am[w]); risk |= am[w] & td[w]; }
  if (L) {
    pings += d.P < L ? d.P : L;                                      // Ping (Core.hs:246), one per probe of the period
    if (risk) need |= probe_fails<W>(d, am, td, L, tdraw, ldraw, round, self);
  }
  return need;
}

// The tick decision of `tick_round` for a live local node from its freshly updated row (what K1a computes from the meta
// record): counts its Pings and, if it needs K1b, appends it to that round's work list and marks it in `listbits`.
template <int W>
__device__ __forceinline__ void tick_decide(const SimDev &d, uint32_t tick_round, uint32_t ln, const Row<W> &row, uint32_t pbcnt,
                                            const uint32_t (&td)[W], int lane, Ctr &c, uint32_t *listbits) {
  const uint32_t self = d.first + ln;
  uint32_t am[W], sus = 0, L = 0, risk = d.loss_ppm;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    am[w] = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_ALIVE);
    sus |= __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_SUSPECT);
    L += __popc(am[w]);
    risk |= am[w] & td[w];
  }
  bool need = pbcnt != 0 || sus != 0;
  if (L && risk && !need) { // only now does the decision depend on the node's draws
    const uint4 x = target_block<W>(d, tick_round, self >> 2);
    uint32_t ldraw = 0;
    if (d.loss_ppm) ldraw = word_of(philox4x32_10(make_uint4(tick_round, self >> 2, P_LOSS0, 0), d.key0, d.key1), self & 3);
    need = probe_fails<W>(d, am, td, L, word_of(x, self & 3), ldraw, tick_round, self);
  }
  if (lane == 0) {
    if (L) c.v[SWIM_CTR_PINGS] += d.P < L ? d.P : L;
    if (need) {
      wl_of(d, tick_round)[atomicAdd(&d.wl_cnt[ci(tick_round)], 1u)] = ln;
      if (listbits) atomicOr(&listbits[ln >> 5], 1u << (ln & 31));
    }
  }
}

// The summary words of the 4 U nodes a lane takes in one trip of a scan: word j of s[u] = node 4 (gb + 32 u + lane) + j
// (0 outside the shard). Returns the nodes that lie in the shard (bit 4 u + j).
__device__ __forceinline__ uint32_t load_nsum_group(const SimDev &d, uint32_t gb, int lane, uint4 (&s)[kScanGroups]) {
  constexpr int U = kScanGroups;
  uint32_t valid = 0;
  if ((d.first & 3u) == 0 && 4 * gb >= d.first && 4 * (gb + 32 * U) <= d.first + d.n) { // an interior warp: all its nodes are the shard's
    const uint4 *p = reinterpret_cast<const uint4 *>(d.nsum + 4 * (gb + lane) - d.first);
#pragma unroll
    for (int u = 0; u < U; ++u) s[u] = p[u * 32]; // U independent 16-byte loads in flight, 512 contiguous bytes per warp each
    valid = (1u << (4 * U)) - 1u;
  } else {
#pragma unroll
    for (int u = 0; u < U; ++u) {
      uint32_t w[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t node = 4 * (gb + u * 32 + lane) + j;
        const bool ok = node >= d.first && node < d.first + d.n;
        valid |= (uint32_t)ok << (u * 4 + j);
        w[j] = ok ? d.nsum[node - d.first] : 0u;
      }
      s[u] = make_uint4(w[0], w[1], w[2], w[3]);
    }
  }
  return valid;
}

// Local node l's alive and crashed-member bitmaps (an exposed node's: the scans need them for no other).
template <int W>
__device__ __forceinline__ uint32_t node_meta(const SimDev &d, uint32_t l, uint32_t (&am)[W], uint32_t (&td)[W]) {
  uint32_t L = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    const uint4 mw = d.meta[(size_t)l * W + w];
    am[w] = mw.x; td[w] = mw.z;
    L += __popc(mw.x);
  }
  return L;
}

// K1a — streaming pass over every node of the shard, EIGHT nodes per lane: a lane loads the summary words (SimDev::nsum)
// of two Philox groups of four nodes, two 16-byte loads; a warp covers 256 consecutive nodes = 1 KB contiguous. Only an
// exposed node gathers its meta bitmaps and spends a Philox block (four nodes share one) and r-th-set-bit picks (shuffle,
// Util.hs:36-42) tested against the crashed-member bitmap. Nodes that need more — a Suspect slot to count down, a failed
// probe, a non-empty piggyback buffer — are appended to the round's work list for K1b.
template <int W>
__device__ __forceinline__ void scan_pass(const SimDev &d, uint32_t round, uint32_t warp, uint32_t nwarps,
                                          int lane, uint32_t &pings, const uint32_t *skipbits = nullptr,
                                          uint4 *stage = nullptr, const uint32_t *skipbits2 = nullptr, uint32_t *listbits = nullptr) {
  // skipbits / skipbits2: bitmaps of local nodes this scan leaves alone (somebody else takes their tick decision);
  // listbits: bitmap in which every node appended to the work list is marked (round_kernel_x)
  constexpr int U = kScanGroups;
  uint32_t *wl_cnt = d.wl_cnt + ci(round);
  uint32_t *const wl = wl_of(d, round);
  const uint32_t g0 = d.first >> 2, g1 = (d.first + d.n + 3) >> 2; // Philox groups touching this shard
  for (uint32_t gb = g0 + warp * (32 * U); gb < g1; gb += nwarps * (32 * U)) {
    uint4 s[U];
    uint32_t valid = load_nsum_group(d, gb, lane, s); // bit u*4+j
    if ((skipbits || skipbits2) && valid == (1u << (4 * U)) - 1u && (d.first & 3u) == 0) {
      // (the lane's four nodes of a group are consecutive and 4-aligned in the shard: one bitmap word holds their bits)
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const uint32_t l0 = 4 * (gb + u * 32 + lane) - d.first;
        uint32_t sk = 0;
        if (skipbits) sk = skipbits[l0 >> 5];
        if (skipbits2) sk |= skipbits2[l0 >> 5];
        valid &= ~((sk >> (l0 & 31) & 0xFu) << (u * 4));
      }
    } else if (skipbits || skipbits2) { // nodes with mail from last round belong to the warps that apply it (recv_one takes their tick decision)
#pragma unroll
      for (int u = 0; u < U; ++u)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (valid >> (u * 4 + j) & 1u) {
            const uint32_t l = 4 * (gb + u * 32 + lane) + j - d.first;
            uint32_t sk = 0;
            if (skipbits) sk = skipbits[l >> 5];
            if (skipbits2) sk |= skipbits2[l >> 5];
            if (sk >> (l & 31) & 1u) valid &= ~(1u << (u * 4 + j));
          }
    }
    uint32_t work = 0; // bit u*4+j: that node needs K1b
    unsigned fb = 0;     // lanes whose STAGED node (see below) needs K1b ...
    uint32_t fself = 0;  // ... and that node's id
    // Pass 1, every node: what the summary word alone decides (buffer to send, countdown to run, the Ping count). Only an
    // exposed node (or any node, under message loss) depends on its draws — and only if the word has not already sent it
    // to K1b. Those nodes are COMPACTED over the warp through `stage` (the ids of up to 32, in the warp's shared memory):
    // the staged pass then spends one meta gather, one Philox block and one set of picks per lane on up to 32 of them at
    // once, whichever lanes they came from (a burst round of C3 has ~8 per warp: one trip instead of the two or three a
    // per-lane loop needs). Without a stage buffer, under message loss (every node is risky) and for the overflow, the
    // per-lane loop below does the same work.
    uint32_t risky = 0, nstaged = 0;
    const bool can_stage = stage != nullptr && d.loss_ppm == 0;
    uint32_t *const sid = reinterpret_cast<uint32_t *>(stage);
#pragma unroll
    for (int u = 0; u < U; ++u)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int q = u * 4 + j;
        const uint32_t sw = word_of(s[u], j);
        bool rq = false;
        if ((valid >> q & 1u) && ns_up(sw)) { // in range, not left to the receive pass, process up
          const uint32_t L = ns_alive(sw);
          const bool wk = (sw & kNsBusy) != 0;
          if (wk) work |= 1u << q;
          if (L) {
            pings += d.P < L ? d.P : L;
            rq = !wk && ((sw & kNsExposed) || d.loss_ppm);
          }
        }
        if (can_stage) {
          const unsigned rb = __ballot_sync(kFull, rq);
          if (rb) {
            const uint32_t pos = nstaged + __popc(rb & ((1u << lane) - 1u));
            if (rq) {
              if (pos < 32u) sid[pos] = 4 * (gb + u * 32 + lane) + j;
              else risky |= 1u << q; // (more than 32 in one warp's 256 nodes: the per-lane loop takes the rest)
            }
            nstaged += __popc(rb);
          }
        } else if (rq) {
          risky |= 1u << q;
        }
      }
    // The nodes that were not staged, one per lane and trip: a lane pays for its own risky nodes only, not — by
    // divergence — for every risky node of the warp. An exposed node gathers its bitmaps and runs the picks; any other
    // only asks whether a direct leg is lost (probe_lost).
    while (risky) {
      const int q = __ffs(risky) - 1;
      risky &= risky - 1;
      uint32_t sw = 0;
#pragma unroll
      for (int qq = 0; qq < 4 * U; ++qq)
        if (q == qq) sw = word_of(s[qq >> 2], qq & 3);
      const uint32_t g = gb + (q >> 2) * 32 + lane, self = 4 * g + (q & 3);
      uint32_t ldraw = 0;
      if (d.loss_ppm) ldraw = word_of(philox4x32_10(make_uint4(round, g, P_LOSS0, 0), d.key0, d.key1), q & 3);
      bool fails;
      if (sw & kNsExposed) {
        uint32_t am[W], td[W];
        const uint32_t L = node_meta<W>(d, self - d.first, am, td);
        const uint4 x = target_block<W>(d, round, g);
        fails = probe_fails<W>(d, am, td, L, word_of(x, q & 3), ldraw, round, self);
      } else {
        const uint32_t L = ns_alive(sw);
        fails = probe_lost(d, d.P < L ? d.P : L, ldraw, round, self);
      }
      if (fails) work |= 1u << q;
    }
    // ... and the staged nodes (all exposed: staging is off under message loss), up to 32 at once
    if (nstaged) {
      __syncwarp();
      bool fails = false;
      if ((uint32_t)lane < (nstaged < 32u ? nstaged : 32u)) {
        const uint32_t self = sid[lane];
        uint32_t am[W], td[W];
        const uint32_t L = node_meta<W>(d, self - d.first, am, td); // (in flight while the Philox block is computed)
        const uint4 x = target_block<W>(d, round, self >> 2);
        fails = probe_fails<W>(d, am, td, L, word_of(x, self & 3), 0u, round, self);
        fself = self;
      }
      fb = __ballot_sync(kFull, fails);
      __syncwarp(); // the buffer is free again (next trip of this loop, or the passes that follow the scan)
    }
    // warp-aggregated append of up to 4*U x 32 nodes
    if (__any_sync(kFull, work != 0) || fb) {
      unsigned b[4 * U];
      uint32_t total = __popc(fb);
#pragma unroll
      for (int q = 0; q < 4 * U; ++q) { b[q] = __ballot_sync(kFull, work >> q & 1u); total += __popc(b[q]); }
      uint32_t pos = 0;
      if (lane == 0) pos = atomicAdd(wl_cnt, total);
      pos = __shfl_sync(kFull, pos, 0);
#pragma unroll
      for (int q = 0; q < 4 * U; ++q) {
        if (work >> q & 1u) {
          const uint32_t l = 4 * (gb + (q >> 2) * 32 + lane) + (q & 3) - d.first;
          wl[pos + __popc(b[q] & ((1u << lane) - 1))] = l;
          if (listbits) atomicOr(&listbits[l >> 5], 1u << (l & 31));
        }
        pos += __popc(b[q]);
      }
      if (fb >> lane & 1u) { // the staged nodes whose probe fails
        const uint32_t l = fself - d.first;
        wl[pos + __popc(fb & ((1u << lane) - 1))] = l;
        if (listbits) atomicOr(&listbits[l >> 5], 1u << (l & 31));
      }
    }
  }
}

template <int W>
__global__ void __launch_bounds__(kThreads, kMinBlocks) tick_scan_kernel(SimDev d) {
  SWIM_SHARED_2D(uint4, s_stage, kWarpsPerBlock, 32);
  pdl_launch();
  pdl_wait();
  const uint32_t round = d.round;
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t pings = 0;
  scan_pass<W>(d, round, warp, nwarps, lane, pings, nullptr, s_stage[threadIdx.x >> 5]);
  pings = __reduce_add_sync(kFull, pings);
  if (lane == 0 && pings) atomicAdd(&d.ctr[SWIM_CTR_PINGS], (unsigned long long)pings);
}

// K1a over Q consecutive rounds at once, for stretches in which nothing happens. A round whose scan lists no work
// writes nothing, so the scan of the round after it reads the same summary words: one pass loads them once and decides
// rounds round .. round+Q-1 together. Only the probe outcome depends on the round (through the target draw), and only
// for exposed nodes (a crashed process in an Alive slot) — rare once a cluster has converged; everything else a node
// can need (a buffered record, a countdown) holds for every round of the batch. Nothing is listed: the result is the
// lane's mask of rounds that are NOT quiet (bit q: round + q), the caller commits the rounds before the first such bit
// and runs the ordinary scan from there. `pings` is the Ping count of ONE round (the same for each of them).
// Requires loss_ppm == 0 (with loss every probe depends on a draw and there are no quiet stretches to speak of).
template <int W>
__device__ __forceinline__ uint32_t quiet_scan(const SimDev &d, uint32_t round, uint32_t Q, uint32_t warp, uint32_t nwarps,
                                               int lane, uint32_t &pings) {
  constexpr int U = kScanGroups;
  const uint32_t allq = (1u << Q) - 1u;
  uint32_t busy = 0;
  const uint32_t g0 = d.first >> 2, g1 = (d.first + d.n + 3) >> 2;
  for (uint32_t gb = g0 + warp * (32 * U); gb < g1; gb += nwarps * (32 * U)) {
    uint4 s[U];
    const uint32_t valid = load_nsum_group(d, gb, lane, s);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const uint32_t g = gb + u * 32 + lane;
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const uint32_t sw = word_of(s[u], j), L = ns_alive(sw);
        if (!(valid >> (u * 4 + j) & 1u) || !ns_up(sw)) continue;
        if (sw & kNsBusy) busy = allq;
        if (!L) continue;
        pings += d.P < L ? d.P : L;
        if ((sw & kNsBusy) || !(sw & kNsExposed)) continue; // the draw is never looked at: one decision for the batch
        uint32_t am[W], td[W];
        const uint32_t Lt = node_meta<W>(d, 4 * g + j - d.first, am, td);
        for (uint32_t q = 0; q < Q; ++q) {
          uint32_t amq[W];
#pragma unroll
          for (int w = 0; w < W; ++w) amq[w] = am[w];
          const uint4 x = target_block<W>(d, round + q, g);
          if (probe_fails<W>(d, amq, td, Lt, word_of(x, j), 0, round + q, 4 * g + j)) busy |= 1u << q;
        }
      }
    }
  }
  return busy;
}

// This warp's first list entry, to be fetched together with the list count (one memory round trip instead of two); the
// entry is only looked at when warp < n_work. Volatile: the load stays where it is written, ahead of the branch on the count.
__device__ __forceinline__ uint32_t first_work_entry(const SimDev &d, uint32_t round, uint32_t warp) {
  return warp < d.n ? *(volatile const uint32_t *)(wl_of(d, round) + warp) : 0u;
}

// K1b, one node — countdown and expiry -> Dead, probe escalation (k proxies), local suspicion, piggyback send — on a row
// and a piggyback buffer that are already loaded (registers / the warp's shared-memory stage): work_pass walks the work
// list with it; round_kernel_x also runs it right behind a node's mail. Lane s owns view slot s. Everything K1a derived is
// recomputed from the row with warp ballots. Stores the row and the buffer; idx = the node's position on the round's work
// list (its recipient slots, for the datagram export). kSharded = false: a single-shard launch (d.world == 1), in which
// every recipient is local and the peer-memory and exchange-bucket stores do not exist.
template <int W, bool kSharded = true>
__device__ __forceinline__ void work_body(const SimDev &d, uint32_t round, uint32_t ln, uint32_t idx, Row<W> &row, const uint32_t (&rix)[W],
                                          const uint32_t (&td)[W], PbStage &pbs, Ctr &c, int lane, bool &did_remote,
                                          uint32_t next_ln, bool have_next) {
  constexpr bool kCarry = W <= 2;
  const uint32_t self = d.first + ln;
  const uint32_t par = round & 1;
  uint2 *rl_out = d.rl + (size_t)par * d.n * d.fanout;
  uint32_t am[W], L = 0;
#pragma unroll
  for (int w = 0; w < W; ++w) {
    am[w] = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_ALIVE);
    L += __popc(am[w]);
  }
  // T1 [Q8]: countdown on every Suspect slot; expired -> Dead, broadcast Dead(inc, member,
  // from = self) in slot order
#pragma unroll
  for (int w = 0; w < W; ++w) {
    if ((row.st[w] & 3u) == SWIM_SUSPECT) { row.st[w] -= 4u; row.ticked |= 1u << w; } // timer >= 1 while Suspect
    unsigned em = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_SUSPECT && ((row.st[w] >> 2) & d.tmask) == 0);
    if (em >> lane & 1u) { row.st[w] = SWIM_DEAD; row.touched |= 1u << w; }
    while (em) {
      const int s = __ffs(em) - 1;
      em &= em - 1;
      const uint32_t m = __shfl_sync(kFull, row.nb[w], s), i = __shfl_sync(kFull, row.inc[w], s);
      pb_enqueue(pbs, d, make_rec(m, i, self, SWIM_MSG_DEAD), lane, c.v[SWIM_CTR_PB_DROPPED]);
      if (lane == 0) ++c.v[SWIM_CTR_DEAD_TIMEOUT];
    }
  }
  // T2: the period's probe targets — kRandomMembers store P [] (Core.hs:239): ONE shuffle of the alive list, take P
  // (P = cfg.probes_per_round; 1 = SWIM's single probe [Q11]); draw 0 is the node's TARGET word of the group block,
  // draws 1.. come from a per-node stream. Probe 0's proxies — kRandomMembers store k [] (Core.hs:249), a fresh shuffle
  // over the same alive list, neither self nor the target excluded — double as piggyback recipients (T4), so they are
  // drawn whether or not the probe escalates.
  uint32_t tslots[SWIM_MAX_PROBES], nt = 0, np = 0;
  uint32_t prox_l = 0; // lane x < np: proxy x of probe 0 (a view slot)
#pragma unroll
  for (uint32_t j = 0; j < SWIM_MAX_PROBES; ++j) tslots[j] = 0;
  if (L) {
    nt = d.P < L ? d.P : L;
    // Every Philox block this item can ask for, in ONE pass of the warp: lane 0 computes the group's TARGET (or
    // round-robin) block, lanes 1..7 the node's PROXY blocks 0..6 (draws j k + x <= 27), lane 8 its TARGETS block — a
    // draw is then a shuffle from the lane that holds its block, instead of one warp-wide Philox call per block.
    const uint4 tab = item_draws<W>(d, round, self, lane);
    uint32_t tmp[W];
#pragma unroll
    for (int w = 0; w < W; ++w) tmp[w] = am[w];
    uint32_t draw = tab_draw(tab, 0, self & 3);
#pragma unroll
    for (uint32_t j = 0; j < SWIM_MAX_PROBES; ++j) {
      if (j >= nt) break;
      if (j && !(d.flags & SWIM_F_ROUND_ROBIN)) // (round-robin order: one walk, one word, for all probes of the period)
        draw = tab_draw(tab, 8, j - 1);          // TARGETS draw j - 1 (j - 1 <= 2: block 0)
      tslots[j] = pick_target_warp<W>(d, tmp, draw, L - j, round, lane);
      clear_slot<W>(tmp, tslots[j]);
    }
#pragma unroll
    for (int w = 0; w < W; ++w) tmp[w] = am[w];
    np = d.k < L ? d.k : L;
    for (uint32_t j = 0; j < np; ++j) {
      const uint32_t pick = pick_remove_warp<W>(tmp, bounded(tab_draw(tab, 1 + (j >> 2), j & 3), L - j), lane);
      if ((uint32_t)lane == j) prox_l = pick;
    }
    // T3: the probes one after the other (mapM_ probeNode', Core.hs:240) — Ping (Core.hs:246); unlessAck ->
    // IndirectPings (247-250); unlessAck -> suspectNode (251-254). The incarnations are those of the moment the targets
    // were chosen; a later probe's proxies are drawn from the store as the earlier probes left it.
    uint32_t tincs = 0, tnodes = 0; // lane j: incarnation / id of target j as loaded (captured before any suspicion)
#pragma unroll
    for (uint32_t j = 0; j < SWIM_MAX_PROBES; ++j) {
      if (j >= nt) break;
      uint32_t a = 0, b = 0;
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const uint32_t x = __shfl_sync(kFull, row.inc[w], tslots[j] & 31), y = __shfl_sync(kFull, row.nb[w], tslots[j] & 31);
        if ((uint32_t)w == (tslots[j] >> 5)) { a = x; b = y; }
      }
      if ((uint32_t)lane == j) { tincs = a; tnodes = b; }
    }
    uint32_t cur[W], Lc = L; // the alive list as the probes so far left it
#pragma unroll
    for (int w = 0; w < W; ++w) cur[w] = am[w];
#pragma unroll
    for (uint32_t j = 0; j < SWIM_MAX_PROBES; ++j) {
      if (j >= nt) break;
      const uint32_t tslot = tslots[j];
      const bool t_up = (td[tslot >> 5] >> (tslot & 31) & 1u) == 0;
      const bool acked = t_up && !direct_leg_lost(d, round, self, j);
      if (acked) continue;
      uint32_t npj = np;
      uint32_t ps = (uint32_t)lane < np ? prox_l : 0u; // lane x: proxy x of this probe
      if (j) { // kRandomMembers store k [] on the store as it is now: draws j k .. j k + k - 1 of the PROXY stream
        uint32_t t2[W];
#pragma unroll
        for (int w = 0; w < W; ++w) t2[w] = cur[w];
        npj = d.k < Lc ? d.k : Lc;
        ps = 0;
        for (uint32_t x = 0; x < npj; ++x) {
          const uint32_t q = j * d.k + x;
          const uint32_t pick = pick_remove_warp<W>(t2, bounded(tab_draw(tab, 1 + (q >> 2), q & 3), Lc - x), lane);
          if ((uint32_t)lane == x) ps = pick;
        }
      }
      if (lane == 0) { ++c.v[SWIM_CTR_DIRECT_FAIL]; c.v[SWIM_CTR_INDIRECT_PINGS] += npj; }
      bool ok = false;
      if ((uint32_t)lane < npj && t_up)
        ok = (td[ps >> 5] >> (ps & 31) & 1u) == 0 && !leg_lost(d, round, self, 1 + j * d.k + lane);
      if (!__any_sync(kFull, ok)) {
        // Suspect (memberIncarnation m) (memberName m) with m captured at probe start
        const uint32_t tinc = __shfl_sync(kFull, tincs, j), tnode = __shfl_sync(kFull, tnodes, j);
        uint4 rb;
        uint32_t no_self_inc = 0xFFFFFFFFu; // a probe never targets self
        if (row_apply<W>(row, d, self, no_self_inc, make_rec(tnode, tinc, 0, SWIM_MSG_SUSPECT), rb, lane,
                         c.v[SWIM_CTR_REFUTES], false) == 1) {
          pb_enqueue(pbs, d, rb, lane, c.v[SWIM_CTR_PB_DROPPED]); // yield . Broadcast (Core.hs:254)
          if (lane == 0) ++c.v[SWIM_CTR_SUSPECT_LOCAL];
          clear_slot<W>(cur, tslot);
          --Lc;
        }
      }
    }
  }
  row_store<W>(row, d, ln, lane, round, td);
#ifndef SWIM_EMU
  if (have_next && lane < 5) { // next item's rows -> L2 (one 128-byte line each at cap 32)
    const size_t nb = (size_t)next_ln * d.cap;
    const void *pf = lane == 0 ? (const void *)(d.nbr + nb) : lane == 1 ? (const void *)(d.vinc + nb) : lane == 2 ? (const void *)(d.vst + nb)
                   : lane == 3 ? (const void *)(d.pb + (size_t)next_ln * d.B) : (const void *)(d.ridx + nb);
    asm volatile("prefetch.global.L2 [%0];" ::"l"(pf));
  }
#endif
  // T4 [Q5]: the buffer rides on the messages to the target and the first proxies
  uint2 cand = make_uint2(0xFFFFFFFFu, ln); // lane f < fanout: recipient slot f
  if (L && pbs.cnt) {
    // recipients: the probe targets in order, then probe 0's proxies that are no targets, the first `fanout` of them;
    // lane f carries recipient f
    uint32_t nr = nt < d.fanout ? nt : d.fanout, rslot = 0;
#pragma unroll
    for (uint32_t j = 0; j < SWIM_MAX_PROBES; ++j)
      if ((uint32_t)lane == j && j < nr) rslot = tslots[j];
    bool is_target = false; // lane x: proxy x is one of the targets
#pragma unroll
    for (uint32_t t = 0; t < SWIM_MAX_PROBES; ++t) is_target |= t < nt && prox_l == tslots[t];
    unsigned pm = __ballot_sync(kFull, (uint32_t)lane < np && !is_target);
    while (pm && nr < d.fanout) { // the remaining proxies in draw order
      const int x = __ffs(pm) - 1;
      pm &= pm - 1;
      const uint32_t p = __shfl_sync(kFull, prox_l, x);
      if ((uint32_t)lane == nr) rslot = p;
      ++nr;
    }
    uint32_t xs = 0xFFFFFFFFu; // exchange-bucket slot when lane f's recipient lives on another shard
    uint32_t dst_c = 0, ridx_c = 0; // recipient id and in-edge index of lane f's slot, from the lanes that hold them
    if (kCarry)
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const uint32_t a = __shfl_sync(kFull, row.nb[w], rslot & 31), b = __shfl_sync(kFull, rix[w], rslot & 31);
        if ((uint32_t)w == (rslot >> 5)) { dst_c = a; ridx_c = b; }
      }
    uint32_t n_up = 0;
    if ((uint32_t)lane < nr) {
      const size_t e = (size_t)ln * d.cap + rslot;
      const uint32_t dst = kCarry ? dst_c : d.nbr[e], ridx = kCarry ? ridx_c : d.ridx[e];
      // A datagram to a crashed process is lost (the crashed-member bitmap says so without touching alive[]); one to a
      // live process is received (counted here), but it is only DELIVERED — flagged and listed for K2 — if one of its
      // records is about the recipient itself or passes the recipient's membership filter: anything else would run
      // into `we don't know this node. ignore` (Core.hs:147-148) record by record and change nothing.
      const bool r_up = (td[rslot >> 5] >> (rslot & 31) & 1u) == 0;
      n_up = r_up ? 1u : 0u;
      bool deliver = false;
      if (r_up) {
        constexpr uint32_t kBits = 512u * W;
        const uint32_t *bf = d.bloom + (size_t)dst * (kBits / 32);
        // two records per trip: their four filter words are in flight together (most envelopes carry one record)
        for (uint32_t q0 = 0; q0 < pbs.cnt && !deliver; q0 += 2) {
          const uint32_t xa = pbs.s[q0].x, xb = q0 + 1 < pbs.cnt ? pbs.s[q0 + 1].x : xa;
          const uint32_t pa0 = bloom_pos(xa, 0, kBits), pa1 = bloom_pos(xa, 1, kBits);
          const uint32_t pb0 = bloom_pos(xb, 0, kBits), pb1 = bloom_pos(xb, 1, kBits);
          const uint32_t wa0 = bf[pa0 >> 5], wa1 = bf[pa1 >> 5], wb0 = bf[pb0 >> 5], wb1 = bf[pb1 >> 5];
          deliver = xa == dst || xb == dst || ((wa0 >> (pa0 & 31) & 1u) && (wa1 >> (pa1 & 31) & 1u)) ||
                    ((wb0 >> (pb0 & 31) & 1u) && (wb1 >> (pb1 & 31) & 1u));
        }
      }
      const uint32_t owner = (!kSharded || d.world == 1) ? 0u : dst / d.per;
      const uint32_t dl = dst - owner * d.per;
      const bool local = !kSharded || owner == d.rank;
      if (local) cand.x = dl | (deliver ? 0u : 0x80000000u); // bit 31: sent, nothing for K2 to do
      if (!deliver) {
        // dropped at the sender
      } else if (local) {
        d.eflag[(size_t)par * d.estride + ridx] = 1; // raise the in-edge flag (i -> dst)
        if (d.fused) atomicOr(&d.mailbits[(size_t)(round % 3u) * d.mbw + (dl >> 5)], 1u << (dl & 31));
      } else if (d.p2p) {
        // fused exchange: flag and receiver-list entry go straight into the owner GPU's memory over NVLink (plain
        // stores, nothing comes back); the receiver pulls our snapshot
        d.eflag_p[owner][(size_t)par * d.estride_p[owner] + ridx] = 1;
        const uint32_t k = atomicAdd(&d.xcnt[owner], 1u);
        d.rlr_p[owner][((size_t)par * d.world + d.rank) * d.rcap + k] = dl;
        if (d.fused) atomicOr(&d.mailbits_p[owner][(size_t)(round % 3u) * d.mbw + (dl >> 5)], 1u << (dl & 31));
        did_remote = true;
      } else {
        const uint32_t k = atomicAdd(&d.xsend_cnt[owner], 1u);
        if (k < d.xcap) {
          xs = owner * d.xcap + k;
          d.xsend[(size_t)xs * (1 + d.B)] = make_uint4(ridx, pbs.cnt, self, dl);
        } else {
          d.xsend_cnt[d.world] = 1; // overflow: reported by the host as SWIM_ECAP, never silent
        }
      }
    }
    n_up = __reduce_add_sync(kFull, n_up);
    const unsigned dm = __ballot_sync(kFull, cand.x < 0x80000000u); // delivered to a local receiver
    if (dm) { // compact list for K2: one counter bump per sender that delivered anything (few do)
      uint32_t pos = 0;
      if (lane == 0) pos = atomicAdd(&d.ncand[ci(round)], (uint32_t)__popc(dm));
      pos = __shfl_sync(kFull, pos, 0);
      if (dm >> lane & 1u) d.cl[(size_t)par * d.n * d.fanout + pos + __popc(dm & ((1u << lane) - 1))] = cand;
    }
    if (lane == 0) {
      d.out_cnt[(size_t)par * d.per + ln] = (uint8_t)pbs.cnt;
      c.v[SWIM_CTR_MSGS] += nr;
      c.v[SWIM_CTR_RECS_SENT] += nr * pbs.cnt;
      c.v[SWIM_CTR_MSGS_RECV] += n_up; // envelopes that reach a live process
    }
    // snapshot, then one transmission is spent on every record
    uint4 mine = make_uint4(0, 0, 0, 0);
    const bool have = (uint32_t)lane < pbs.cnt;
    if (have) { mine = pbs.s[lane]; d.out[((size_t)par * d.per + ln) * d.B + lane] = mine; }
    if (kSharded) {
      unsigned xm = __ballot_sync(kFull, xs != 0xFFFFFFFFu);
      while (xm) { // cross-shard envelopes carry the records themselves (staged NCCL path)
        const int f = __ffs(xm) - 1;
        xm &= xm - 1;
        const uint32_t xslot = __shfl_sync(kFull, xs, f);
        if (have) d.xsend[(size_t)xslot * (1 + d.B) + 1 + lane] = mine;
      }
    }
    const bool keep = have && rec_ttl(mine) > 1;
    const unsigned km = __ballot_sync(kFull, keep);
    __syncwarp();
    if (keep) {
      mine.w -= 1u << 8;
      pbs.s[__popc(km & ((1u << lane) - 1))] = mine;
    }
    pbs.cnt = __popc(km);
    pbs.dirty = true;
    __syncwarp();
  }
  pb_store(pbs, d, ln, lane);
  if ((uint32_t)lane < d.fanout) rl_out[(size_t)idx * d.fanout + lane] = cand; // no atomics, no shared counter
}

// K1b — warp-per-node over the work list.
template <int W, bool kSharded = true>
__device__ __forceinline__ bool work_pass(const SimDev &d, uint32_t round, uint32_t warp, uint32_t nwarps, int lane,
                                          PbStage &pbs, Ctr &c, uint32_t first_ln, bool fence_remote = true) {
  const uint32_t n_work = d.wl_cnt[ci(round)];
  bool did_remote = false; // this lane stored into a peer GPU's memory
  uint32_t next_ln = first_ln;
  for (uint32_t idx = warp; idx < n_work; idx += nwarps) {
    const uint32_t ln = next_ln;
    Row<W> row;
    row_load<W>(row, d, ln, lane);
    pb_load(pbs, d, ln, lane);
    // the next item's list entry is fetched now, and — once it is known, further down — its rows are pulled towards L2:
    // a warp walks its items one after the other, so each dependent round trip it can start early is one it does not wait for
    const bool have_next = idx + nwarps < n_work;
    if (have_next) next_ln = *(volatile const uint32_t *)(wl_of(d, round) + idx + nwarps);
    // the row's edge indices travel with the row (narrow rows): the send step needs the recipients' in-edge
    // indices, and loading them there would be one more dependent memory round trip per item
    uint32_t rix[W], td[W];
#pragma unroll
    for (int w = 0; w < W; ++w) {
      rix[w] = W <= 2 ? d.ridx[(size_t)ln * d.cap + w * 32 + lane] : 0u;
      td[w] = d.meta[(size_t)ln * W + w].z;
    }
    work_body<W, kSharded>(d, round, ln, idx, row, rix, td, pbs, c, lane, did_remote, next_ln, have_next);
  }
  if (did_remote && fence_remote) __threadfence_system(); // peer-memory stores are performed before the grid reports completion
  return did_remote;
}

template <int W>
__global__ void __launch_bounds__(kThreads, kMinBlocks) tick_work_kernel(SimDev d) {
  SWIM_SHARED_2D(uint4, s_pb, kWarpsPerBlock, 32);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarpsPerBlock + wib, nwarps = gridDim.x * kWarpsPerBlock;
  pdl_launch();
  pdl_wait();
  const uint32_t round = d.round;
  if (warp == 0 && lane == 0) { d.wl_cnt[ci(round + 1)] = 0; d.ncand[ci(round + 1)] = 0; }
  Ctr c; c.clear();
  PbStage pbs; pbs.s = s_pb[wib];
  work_pass<W>(d, round, warp, nwarps, lane, pbs, c, first_work_entry(d, round, warp));
  c.flush(d.ctr, lane);
}

// =================================================================== cross-GPU synchronisation
// Fused exchange: before a rank applies round `mail_round`'s mail it must know that every peer has finished K1b of that
// round (all flags / list entries have landed in its memory) and how many receivers each peer listed there.
// peer_handshake_cta is run by ALL threads of one CTA, once every CTA of this rank has finished its K1b of the round and
// those that stored into peer memory have fenced at system scope: the last CTA to arrive at a grid barrier of the round
// kernels, or peer_barrier_kernel. Thread q publishes to peer q the number of receivers this rank listed there and then,
// with release semantics, this rank's round word; it then waits (acquire) for peer q's word. One thread per peer, all
// peers in parallel; the wait is bounded (a missing peer sets *bar_err instead of hanging the GPU).
__device__ __forceinline__ void peer_handshake_cta(const SimDev &d, uint32_t mail_round) {
  const uint32_t q = threadIdx.x;
  if (q < d.world && q != d.rank) {
    d.rcnt_p[q][(mail_round & 1) * d.world + d.rank] = atomicExch(&d.xcnt[q], 0u);
    st_release_sys(d.bar_p[q] + d.rank, mail_round);
    const uint32_t *mine = d.bar_p[d.rank] + q;
    const long long t0 = clock64();
    uint32_t polls = 0;
    while ((int32_t)(ld_acquire_sys(mine) - mail_round) < 0)
      if (wait_expired(d, t0, kPeerWaitCycles, polls, 1)) break; // a peer stopped stepping
  }
}

// stand-alone form of the same synchronisation (split launch sequence): one CTA, launched between K1b and K2
static __global__ void peer_barrier_kernel(SimDev d) {
  pdl_launch();
  pdl_wait(); // K1b of this rank is complete and flushed
  peer_handshake_cta(d, d.round);
}

// =================================================================== K2: receive
// The mail of `round` for local node ln, applied to a row and a piggyback buffer that are already loaded: in-edge flags
// [e0, e1) in ascending sender order -> the senders' snapshots (the one fetched early, local HBM, or a peer GPU's memory)
// -> row_apply per record, re-broadcast enqueue.
template <int W>
__device__ __forceinline__ void apply_mail(const SimDev &d, uint32_t round, uint32_t ln, uint32_t e0, uint32_t e1, bool early,
                                           uint32_t snd, uint4 early_rec, uint32_t early_cnt, Row<W> &row, PbStage &pbs,
                                           uint32_t &self_inc, int lane, Ctr &c) {
  const uint32_t par = round & 1;
  const size_t ebase = (size_t)par * d.estride;
  const uint32_t self = d.first + ln;
  for (uint32_t eb = e0; eb < e1; eb += 32) {
    const uint32_t e = eb + lane;
    uint32_t f = 0, src = 0;
    if (e < e1) { f = d.eflag[ebase + e]; src = d.in_src[e]; }
    if (f) d.eflag[ebase + e] = 0;
    unsigned fm = __ballot_sync(kFull, f != 0);
    while (fm) { // ascending sender id: the in-list is sorted
      const int q = __ffs(fm) - 1;
      fm &= fm - 1;
      const uint32_t s_id = __shfl_sync(kFull, src, q), s_kind = __shfl_sync(kFull, f, q);
      uint32_t cnt;
      uint4 mine = make_uint4(0, 0, 0, 0);
      if (s_kind == 1 && early && s_id == d.first + snd) { // the sender this slot came from: already here
        mine = early_rec;
        cnt = early_cnt;
      } else if (s_kind == 1) { // pull the sender's snapshot (from a peer GPU's memory if it lives there)
        const uint32_t s_rank = d.world == 1 ? 0u : s_id / d.per, sl = s_id - s_rank * d.per;
        if (s_rank == d.rank) {
          if ((uint32_t)lane < d.B) mine = d.out[((size_t)par * d.per + sl) * d.B + lane];
          cnt = d.out_cnt[(size_t)par * d.per + sl];
        } else {
          if ((uint32_t)lane < d.B) mine = ld_sys_u4(d.out_p[s_rank] + ((size_t)par * d.per + sl) * d.B + lane);
          cnt = ld_sys_u8(d.out_cnt_p[s_rank] + (size_t)par * d.per + sl);
        }
      } else {           // staged NCCL path: the envelope arrived in the exchange buffer
        const uint32_t xslot = d.eslot[eb + q];
        const uint4 *env = d.xrecv + (size_t)xslot * (1 + d.B);
        if ((uint32_t)lane < d.B) mine = env[1 + lane];
        cnt = env[0].y;
      }
      for (uint32_t r = 0; r < cnt; ++r) { // records in buffer order (newest first)
        uint4 rec;
        rec.x = __shfl_sync(kFull, mine.x, r); rec.y = __shfl_sync(kFull, mine.y, r);
        rec.z = __shfl_sync(kFull, mine.z, r); rec.w = __shfl_sync(kFull, mine.w, r);
        uint4 rb;
        if (row_apply<W>(row, d, self, self_inc, rec, rb, lane, c.v[SWIM_CTR_REFUTES]) == 1) {
          pb_enqueue(pbs, d, rb, lane, c.v[SWIM_CTR_PB_DROPPED]); // maybeBroadcast (Core.hs:119-121)
          if (lane == 0) ++c.v[SWIM_CTR_RECS_APPLIED];
        }
      }
    }
  }
}


// One receiver of `round`: claim, in-edge flags -> sender snapshots (local or peer-GPU memory) -> row_apply per record,
// re-broadcast enqueue. Loads that do not depend on each other are issued together: (claim, row, buffer, in-list bounds,
// the snapshot of the sender the slot names) -> (edge flags, sender ids) -> (other senders' snapshots).
// tick_round != 0 (fused kernel: the mail of `round` is applied during the scan phase of tick_round = round + 1, and the
// scan leaves the node alone): after the mail, the node's tick decision of tick_round — what K1a would have computed —
// is taken here from the fresh row, and the node is appended to that round's work list if it needs K1b.
template <int W>
__device__ __forceinline__ void recv_one(const SimDev &d, uint32_t round, uint32_t ln, bool early, uint32_t snd, int lane,
                                         PbStage &pbs, Ctr &c, uint32_t tick_round = 0) {
  const uint32_t par = round & 1;
  const size_t ebase = (size_t)par * d.estride;
  // the claim and every load that depends only on `ln` are issued together (one memory round trip)
  uint32_t old = 0;
  if (lane == 0) old = atomicExch(&d.claim[ln], round);
  const uint32_t self = d.first + ln;
  const uint32_t e0 = d.in_off[ln], e1 = d.in_off[ln + 1];
  Row<W> row;
  row_load<W>(row, d, ln, lane);
  pb_load(pbs, d, ln, lane);
  uint32_t self_inc = d.self_inc[ln];
  const uint32_t self_inc0 = self_inc;
  uint32_t td[W]; // crashed-member bits (events only, not touched by mail): needed by the tick decision at the very end —
#pragma unroll    // fetched now, with everything else, so that it is no dependent round trip there
  for (int w = 0; w < W; ++w) td[w] = tick_round ? d.meta[(size_t)ln * W + w].z : 0u;
  // A recipient slot names one sender of its receiver; that sender's snapshot is fetched together with the receiver's
  // row, ahead of the in-edge flags that will ask for it — for the usual envelope (one sender per receiver per round) the
  // pass is one dependent round trip shorter. The flags still decide what is applied and in which order.
  uint4 early_rec = make_uint4(0, 0, 0, 0);
  uint32_t early_cnt = 0;
  if (early) {
    if ((uint32_t)lane < d.B) early_rec = d.out[((size_t)par * d.per + snd) * d.B + lane];
    early_cnt = d.out_cnt[(size_t)par * d.per + snd];
  }
  if (__shfl_sync(kFull, old, 0) == round) return; // another warp has this receiver
  // (a listed receiver is a live process: senders deliver only to members whose crashed-member bit is clear)
  apply_mail<W>(d, round, ln, e0, e1, early, snd, early_rec, early_cnt, row, pbs, self_inc, lane, c);
  if (!tick_round) // row_store needs them too (loaded only now: not held across the mail without a tick decision)
#pragma unroll
    for (int w = 0; w < W; ++w) td[w] = d.meta[(size_t)ln * W + w].z;
  row_store<W>(row, d, ln, lane, round, td);
  pb_store(pbs, d, ln, lane);
  if (lane == 0 && self_inc != self_inc0) d.self_inc[ln] = self_inc;
  if (tick_round) {
    uint32_t am[W], sus = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      am[w] = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_ALIVE);
      sus |= __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_SUSPECT);
    }
    const uint4 x = target_block<W>(d, tick_round, self >> 2);
    uint4 y = make_uint4(0, 0, 0, 0);
    if (d.loss_ppm) y = philox4x32_10(make_uint4(tick_round, self >> 2, P_LOSS0, 0), d.key0, d.key1);
    uint32_t pings = 0;
    const bool need = node_needs_work<W>(d, 1u | (pbs.cnt << 8), am, td, sus, word_of(x, self & 3), word_of(y, self & 3),
                                         tick_round, pings, self); // (a receiver is a live process)
    if (lane == 0) {
      c.v[SWIM_CTR_PINGS] += pings;
      if (need) wl_of(d, tick_round)[atomicAdd(&d.wl_cnt[ci(tick_round)], 1u)] = ln;
    }
  }
}

// Warp-per-receiver walk over the receivers of `round`, f(ln, early, snd) for each: the compact list of delivered slots
// K1b wrote (early = true: the slot names one sender, snd, whose snapshot can be fetched with the row), then one list per
// source rank (cross-shard senders). A receiver can be listed more than once: the claim stamp lets exactly one warp
// process it. kSharded = false: a single-shard launch, which has no per-source-rank lists.
template <bool kSharded = true, typename F>
__device__ __forceinline__ void for_each_receiver(const SimDev &d, uint32_t round, uint32_t warp, uint32_t nwarps, F f) {
  const uint32_t par = round & 1;
  // items go to the warps from the top down: in the fused kernels the walk shares a phase with the scan, whose node ranges
  // fill the warps from the bottom up (at C3 the last 128 of 4,224 warps have no nodes to scan)
  const uint32_t w0 = nwarps - 1 - warp;
  const uint2 *cl_in = d.cl + (size_t)par * d.n * d.fanout;
  // this warp's first entry travels with the list's length (one memory round trip instead of two); only looked at if w0 < n_cl
  uint2 e_first = make_uint2(0u, 0u);
  if ((size_t)w0 < (size_t)d.n * d.fanout) {
    e_first.x = *(volatile const uint32_t *)&cl_in[w0].x;
    e_first.y = *(volatile const uint32_t *)&cl_in[w0].y;
  }
  const uint32_t n_cl = d.ncand[ci(round)];
  for (uint32_t item = w0; item < n_cl; item += nwarps) {
    const uint2 e = item == w0 ? e_first : cl_in[item];
    f(e.x, true, e.y);
  }
  if (kSharded && d.world > 1) {
    uint32_t seg_end[SWIM_MAX_WORLD + 1];
    uint32_t n_recv = 0;
    seg_end[0] = 0;
    for (uint32_t a = 0; a < d.world; ++a) {
      if (a != d.rank) n_recv += d.rcnt[par * d.world + a];
      seg_end[1 + a] = n_recv;
    }
    for (uint32_t item = w0; item < n_recv; item += nwarps) {
      uint32_t a = 0;
      while (item >= seg_end[1 + a]) ++a;
      f(d.rlr[((size_t)par * d.world + a) * d.rcap + (item - seg_end[a])], false, 0u);
    }
  }
}

template <int W, bool kSharded = true>
__device__ __forceinline__ void recv_pass(const SimDev &d, uint32_t round, uint32_t warp, uint32_t nwarps,
                                          int lane, PbStage &pbs, Ctr &c, uint32_t tick_round = 0) {
  for_each_receiver<kSharded>(d, round, warp, nwarps, [&](uint32_t ln, bool early, uint32_t snd) {
    recv_one<W>(d, round, ln, early, snd, lane, pbs, c, tick_round);
  });
}

// stand-alone K2 (profiling, staged NCCL exchange, sharded runs)
template <int W>
__global__ void __launch_bounds__(kThreads, kMinBlocks) recv_kernel(SimDev d) {
  SWIM_SHARED_2D(uint4, s_pb, kWarpsPerBlock, 32);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarpsPerBlock + wib, nwarps = gridDim.x * kWarpsPerBlock;
  pdl_launch();
  pdl_wait();
  const uint32_t round = d.round;
  Ctr c; c.clear();
  PbStage pbs; pbs.s = s_pb[wib];
  recv_pass<W>(d, round, warp, nwarps, lane, pbs, c); // sharded runs: the host launched peer_barrier_kernel before this
  c.flush(d.ctr, lane);
}

// =================================================================== one kernel per round
// Default path: K1a, K1b and K2 of one round in ONE launch, separated by grid-wide barriers (all CTAs
// are resident: the grid is one wave). A round in which nobody has anything to do beyond the probe
// (the steady state of a healthy cluster) ends after the scan: no K1b, no K2, no extra launches.
// Thread 0 of a CTA keeps its own copy of the generation word in shared memory: read once at kernel start
// (barrier_begin; no barrier of this launch can complete before every CTA has arrived, and the previous launch is over),
// then counted — every CTA takes part in every barrier — so arriving costs no global load ahead of the atomic.
__device__ __forceinline__ uint32_t *barrier_generation() {
  SWIM_SHARED_1D(uint32_t, s_bar_gen, 1);
  return s_bar_gen;
}
__device__ __forceinline__ void barrier_begin(const SimDev &d) {
  if (threadIdx.x == 0) *barrier_generation() = *(volatile uint32_t *)(d.gbar + 1);
}
// The grid barrier. Thread 0 of every CTA arrives behind a fence (at system scope with fence_sys: this CTA stored into
// peer memory since the last barrier); the last CTA to arrive does the barrier's job, if it has one, and releases the
// grid, while the others spin on the generation word. The jobs:
//   * cnt_dst: freeze a work-list length, *cnt_src -> *cnt_dst (round_kernel_x);
//   * kHandshake: the cross-GPU handshake of `round` (peer_handshake_cta, by all threads of the last CTA), if want() —
//     evaluated by the last CTA only, after every arrival is visible — says it is due (round_kernel folds it into the scan
//     barrier of a round that listed no work).
// Without kHandshake the barrier stays with thread 0 of each CTA: the form for call sites that cannot shard. The wait
// gives up after 6e9 cycles, or kPeerWaitCycles more where the last CTA may be handshaking. tl_slot: timeline slot of the
// last arrival (tl_mark_last).
struct Always {
  __device__ bool operator()() const { return true; }
};
// the last arrival's release of the grid, and everybody else's bounded wait for it (thread 0 of a CTA)
__device__ __forceinline__ void barrier_release(const SimDev &d, const uint32_t *cnt_src, uint32_t *cnt_dst) {
  if (cnt_dst) *(volatile uint32_t *)cnt_dst = *(volatile const uint32_t *)cnt_src;
  d.gbar[0] = 0;
  __threadfence();
  atomicAdd(d.gbar + 1, 1u);
}
__device__ __forceinline__ void barrier_wait(const SimDev &d, volatile uint32_t *gen, uint32_t g, long long limit) {
  const long long t0 = clock64();
  uint32_t polls = 0;
  while (*gen == g) {
    if (wait_expired(d, t0, limit, polls, 2)) break;
    __nanosleep(20);
  }
}
template <bool kHandshake = false, typename Want = Always>
__device__ __forceinline__ void grid_barrier(const SimDev &d, uint32_t round = 0, int tl_slot = -1, const uint32_t *cnt_src = nullptr,
                                             uint32_t *cnt_dst = nullptr, bool fence_sys = false, Want want = Want()) {
  __syncthreads();
  if constexpr (!kHandshake) {
    if (threadIdx.x == 0) {
      volatile uint32_t *gen = d.gbar + 1;
      const uint32_t g = (*barrier_generation())++;
      __threadfence();
      if (atomicAdd(d.gbar, 1u) == gridDim.x - 1) {
        if (cnt_dst) __threadfence(); // acquire side of the arrivals, ahead of the job
        tl_mark_last(d, round, tl_slot);
        barrier_release(d, cnt_src, cnt_dst);
      } else {
        barrier_wait(d, gen, g, 6000000000ll);
      }
      __threadfence();
    }
  } else {
    SWIM_SHARED_1D(uint32_t, s_last, 1);
    if (threadIdx.x == 0) {
      if (fence_sys) __threadfence_system(); else __threadfence();
      const bool last = atomicAdd(d.gbar, 1u) == gridDim.x - 1;
      if (last) { __threadfence(); tl_mark_last(d, round, tl_slot); } // acquire side of the arrivals
      s_last[0] = last ? 1u : 0u;
    }
    __syncthreads();
    if (s_last[0]) {
      if (want()) peer_handshake_cta(d, round);
      __syncthreads();
      if (threadIdx.x == 0) {
        (*barrier_generation())++;
        barrier_release(d, cnt_src, cnt_dst);
      }
    } else if (threadIdx.x == 0) {
      volatile uint32_t *gen = d.gbar + 1;
      const uint32_t g = (*barrier_generation())++;
      barrier_wait(d, gen, g, kPeerWaitCycles + 6000000000ll);
      __threadfence();
    }
  }
  __syncthreads();
}

// CTA-wide OR of a per-thread predicate (every thread of the CTA must call it)
__device__ __forceinline__ bool cta_or(bool pred) {
  SWIM_SHARED_1D(uint32_t, s_or, 1);
  if (threadIdx.x == 0) s_or[0] = 0;
  __syncthreads();
  if (pred) s_or[0] = 1; // same value from every writer
  __syncthreads();
  return s_or[0] != 0;
}

// zero one slot (mbw words) of a per-node bitmap — mailbits, workbits —, grid-strided over the warps of the launch
__device__ __forceinline__ void clear_bitmap(const SimDev &d, uint32_t *bits, uint32_t warp, uint32_t nwarps, int lane) {
  for (uint32_t x = warp * 32 + lane; x < d.mbw; x += nwarps * 32) bits[x] = 0;
}

// One batched quiet scan of the Q rounds first .. first+Q-1 (quiet_scan) and its grid barrier, in the interval of `round`:
// returns fb, the number of leading rounds that are quiet, and counts their Pings. The busy masks of the warps are OR-ed
// into qm[nb % 3]; slot (nb + 1) % 3 is cleared for the next batch, two barriers ahead of its use (the caller clears slot
// 0 before the first).
template <int W>
__device__ __forceinline__ uint32_t quiet_batch(const SimDev &d, uint32_t round, uint32_t first, uint32_t Q, uint32_t &nb,
                                                uint32_t warp, uint32_t nwarps, int lane, Ctr &c) {
  if (warp == 0 && lane == 0) d.qm[(nb + 1) % 3] = 0;
  uint32_t p1 = 0;
  uint32_t busy = quiet_scan<W>(d, first, Q, warp, nwarps, lane, p1);
  busy = __reduce_or_sync(kFull, busy);
  if (lane == 0 && busy) atomicOr(&d.qm[nb % 3], busy);
  tl_mark(d, round, 1);
  grid_barrier(d, round, 5);
  const uint32_t mask = *(volatile uint32_t *)&d.qm[nb % 3];
  ++nb;
  const uint32_t fb = mask ? (uint32_t)__ffs(mask) - 1u : Q;
  tl_mark(d, round, 2);
  c.v[SWIM_CTR_PINGS] += p1 * fb;
  return fb;
}

// Was mail of `round` delivered to nodes of this rank (behind the barrier that ends the round's K1b)? The length of the
// round's compact list of local deliveries — zero if nobody sent: the slot is cleared before the round starts — and,
// kSharded, the peers' counts of the receivers they listed here.
template <bool kSharded>
__device__ __forceinline__ bool mail_arrived(const SimDev &d, uint32_t round) {
  uint32_t got = *(volatile uint32_t *)&d.ncand[ci(round)];
  if (kSharded)
    for (uint32_t a = 0; a < d.world; ++a)
      if (a != d.rank) got |= *(volatile uint32_t *)&d.rcnt[(round & 1) * d.world + a];
  return got != 0;
}

// kSharded: the launch is one shard of a multi-GPU run with the fused peer-memory exchange (d.world > 1 && d.p2p); the
// single-shard instance has no handshake, no per-source-rank receive lists and no peer stores.
template <int W, bool kSharded>
__global__ void __launch_bounds__(kThreads, kMinBlocks) round_kernel(SimDev d) {
  SWIM_SHARED_2D(uint4, s_pb, kWarpsPerBlock, 32);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarpsPerBlock + wib, nwarps = gridDim.x * kWarpsPerBlock;
  pdl_launch();
  pdl_wait();
  barrier_begin(d);
  Ctr c; c.clear();
  PbStage pbs; pbs.s = s_pb[wib];
  // d.nrounds consecutive event-free rounds in this launch (the host splits calls at rounds that carry events). Per round:
  //   phase S  receive(round - 1) by the warps from the top down  ||  scan(round) by the warps from the bottom up
  //   barrier  (sharded: + cross-GPU handshake, when the round has no work to do)
  //   phase W  K1b(round): tick work and piggyback send            (skipped when the scan listed nothing)
  //   barrier  (sharded: + cross-GPU handshake)
  // The receive phase of a round has no barrier of its own: the few envelopes that survive the senders' membership
  // filter are applied while the next round's scan runs; the scan leaves their receivers alone (mail bitmap) and the
  // receiving warp takes their tick decision itself (recv_one). The last round's mail is applied before the launch ends.
  // Batched quiet scans (single shard, no loss): after a round that listed no work and got no mail, the next up to
  // d.qbatch rounds are decided by ONE pass over the meta records and ONE barrier (quiet_scan). Its busy mask is OR-ed
  // into qm[batch % 3]; a slot is cleared two batches (>= two barriers) before it is used again, slot 0 here, ahead of the
  // first round's barrier. While rounds are quiet all three list counters stay zero, so the ordinary path resumes at any round.
  const bool batching = d.qbatch > 1 && d.world == 1 && d.loss_ppm == 0;
  bool prev_quiet = false, mail = false; // mail: round - 1 delivered envelopes to nodes of this rank
  uint32_t nb = 0;
  if (batching && warp == 0 && lane == 0) d.qm[0] = 0;
  for (uint32_t it = 0; it < d.nrounds; ++it) {
    const uint32_t round = d.round + it;
    tl_mark(d, round, 0);
    // slot (round + 1) % 3 of the list counters was last used two rounds ago: clear it now, well before the
    // next round's scan (which starts after this round's first barrier) appends to it
    if (warp == 0 && lane == 0) { d.wl_cnt[ci(round + 1)] = 0; d.ncand[ci(round + 1)] = 0; }
    if (batching && prev_quiet && d.nrounds - it >= 2) {
      const uint32_t Q = d.qbatch < d.nrounds - it ? d.qbatch : d.nrounds - it;
      const uint32_t fb = quiet_batch<W>(d, round, round, Q, nb, warp, nwarps, lane, c); // rounds round .. round+fb-1: committed
      tl_mark(d, round, 7, fb);
      prev_quiet = fb == Q;
      if (fb) { it += fb - 1; continue; }
      // fb == 0: this very round has work — the ordinary scan below lists it
    }
    // ---- phase S
    const uint32_t *skip = nullptr;
    if (mail) {
      recv_pass<W, kSharded>(d, round - 1, warp, nwarps, lane, pbs, c, round); // K2 of the round before + those nodes' tick decision
      skip = d.mailbits + (size_t)((round - 1) % 3u) * d.mbw;
    }
    uint32_t pings = 0;
    scan_pass<W>(d, round, warp, nwarps, lane, pings, skip, pbs.s);       // K1a (the warp's staging area is free here)
    c.v[SWIM_CTR_PINGS] += pings;
    tl_mark(d, round, 1);
    const uint32_t *wl_cnt_r = d.wl_cnt + ci(round);
    // the work list is complete. Sharded: a rank that listed nothing has no K1b to run, so its cross-GPU handshake of the
    // round happens right here, inside this barrier (one barrier for a quiet round)
    if constexpr (kSharded) grid_barrier<true>(d, round, 5, nullptr, nullptr, false, [&] { return *(volatile const uint32_t *)wl_cnt_r == 0; });
    else grid_barrier(d, round, 5);
    tl_mark(d, round, 2);
    const uint32_t n_work = d.wl_cnt[ci(round)];
    const uint32_t first_ln = first_work_entry(d, round, warp);                  // in flight together with the count
    // last round's mail bitmap has been read by every scanner: clear it (its next writers: senders of round + 2)
    if (mail) clear_bitmap(d, d.mailbits + (size_t)((round - 1) % 3u) * d.mbw, warp, nwarps, lane);
    prev_quiet = n_work == 0 && !mail;
    // ---- phase W
    if (n_work) {
      const bool remote = work_pass<W, kSharded>(d, round, warp, nwarps, lane, pbs, c, first_ln, false); // K1b
      tl_mark(d, round, 3);
      // every flag and snapshot is written; sharded: ... on every rank (the last CTA talks to the peers)
      if constexpr (kSharded) grid_barrier<true>(d, round, 6, nullptr, nullptr, cta_or(remote));
      else grid_barrier(d, round, 6);
      tl_mark(d, round, 4);
    }
    // (no barrier is owed to the bitmap clear: that slot is written again by the senders of round + 2 and read again by
    // the scan of round + 3 — both behind the next round's barriers, on this rank and, through the handshake, on its peers)
    // Was anything delivered here in this round? (every envelope dropped at its sender, or nobody sent: no)
    mail = mail_arrived<kSharded>(d, round);
    if (mail) prev_quiet = false;
  }
  if (mail) { // the last round's mail, before the launch ends (no tick decision: the next launch scans everybody)
    recv_pass<W, kSharded>(d, d.round + d.nrounds - 1, warp, nwarps, lane, pbs, c, 0);
    // its bitmap is not needed by anybody: clear it. (The receive pass does not read it, so no barrier in between.)
    clear_bitmap(d, d.mailbits + (size_t)((d.round + d.nrounds - 1) % 3u) * d.mbw, warp, nwarps, lane);
  }
  c.flush(d.ctr, lane);
}

// =================================================================== one kernel per round, ONE grid barrier per round
// round_kernel_x: the two phases of round_kernel merged. Between the barriers B(r-1) and B(r) a warp does, for round r,
//   * the mail of round r-1 for the receivers it is given (x_node from the delivered-slot lists): apply it, take the node's
//     FINAL tick decision of round r, run K1b of round r right there if the node needs it, then its tick decision of r+1;
//   * K1b of round r for its items of the work list of round r (complete and frozen at B(r-1)); a listed node that also has
//     mail of round r-1 gets it applied first, by the same warp, on the row it has loaded anyway; then the decision of r+1;
//   * K1a of round r+1 for its slice of all other nodes (neither on the work list of r nor receivers of round r-1: nothing
//     touches them in this interval) — appending to the work list of r+1.
// A tick decision of round r+1 taken before B(r) is TENTATIVE for a node that turns out to receive mail in round r: the
// mail is applied behind B(r), and whoever applies it re-decides (and corrects the Ping count by the difference). Nothing
// else depends on the order of things inside an interval: a node's row, buffer and meta record are written by exactly one
// warp per interval, mail flags and snapshots are round-parity double-buffered, and the bitmaps (mail of round r in slot
// r % 3, work list of round r in slot r % 3) are cleared one interval after their last reader and one before their next
// writer. Result: bit-identical to round_kernel, one barrier (and one cross-GPU handshake) per round instead of two.

// One node of the interval of round `round` (see above). from_wl: the node is item `idx` of the round's work list; else it
// is a receiver of round - 1 named by a delivered slot (early / snd as in recv_one). mail: round - 1 delivered mail to
// nodes of this rank at all. decide: take the tick decision of round + 1 (false in the last round of a launch).
template <int W, bool kSharded>
__device__ __forceinline__ void x_node(const SimDev &d, uint32_t round, uint32_t ln, uint32_t idx, bool from_wl, bool mail, bool early,
                                       uint32_t snd, int lane, PbStage &pbs, Ctr &c, bool decide, bool &did_remote,
                                       uint32_t next_ln, bool have_next) {
  const uint32_t mround = round - 1, mpar = mround & 1;
  // everything that depends only on `ln` is issued together (one memory round trip)
  uint32_t old = 0, wbit = 0, mbit = 0;
  if (!from_wl) {
    if (lane == 0) old = atomicExch(&d.claim[ln], mround);
    wbit = d.workbits[(size_t)(round % 3u) * d.mbw + (ln >> 5)] >> (ln & 31) & 1u;
  } else if (mail) {
    mbit = d.mailbits[(size_t)(mround % 3u) * d.mbw + (ln >> 5)] >> (ln & 31) & 1u;
  }
  Row<W> row;
  row_load<W>(row, d, ln, lane);
  pb_load(pbs, d, ln, lane);
  uint32_t rix[W], td[W];
#pragma unroll
  for (int w = 0; w < W; ++w) {
    rix[w] = W <= 2 ? d.ridx[(size_t)ln * d.cap + w * 32 + lane] : 0u;
    td[w] = d.meta[(size_t)ln * W + w].z; // crashed-member bits: events only, not touched by mail or ticks
  }
  uint32_t e0 = 0, e1 = 0, self_inc = 0;
  uint4 early_rec = make_uint4(0, 0, 0, 0);
  uint32_t early_cnt = 0;
  if (!from_wl || mail) { // (loaded before the bits are known: a listed node without mail simply does not use them)
    e0 = d.in_off[ln]; e1 = d.in_off[ln + 1];
    self_inc = d.self_inc[ln];
    if (early) {
      if ((uint32_t)lane < d.B) early_rec = d.out[((size_t)mpar * d.per + snd) * d.B + lane];
      early_cnt = d.out_cnt[(size_t)mpar * d.per + snd];
    }
  }
  if (!from_wl) {
    // a receiver that is on this round's work list belongs to the warp that has it as an item; otherwise one warp per receiver
    if (wbit || __shfl_sync(kFull, old, 0) == mround) return;
  }
  const bool has_mail = !from_wl || mbit != 0;
  bool do_work = from_wl;
  if (has_mail) {
    uint32_t l_pre = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) l_pre += __popc(__ballot_sync(kFull, (row.st[w] & 3u) == SWIM_ALIVE));
    const uint32_t self_inc0 = self_inc;
    apply_mail<W>(d, mround, ln, e0, e1, early, snd, early_rec, early_cnt, row, pbs, self_inc, lane, c);
    row_store<W>(row, d, ln, lane, mround, td); // (lastChange = the round of the mail)
    row.touched = 0;
    row.ticked = 0;
    if (lane == 0 && self_inc != self_inc0) d.self_inc[ln] = self_inc;
    // The node's tick decision of `round` was taken before its mail was known: its Pings were counted from the row as it
    // was then — the row this warp loaded. Correct the count; a receiver that was not listed is decided again.
    uint32_t am[W], sus = 0, l_post = 0, risk = d.loss_ppm;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      am[w] = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_ALIVE);
      sus |= __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_SUSPECT);
      l_post += __popc(am[w]);
      risk |= am[w] & td[w];
    }
    const uint32_t p_pre = d.P < l_pre ? d.P : l_pre, p_post = d.P < l_post ? d.P : l_post;
    if (lane == 0) c.v[SWIM_CTR_PINGS] += p_post - p_pre; // (modulo 2^32; Ctr::flush extends the sign of this counter)
    if (!from_wl) {
      do_work = pbs.cnt != 0 || sus != 0;
      if (l_post && risk && !do_work) {
        const uint32_t self = d.first + ln;
        const uint4 x = target_block<W>(d, round, self >> 2);
        uint32_t ldraw = 0;
        if (d.loss_ppm) ldraw = word_of(philox4x32_10(make_uint4(round, self >> 2, P_LOSS0, 0), d.key0, d.key1), self & 3);
        do_work = probe_fails<W>(d, am, td, l_post, word_of(x, self & 3), ldraw, round, self);
      }
      if (do_work) { // behind the frozen part of the list: nobody walks it, its position carries the node's recipient slots
        if (lane == 0) {
          idx = atomicAdd(&d.wl_cnt[ci(round)], 1u);
          wl_of(d, round)[idx] = ln;
        }
        idx = __shfl_sync(kFull, idx, 0);
      }
    }
  }
  if (do_work) work_body<W, kSharded>(d, round, ln, idx, row, rix, td, pbs, c, lane, did_remote, next_ln, have_next);
  else pb_store(pbs, d, ln, lane);
  if (decide) tick_decide<W>(d, round + 1, ln, row, pbs.cnt, td, lane, c, d.workbits + (size_t)((round + 1) % 3u) * d.mbw);
}

template <int W, bool kSharded> // (kSharded: as for round_kernel)
__global__ void __launch_bounds__(kThreads, kMinBlocks) round_kernel_x(SimDev d) {
  SWIM_SHARED_2D(uint4, s_pb, kWarpsPerBlock, 32);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarpsPerBlock + wib, nwarps = gridDim.x * kWarpsPerBlock;
  pdl_launch();
  pdl_wait();
  barrier_begin(d);
  Ctr c; c.clear();
  PbStage pbs; pbs.s = s_pb[wib];
  const bool batching = d.qbatch > 1 && d.world == 1 && d.loss_ppm == 0;
  const uint32_t last_round = d.round + d.nrounds - 1;
  bool mail = false;       // round - 1 delivered envelopes to nodes of this rank
  bool have_wl = false;    // the work list of `round` exists (its length frozen in wl_n)
  bool known_empty = false; // ... and is known to be empty (a batched quiet scan decided the round)
  bool wb_prev = false;    // the work list of round - 1 had entries (its bitmap slot wants clearing)
  bool mail_prev = false;  // round - 2 delivered mail (its bitmap slot wants clearing)
  uint32_t nb = 0;
  if (batching && warp == 0 && lane == 0) d.qm[0] = 0;
  for (uint32_t it = 0; it < d.nrounds; ++it) {
    const uint32_t round = d.round + it;
    if (!have_wl) {
      // K1a of `round` over every node on its own (the first round of a launch, and the first busy round behind a batch of
      // quiet ones): nothing is pending — no mail, no list — so nothing is skipped
      if (warp == 0 && lane == 0) { d.wl_cnt[ci(round + 1)] = 0; d.ncand[ci(round)] = 0; }
      uint32_t pings = 0;
      scan_pass<W>(d, round, warp, nwarps, lane, pings, nullptr, pbs.s, nullptr, d.workbits + (size_t)(round % 3u) * d.mbw);
      c.v[SWIM_CTR_PINGS] += pings;
      grid_barrier(d, round, -1, d.wl_cnt + ci(round), d.wl_n + ci(round));
      have_wl = true;
      known_empty = false;
    }
    tl_mark(d, round, 0);
    const uint32_t n_work = known_empty ? 0u : *(volatile const uint32_t *)&d.wl_n[ci(round)];
    const bool last = round == last_round;
    // the bitmap of the work list of round - 1: read in the last interval, written again in the next one; the mail bitmap
    // of round - 2 likewise (its next writers: the senders of round + 1)
    if (wb_prev) clear_bitmap(d, d.workbits + (size_t)((round - 1) % 3u) * d.mbw, warp, nwarps, lane);
    if (mail_prev) clear_bitmap(d, d.mailbits + (size_t)((round - 2) % 3u) * d.mbw, warp, nwarps, lane);
    if (batching && n_work == 0 && !mail && !last) {
      // `round` is quiet — nothing to apply, nothing to run — and so committed. One pass decides rounds round+1 .. round+Q.
      // (No list is appended to and no mail counted while rounds are quiet: all counters of the three slots are cleared.)
      const uint32_t Q = d.qbatch < last_round - round ? d.qbatch : last_round - round;
      if (warp == 0 && lane == 0) { d.wl_cnt[ci(round + 1)] = 0; d.wl_cnt[ci(round + 2)] = 0; d.ncand[ci(round + 1)] = 0; }
      const uint32_t fb = quiet_batch<W>(d, round, round + 1, Q, nb, warp, nwarps, lane, c); // rounds round+1 .. round+fb are quiet too
      tl_mark(d, round, 7, fb == Q ? Q : fb + 1); // rounds committed by this pass
      // fb == Q: round+Q is decided (quiet) but not yet committed: it is the next current round, with a list known to be
      // empty. fb < Q: round+fb+1 is busy: it gets the ordinary scan above.
      if (fb == Q) { it += Q - 1; known_empty = true; }
      else { it += fb; have_wl = false; known_empty = false; }
      wb_prev = false;
      mail_prev = false;
      continue;
    }
    // ---- the interval of `round`
    if (warp == 0 && lane == 0) { d.wl_cnt[ci(round + 2)] = 0; d.ncand[ci(round + 1)] = 0; }
    bool did_remote = false;
    if (mail) { // receivers of round - 1: from the top warp down (the scan below fills the warps from the bottom up)
      const uint32_t mpar = (round - 1) & 1;
      const uint32_t w0 = nwarps - 1 - warp;
      const uint32_t n_cl = d.ncand[ci(round - 1)];
      const uint2 *cl_in = d.cl + (size_t)mpar * d.n * d.fanout;
      for (uint32_t item = w0; item < n_cl; item += nwarps) {
        const uint2 e = cl_in[item];
        x_node<W, kSharded>(d, round, e.x, 0u, false, true, true, e.y, lane, pbs, c, !last, did_remote, 0u, false);
      }
      if (kSharded) {
        uint32_t seg_end[SWIM_MAX_WORLD + 1];
        uint32_t n_recv = 0;
        seg_end[0] = 0;
        for (uint32_t a = 0; a < d.world; ++a) {
          if (a != d.rank) n_recv += d.rcnt[mpar * d.world + a];
          seg_end[1 + a] = n_recv;
        }
        for (uint32_t item = w0; item < n_recv; item += nwarps) {
          uint32_t a = 0;
          while (item >= seg_end[1 + a]) ++a;
          const uint32_t ln = d.rlr[((size_t)mpar * d.world + a) * d.rcap + (item - seg_end[a])];
          x_node<W, kSharded>(d, round, ln, 0u, false, true, false, 0u, lane, pbs, c, !last, did_remote, 0u, false);
        }
      }
    }
    if (n_work) { // K1b of `round` (+ a listed node's own mail) (+ its tick decision of round + 1)
      const uint32_t *wl = wl_of(d, round);
      uint32_t next_ln = warp < n_work ? *(volatile const uint32_t *)(wl + warp) : 0u;
      for (uint32_t idx = warp; idx < n_work; idx += nwarps) {
        const uint32_t ln = next_ln;
        const bool have_next = idx + nwarps < n_work;
        if (have_next) next_ln = *(volatile const uint32_t *)(wl + idx + nwarps);
        x_node<W, kSharded>(d, round, ln, idx, true, mail, false, 0u, lane, pbs, c, !last, did_remote, next_ln, have_next);
      }
    }
    if (!last) { // K1a of round + 1 for everybody else
      uint32_t pings = 0;
      scan_pass<W>(d, round + 1, warp, nwarps, lane, pings, mail ? d.mailbits + (size_t)((round - 1) % 3u) * d.mbw : nullptr, pbs.s,
                   n_work ? d.workbits + (size_t)(round % 3u) * d.mbw : nullptr, d.workbits + (size_t)((round + 1) % 3u) * d.mbw);
      c.v[SWIM_CTR_PINGS] += pings;
    }
    tl_mark(d, round, 1);
    // every flag, snapshot and list entry of the round is written (sharded: ... on every rank — the last CTA talks to the peers)
    if constexpr (kSharded) grid_barrier<true>(d, round, 5, d.wl_cnt + ci(round + 1), d.wl_n + ci(round + 1), cta_or(did_remote));
    else grid_barrier(d, round, 5, d.wl_cnt + ci(round + 1), d.wl_n + ci(round + 1));
    tl_mark(d, round, 2);
    tl_mark(d, round, 4, (unsigned long long)(n_work || mail)); // 1: a busy round (bench.py tells busy from quiet rounds by it)
    mail_prev = mail;
    wb_prev = n_work != 0;
    mail = mail_arrived<kSharded>(d, round);
    known_empty = false;
  }
  // the last round's mail, before the launch ends (no tick decision: the next launch scans everybody)
  if (mail) recv_pass<W, kSharded>(d, last_round, warp, nwarps, lane, pbs, c, 0);
  // bitmaps still set: the mail of the last two rounds and the work lists (this rank's own affair: all three slots). Never
  // the mail slot of last + 1: a peer that is already in its next launch may be marking receivers there.
  clear_bitmap(d, d.mailbits + (size_t)(last_round % 3u) * d.mbw, warp, nwarps, lane);
  clear_bitmap(d, d.mailbits + (size_t)((last_round + 2u) % 3u) * d.mbw, warp, nwarps, lane); // (= last - 1)
  for (uint32_t s = 0; s < 3; ++s) clear_bitmap(d, d.workbits + (size_t)s * d.mbw, warp, nwarps, lane);
  c.flush(d.ctr, lane);
}

// =================================================================== events (phase E)
// Keep the crashed-member bitmaps in step with alive[]: every row of this shard that lists
// `node` has the corresponding bit set (crash) or cleared (rejoin), and a crash marks the row exposed.
__device__ __forceinline__ void mark_observers(const SimDev &d, uint32_t node, bool crashed, int lane) {
  const uint32_t W = d.cap >> 5;
  for (uint32_t x = d.obs_off[node] + lane, end = d.obs_off[node + 1]; x < end; x += 32) {
    const uint32_t slot = d.obs_slot[x], l = slot / d.cap, s = slot % d.cap;
    uint32_t *word = reinterpret_cast<uint32_t *>(d.meta + (size_t)l * W + (s >> 5)) + 2;
    if (crashed) {
      atomicOr(word, 1u << (s & 31));
      atomicOr(&d.nsum[l], kNsExposed); // whatever the slot's liveness: an INJECT on row l may be making it Alive right now
    } else {
      atomicAnd(word, ~(1u << (s & 31))); // (the exposed bit stays: spurious until the row's next store, never missing)
    }
  }
}

// Rebuild every per-node meta record and summary word from the primary arrays (after bulk edits of alive[], rows
// or buffers through the ABI): bitmaps from the row's liveness, crashed members from alive[nbr].
static __global__ void __launch_bounds__(kThreads) derive_meta_kernel(SimDev d) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  const uint32_t W = d.cap >> 5;
  for (uint32_t l = warp; l < d.n; l += nwarps) {
    uint32_t L = 0, sus = 0, ex = 0;
    for (uint32_t w = 0; w < W; ++w) {
      const size_t x = (size_t)l * d.cap + w * 32 + lane;
      const uint32_t live = d.vst[x] & 3u;
      const unsigned am = __ballot_sync(kFull, live == SWIM_ALIVE);
      const unsigned sm = __ballot_sync(kFull, live == SWIM_SUSPECT);
      const unsigned td = __ballot_sync(kFull, live != SWIM_VACANT && d.alive[d.nbr[x]] == 0);
      if (lane == 0) d.meta[(size_t)l * W + w] = make_uint4(am, sm, td, 0u);
      L += __popc(am);
      sus |= sm;
      ex |= am & td;
    }
    if (lane == 0)
      d.nsum[l] = (d.alive[d.first + l] ? 1u : 0u) | ((uint32_t)d.pb_cnt[l] << 8) |
                  ((L < 4u ? L : 4u) << 16) | (sus ? kNsSus : 0u) | (ex ? kNsExposed : 0u);
  }
}

struct DevEvent {
  uint32_t node;
  uint32_t kind;
  uint4 rec; // SWIM_EV_INJECT
};

// Phase C — seeded churn (BASELINE config C5), one thread per Philox group of four nodes, every rank for all N nodes
// (alive[] and back_at[] are replicated): a live process crashes with probability churn_ppm / 1e6 and is given its rejoin
// round; a crashed process whose round has come rejoins. The kernel only decides and schedules: the effects (alive[],
// crashed-member bitmaps of the observers, incarnation + 1 and the Alive broadcast of a rejoin) are event_kernel's, fed
// with the list written here — the very code path of host-injected SWIM_EV_CRASH / SWIM_EV_REJOIN events.
static __global__ void __launch_bounds__(256) churn_kernel(SimDev d) {
  pdl_launch();
  pdl_wait();
  const uint32_t round = d.round;
  uint32_t *const cnt = d.churn_cnt + (round & 1u); // this round's list counter; the other slot is cleared for round + 1
  if (blockIdx.x == 0 && threadIdx.x == 0) d.churn_cnt[(round + 1u) & 1u] = 0;
  for (uint32_t g = blockIdx.x * blockDim.x + threadIdx.x; 4 * g < d.N; g += gridDim.x * blockDim.x) {
    const uint32_t base = 4 * g;
    uint32_t up4 = 0; // alive bytes of the four nodes
    if (base + 4 <= d.N) up4 = *reinterpret_cast<const uint32_t *>(d.alive + base);
    else for (uint32_t j = 0; base + j < d.N; ++j) up4 |= (uint32_t)d.alive[base + j] << (8 * j);
    const uint4 x = philox4x32_10(make_uint4(round, g, P_CHURN, 0), d.key0, d.key1);
    uint4 y = make_uint4(0, 0, 0, 0);
    bool have_y = false;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const uint32_t i = base + j;
      if (i >= d.N) break;
      uint32_t kind = 0xFFFFFFFFu;
      if (up4 >> (8 * j) & 0xFFu) {
        if (bounded(word_of(x, j), 1000000u) < d.churn_ppm) {
          if (!have_y) { y = philox4x32_10(make_uint4(round, g, P_CHURN, 1), d.key0, d.key1); have_y = true; }
          d.back_at[i] = round + d.rejoin_min + bounded(word_of(y, j), d.rejoin_span);
          kind = SWIM_EV_CRASH;
        }
      } else if (d.back_at[i] == round) {
        d.back_at[i] = 0;
        kind = SWIM_EV_REJOIN;
      }
      if (kind != 0xFFFFFFFFu) {
        const uint32_t k = atomicAdd(cnt, 1u);
        if (k < d.churn_cap) { d.churn_ev[k].node = i; d.churn_ev[k].kind = kind; d.churn_ev[k].rec = make_uint4(0, 0, 0, 0); }
        else *d.bar_err = 3; // list overflow: reported by swim_sim_sync, never silent
      }
    }
  }
}

template <int W>
__global__ void __launch_bounds__(kThreads) event_kernel(SimDev d, const DevEvent *ev, uint32_t n_ev, const uint32_t *n_ev_dev) {
  SWIM_SHARED_2D(uint4, s_pb, kWarpsPerBlock, 32);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarpsPerBlock + wib, nwarps = gridDim.x * kWarpsPerBlock;
  pdl_launch();
  pdl_wait();
  Ctr c; c.clear();
  PbStage pbs; pbs.s = s_pb[wib];
  const uint32_t round = d.round;
  if (n_ev_dev) n_ev = *n_ev_dev < d.churn_cap ? *n_ev_dev : d.churn_cap; // device-generated list (churn_kernel)
  // The host hands over one round's events grouped by node (stable: a node's events keep the order they were given in).
  // A run of same-node events belongs to the warp whose stride position is the run's first event, so a warp looks at
  // n_ev / nwarps list entries plus the runs it owns — not at the whole list.
  for (uint32_t x0 = warp; x0 < n_ev; x0 += nwarps) {
   const uint32_t node = ev[x0].node;
   if (x0 && ev[x0 - 1].node == node) continue; // inside somebody else's run
   for (uint32_t x = x0; x < n_ev && ev[x].node == node; ++x) {
    const uint32_t kind = ev[x].kind;
    const bool local = node >= d.first && node < d.first + d.n;
    const uint32_t ln = node - d.first;
    if (kind == SWIM_EV_CRASH) {
      const bool was_up = d.alive[node] != 0;
      __syncwarp();
      if (lane == 0) {
        d.alive[node] = 0;
        if (was_up) d.last_crash[node] = round;
        if (local) atomicAnd(&d.nsum[ln], ~0xFFu); // byte 0: up
      }
      mark_observers(d, node, true, lane);
    } else if (kind == SWIM_EV_REJOIN) {
      const bool was_up = d.alive[node] != 0;
      __syncwarp();
      if (!was_up) {
        if (lane == 0) {
          d.alive[node] = 1;
          d.last_rejoin[node] = round;
          if (local) atomicOr(&d.nsum[ln], 1u);
        }
        mark_observers(d, node, false, lane);
        if (local) { // restart with incarnation + 1 and announce Alive
          uint32_t inc = d.self_inc[ln] + 1;
          __syncwarp();
          if (lane == 0) d.self_inc[ln] = inc;
          pb_load(pbs, d, ln, lane);
          pb_enqueue(pbs, d, make_rec(node, inc, 0, SWIM_MSG_ALIVE), lane, c.v[SWIM_CTR_PB_DROPPED]);
          pb_store(pbs, d, ln, lane, true);
        }
      }
    } else if (local && d.alive[node] != 0) { // SWIM_EV_INJECT: one datagram through `process`
      Row<W> row;
      row_load<W>(row, d, ln, lane);
      pb_load(pbs, d, ln, lane);
      uint32_t td[W];
#pragma unroll
      for (int w = 0; w < W; ++w) td[w] = d.meta[(size_t)ln * W + w].z;
      uint32_t self_inc = d.self_inc[ln];
      const uint32_t self_inc0 = self_inc;
      uint4 rb;
      if (row_apply<W>(row, d, node, self_inc, ev[x].rec, rb, lane, c.v[SWIM_CTR_REFUTES]) == 1) {
        pb_enqueue(pbs, d, rb, lane, c.v[SWIM_CTR_PB_DROPPED]);
        if (lane == 0) ++c.v[SWIM_CTR_RECS_APPLIED];
      }
      row_store<W>(row, d, ln, lane, round, td, true);
      pb_store(pbs, d, ln, lane, true);
      if (lane == 0 && self_inc != self_inc0) d.self_inc[ln] = self_inc;
    }
    __syncwarp();
   }
  }
  c.flush(d.ctr, lane);
}

// =================================================================== digest / convergence
__device__ __forceinline__ uint64_t fmix64(uint64_t x) {
  x ^= x >> 33; x *= 0xff51afd7ed558ccdull; x ^= x >> 33; x *= 0xc4ceb9fe1a85ec53ull; x ^= x >> 33;
  return x;
}
// digest term of one element group: tag 1 = node scalars, 2 = view slot, 3 = piggyback record
__device__ __forceinline__ uint64_t dg3(uint64_t tag, uint64_t idx, uint64_t w0, uint64_t w1) {
  return fmix64(fmix64(fmix64(idx + (tag << 56)) ^ w0) ^ w1);
}

// One thread per view slot / node / record, grid-stride, fully coalesced; three fmix64 per element group.
static __global__ void __launch_bounds__(kThreads) digest_kernel(SimDev d, unsigned long long *out) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nthr = (size_t)gridDim.x * blockDim.x;
  uint64_t acc = 0;
  const size_t slots = (size_t)d.n * d.cap;
  for (size_t x = tid; x < slots; x += nthr) {
    const uint64_t gi = (uint64_t)d.first * d.cap + x;
    acc += dg3(2, gi, (uint64_t)d.nbr[x] | ((uint64_t)d.vinc[x] << 32), (uint64_t)d.vst[x] | ((uint64_t)d.vlast[x] << 8));
  }
  for (size_t l = tid; l < d.n; l += nthr) {
    const uint64_t g = d.first + l;
    acc += dg3(1, g, (uint64_t)d.self_inc[l] | ((uint64_t)d.seqno[l] << 32), (uint64_t)d.alive[g] | ((uint64_t)d.pb_cnt[l] << 8));
  }
  const size_t recs = (size_t)d.n * d.B;
  for (size_t x = tid; x < recs; x += nthr) {
    const size_t l = x / d.B, q = x % d.B;
    if (q >= d.pb_cnt[l]) continue;
    const uint4 r = d.pb[x];
    acc += dg3(3, (uint64_t)d.first * d.B + x, (uint64_t)r.x | ((uint64_t)r.y << 32),
               (uint64_t)r.z | ((uint64_t)(r.w & 0xFFu) << 32) | ((uint64_t)((r.w >> 8) & 0xFFu) << 40));
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) acc += __shfl_xor_sync(kFull, acc, o);
  if ((threadIdx.x & 31) == 0 && acc) atomicAdd(out, (unsigned long long)acc);
}

// Convergence detector: view entries of live observers that disagree with the truth. Uses the
// crashed-member bitmap of the meta record (current: the host rebuilds it first when it is dirty),
// so a slot costs one state byte and a shared 16-byte record instead of two gathers.
// Convergence count from the per-node meta records alone (16 B per node; the kernels keep them in step with the rows):
// a view entry of a live observer is wrong when the member is down and the entry is not Dead, or the member is up and
// the entry is not Alive. Only entries that are neither Alive nor Suspect of members that are up need the state byte
// (Dead is wrong, vacant is not counted) — none on a full row in steady state.
__device__ __forceinline__ uint32_t count_mismatches(const SimDev &d) {
  const uint32_t W = d.cap >> 5;
  uint32_t bad = 0;
  for (size_t l = (size_t)blockIdx.x * blockDim.x + threadIdx.x; l < d.n; l += (size_t)gridDim.x * blockDim.x) {
    if (!ns_up(d.nsum[l])) continue; // a crashed observer's view does not count
    for (uint32_t w = 0; w < W; ++w) {
      const uint4 m = d.meta[l * W + w];
      bad += __popc(m.z & (m.x | m.y)) + __popc(m.y & ~m.z);
      uint32_t rest = ~(m.x | m.y | m.z);
      while (rest) {
        const uint32_t s = __ffs(rest) - 1;
        rest &= rest - 1;
        bad += (d.vst[l * d.cap + w * 32 + s] & 3u) == SWIM_DEAD;
      }
    }
  }
  return bad;
}

static __global__ void __launch_bounds__(kThreads) mismatch_kernel(SimDev d, unsigned long long *out) {
  const uint32_t bad = __reduce_add_sync(kFull, count_mismatches(d));
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(out, (unsigned long long)bad);
}

// swim_sim_step_observe: the read-back of a convergence-study loop without a copy engine operation and without a stream
// synchronisation. Chained behind the round kernel (programmatic stream serialization), it counts the view entries
// that disagree with the truth; the last CTA to finish writes the cumulative counters, that count and finally a sequence
// number into pinned host memory mapped into the device (PCIe writes), and re-arms the accumulators. The host polls the
// sequence number.
static __global__ void __launch_bounds__(kThreads) observe_kernel(SimDev d, unsigned long long *acc, uint32_t *done,
                                                                  volatile unsigned long long *host_out, unsigned long long seq) {
  SWIM_SHARED_1D(uint32_t, s_last, 1);
  pdl_launch();
  pdl_wait();
  const uint32_t bad = __reduce_add_sync(kFull, count_mismatches(d));
  if ((threadIdx.x & 31) == 0 && bad) atomicAdd(acc, (unsigned long long)bad);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    s_last[0] = atomicAdd(done, 1u) == gridDim.x - 1 ? 1u : 0u;
    __threadfence();
  }
  __syncthreads();
  if (!s_last[0]) return;
  if (threadIdx.x < SWIM_CTR__COUNT) host_out[threadIdx.x] = *(volatile unsigned long long *)&d.ctr[threadIdx.x];
  if (threadIdx.x == 0) {
    host_out[SWIM_CTR__COUNT] = atomicExch(acc, 0ull); // ... and the accumulator is zero again for the next call
    host_out[SWIM_CTR__COUNT + 1] = *(volatile uint32_t *)d.bar_err;
    *done = 0;
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) host_out[SWIM_CTR__COUNT + 2] = seq;
}

} // namespace swim
