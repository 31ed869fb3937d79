// swim_scalar.cu — scalar Core.hs parity calls on ONE simulated node's store.
//
// Each call launches a single warp that runs the same device functions as the bulk kernels
// (row_apply = suspectOrDeadNode'/aliveNode, pick_remove = shuffle), so the reference's unit
// tests (test/Spec.hs) can be restated against the accelerated implementation.
#include <algorithm>
#include <cstring>
#include <vector>

#include "swim_host.h"

using namespace swim;

#define CUDA_TRY(sim, call)                                                                       \
  do {                                                                                            \
    cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) {                                                                      \
      set_error(sim, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return SWIM_ECUDA;                                                                          \
    }                                                                                             \
  } while (0)

namespace {

enum : uint32_t { OP_APPLY = 0, OP_KRANDOM = 1, OP_REMOVE_DEAD = 2, OP_NEXT_SEQNO = 3, OP_NEXT_INC = 4, OP_ENQUEUE = 5, OP_TICK_TIMERS = 6, OP_SPEND = 7 };

struct ScalarArgs {
  uint32_t op, node, n, allow_insert;
  uint32_t call; // Philox counter word 0 of this kRandomMembers call
  uint32_t excl[8];
  uint4 rec;
  // results
  int32_t err;
  uint32_t verdict, value, n_out;
  uint4 rb;
  uint32_t slots[SWIM_MAX_VIEW];
};

template <int W>
__global__ void scalar_kernel(SimDev d, ScalarArgs *a) {
  SWIM_SHARED_1D(uint4, s_pb, 32);
  const int lane = threadIdx.x;
  const uint32_t ln = a->node - d.first;
  uint32_t dummy = 0;
  if (lane == 0) { a->err = 0; a->verdict = 0; a->n_out = 0; }
  __syncwarp();
  switch (a->op) {
    case OP_NEXT_SEQNO: // nextSeqNo = atomicIncr . storeSeqNo (Core.hs:49-50): returns the new value
      if (lane == 0) a->value = ++d.seqno[ln];
      break;
    case OP_NEXT_INC: // nextIncarnation (Core.hs:52-53)
      if (lane == 0) a->value = ++d.self_inc[ln];
      break;
    case OP_APPLY: { // suspectNode / deadNode / aliveNode (Core.hs:189-218)
      Row<W> row;
      row_load<W>(row, d, ln, lane);
      uint32_t td[W];
      for (int w = 0; w < W; ++w) td[w] = d.meta[(size_t)ln * W + w].z;
      uint32_t self_inc = d.self_inc[ln];
      const uint32_t self_inc0 = self_inc;
      uint4 rb = make_uint4(0, 0, 0, 0);
      int v = row_apply<W>(row, d, a->node, self_inc, a->rec, rb, lane, dummy);
      row_store<W>(row, d, ln, lane, d.round, td);
      __syncwarp();
      if (lane == 0) {
        if (self_inc != self_inc0) d.self_inc[ln] = self_inc;
        if (v == 2 && a->allow_insert) {
          // addNewMember (Core.hs:206-216): Map.insert keeps the row in key order
          const size_t base = (size_t)ln * d.cap;
          uint32_t used = 0;
          while (used < d.cap && (d.vst[base + used] & 3u) != SWIM_VACANT) ++used;
          if (used == d.cap) {
            a->err = SWIM_ECAP;
            v = 0;
          } else {
            uint32_t pos = 0;
            while (pos < used && d.nbr[base + pos] < a->rec.x) ++pos;
            for (uint32_t x = used; x > pos; --x) {
              d.nbr[base + x] = d.nbr[base + x - 1]; d.vst[base + x] = d.vst[base + x - 1];
              d.vinc[base + x] = d.vinc[base + x - 1]; d.vlast[base + x] = d.vlast[base + x - 1];
            }
            d.nbr[base + pos] = a->rec.x; d.vst[base + pos] = SWIM_ALIVE;
            d.vinc[base + pos] = a->rec.y; d.vlast[base + pos] = d.round;
            rb = a->rec;
            v = 3; // applied by insertion: membership changed
          }
        } else if (v == 2) {
          v = 0;
        }
        a->verdict = (uint32_t)v;
        a->rb = rb;
      }
      break;
    }
    case OP_KRANDOM: { // kRandomMembers (Core.hs:69-74) over shuffle (Util.hs:36-42)
      Row<W> row;
      row_load<W>(row, d, ln, lane);
      uint32_t cand[W], L = 0;
#pragma unroll
      for (int w = 0; w < W; ++w) {
        cand[w] = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_ALIVE) & ~a->excl[w]; // isAlive && notElem
        L += __popc(cand[w]);
      }
      const uint32_t want = a->n < L ? a->n : L;
      if (lane == 0) {
        uint4 blk = make_uint4(0, 0, 0, 0);
        for (uint32_t x = 0; x < want; ++x) {
          if ((x & 3) == 0) blk = philox4x32_10(make_uint4(a->call, a->node, P_SCALAR, x >> 2), d.key0, d.key1);
          a->slots[x] = pick_remove<W>(cand, bounded(word_of(blk, x & 3), L - x));
        }
        a->n_out = want;
      }
      break;
    }
    case OP_ENQUEUE: { // disseminate: Broadcast msg -> enqueue (Core.hs:131,136-138), same buffer code as the bulk kernels
      PbStage pbs;
      pbs.s = s_pb;
      pb_load(pbs, d, ln, lane);
      pb_enqueue(pbs, d, a->rec, lane, dummy);
      pb_store(pbs, d, ln, lane);
      if (lane == 0) a->value = dummy; // 1 = the oldest record fell off a full buffer
      break;
    }
    case OP_TICK_TIMERS: { // phase T1 for one store: the same countdown / expiry code as work_pass
      Row<W> row;
      row_load<W>(row, d, ln, lane);
      uint32_t td[W];
      for (int w = 0; w < W; ++w) td[w] = d.meta[(size_t)ln * W + w].z;
      PbStage pbs;
      pbs.s = s_pb;
      pb_load(pbs, d, ln, lane);
      uint32_t expired = 0;
#pragma unroll
      for (int w = 0; w < W; ++w) {
        if ((row.st[w] & 3u) == SWIM_SUSPECT) { row.st[w] -= 4u; row.ticked |= 1u << w; }
        unsigned em = __ballot_sync(kFull, (row.st[w] & 3u) == SWIM_SUSPECT && ((row.st[w] >> 2) & d.tmask) == 0);
        if (em >> lane & 1u) { row.st[w] = SWIM_DEAD; row.touched |= 1u << w; }
        while (em) {
          const int s = __ffs(em) - 1;
          em &= em - 1;
          const uint32_t m = __shfl_sync(kFull, row.nb[w], s), i = __shfl_sync(kFull, row.inc[w], s);
          pb_enqueue(pbs, d, make_rec(m, i, a->node, SWIM_MSG_DEAD), lane, dummy);
          ++expired;
        }
      }
      row_store<W>(row, d, ln, lane, d.round, td);
      pb_store(pbs, d, ln, lane);
      if (lane == 0) a->value = expired;
      break;
    }
    case OP_SPEND: { // phase T4's "one transmission is spent on every record" for one store
      PbStage pbs;
      pbs.s = s_pb;
      pb_load(pbs, d, ln, lane);
      uint4 mine = make_uint4(0, 0, 0, 0);
      const bool have = (uint32_t)lane < pbs.cnt;
      if (have) mine = pbs.s[lane];
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
      pb_store(pbs, d, ln, lane);
      break;
    }
    case OP_REMOVE_DEAD: // removeDeadNodes (Core.hs:65-67): Map.filter (not . isDead)
      if (lane == 0) {
        const size_t base = (size_t)ln * d.cap;
        uint32_t w = 0;
        for (uint32_t s = 0; s < d.cap; ++s) {
          const uint32_t live = d.vst[base + s] & 3u;
          if (live == SWIM_VACANT || live == SWIM_DEAD) continue;
          d.nbr[base + w] = d.nbr[base + s]; d.vst[base + w] = d.vst[base + s];
          d.vinc[base + w] = d.vinc[base + s]; d.vlast[base + w] = d.vlast[base + s];
          ++w;
        }
        a->value = w;
        for (; w < d.cap; ++w) {
          d.nbr[base + w] = SWIM_NO_MEMBER; d.vst[base + w] = SWIM_VACANT; d.vinc[base + w] = 0; d.vlast[base + w] = 0;
        }
      }
      break;
  }
}

int run_scalar(swim_sim *sim, ScalarArgs &h) {
  cudaSetDevice(sim->device);
  if (!sim->d_sargs) {
    CUDA_TRY(sim, cudaMalloc(&sim->d_sargs, sizeof(ScalarArgs)));
    sim->allocs.push_back(sim->d_sargs);
  }
  SimDev d = sim->dev;
  d.round = sim->round;
  ScalarArgs *da = (ScalarArgs *)sim->d_sargs;
  CUDA_TRY(sim, cudaMemcpyAsync(da, &h, sizeof h, cudaMemcpyHostToDevice, sim->stream));
  switch (d.cap / 32) {
    case 1: SWIM_LAUNCH(scalar_kernel<1>, 1, 32, sim->stream, d, da); break;
    case 2: SWIM_LAUNCH(scalar_kernel<2>, 1, 32, sim->stream, d, da); break;
    case 4: SWIM_LAUNCH(scalar_kernel<4>, 1, 32, sim->stream, d, da); break;
    default: SWIM_LAUNCH(scalar_kernel<8>, 1, 32, sim->stream, d, da); break;
  }
  CUDA_TRY(sim, cudaGetLastError());
  ++sim->launches;
  CUDA_TRY(sim, cudaMemcpyAsync(&h, da, sizeof h, cudaMemcpyDeviceToHost, sim->stream));
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  return h.err;
}

int check_node(swim_sim *sim, uint32_t node) {
  if (!sim) return SWIM_EINVAL;
  if (node < sim->dev.first || node >= sim->dev.first + sim->dev.n) {
    set_error(sim, "node %u is not owned by this rank [%u, %u)", node, sim->dev.first, sim->dev.first + sim->dev.n);
    return SWIM_EINVAL;
  }
  return SWIM_OK;
}

// one view row <-> swim_member_t[]
int fetch_row(swim_sim *sim, uint32_t node, std::vector<swim_member_t> &out) {
  const SimDev &d = sim->dev;
  const size_t base = (size_t)(node - d.first) * d.cap;
  std::vector<uint32_t> nb(d.cap), inc(d.cap), last(d.cap);
  std::vector<uint8_t> st(d.cap);
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(nb.data(), d.nbr + base, d.cap * 4, cudaMemcpyDeviceToHost));
  CUDA_TRY(sim, cudaMemcpy(st.data(), d.vst + base, d.cap, cudaMemcpyDeviceToHost));
  CUDA_TRY(sim, cudaMemcpy(inc.data(), d.vinc + base, d.cap * 4, cudaMemcpyDeviceToHost));
  CUDA_TRY(sim, cudaMemcpy(last.data(), d.vlast + base, d.cap * 4, cudaMemcpyDeviceToHost));
  out.clear();
  for (uint32_t s = 0; s < d.cap; ++s) {
    if ((st[s] & 3u) == SWIM_VACANT) continue;
    swim_member_t m;
    memset(&m, 0, sizeof m);
    m.id = nb[s]; m.addr = nb[s]; m.port = (uint16_t)sim->cfg.base_port;
    m.liveness = st[s] & 3u; m.timer = (st[s] >> 2) & sim->dev.tmask; m.incarnation = inc[s]; m.last_change = last[s];
    out.push_back(m);
  }
  return SWIM_OK;
}

bool member_eq(const swim_member_t &a, const swim_member_t &b) {
  // derived structural Eq over every field (Types.hs:68), not the name-only Ord (Types.hs:72-73)
  return a.id == b.id && a.addr == b.addr && a.port == b.port && a.liveness == b.liveness && a.timer == b.timer &&
         a.incarnation == b.incarnation && a.last_change == b.last_change;
}

void msg_of_rec(const swim_sim *sim, uint4 r, swim_message_t *m) {
  memset(m, 0, sizeof *m);
  m->kind = (uint8_t)(r.w & 0xFF);
  m->node = r.x;
  m->incarnation = r.y;
  if (m->kind == SWIM_MSG_DEAD) m->dead_from = r.z;
  if (m->kind == SWIM_MSG_ALIVE) { m->target = r.x; m->port = (uint16_t)sim->cfg.base_port; }
}

int apply_message(swim_sim *sim, uint32_t node, uint8_t want, const swim_message_t *msg, swim_message_t *out, int *has_out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!msg || !out || !has_out) return SWIM_EINVAL;
  if (msg->kind != want) { // reference: `suspectNode _ _ = undefined` (Core.hs:191,195,218)
    set_error(sim, "message constructor %u does not match the call (expected %u)", msg->kind, want);
    return SWIM_EINVAL;
  }
  if (msg->incarnation < 0 || msg->incarnation > 0xFFFFFFFFll) { set_error(sim, "incarnation does not fit u32"); return SWIM_ERANGE; }
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_APPLY; a.node = node; a.allow_insert = 1;
  a.rec = make_uint4(msg->node, (uint32_t)msg->incarnation, msg->kind == SWIM_MSG_DEAD ? msg->dead_from : 0u, msg->kind);
  rc = run_scalar(sim, a);
  if (rc) { if (rc == SWIM_ECAP) set_error(sim, "view row of node %u is full", node); return rc; }
  *has_out = a.verdict != 0;
  if (a.verdict == 3) { sim->edges_dirty = true; sim->view_set = true; sim->tdead_dirty = true; }
  if (a.verdict) {
    if ((a.rb.w & 0xFF) == msg->kind && a.rb.x == msg->node) *out = *msg; // `Just msg`: the identical message
    else msg_of_rec(sim, a.rb, out);                                       // the Alive refutation (Core.hs:162-166)
  }
  return SWIM_OK;
}

} // namespace

// members (Core.hs:76-77)
extern "C" int swim_get_members(swim_sim_t *sim, uint32_t node, swim_member_t *out, size_t cap, size_t *n_out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!out || !n_out) return SWIM_EINVAL;
  std::vector<swim_member_t> row;
  if ((rc = fetch_row(sim, node, row))) return rc;
  if (row.size() > cap) return SWIM_ECAP;
  std::copy(row.begin(), row.end(), out);
  *n_out = row.size();
  return SWIM_OK;
}

// `swapTVar storeMembers` (Spec.hs:101)
extern "C" int swim_set_members(swim_sim_t *sim, uint32_t node, const swim_member_t *ms, size_t n) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  const SimDev &d = sim->dev;
  if (n > d.cap) { set_error(sim, "swim_set_members: %zu members exceed view_cap %u", n, d.cap); return SWIM_ECAP; }
  if (!ms && n) return SWIM_EINVAL;
  std::vector<swim_member_t> v(ms, ms + n);
  std::sort(v.begin(), v.end(), [](const swim_member_t &a, const swim_member_t &b) { return a.id < b.id; }); // Map.fromList
  for (size_t x = 0; x < n; ++x)
    if (v[x].id >= d.N || v[x].id == node || v[x].liveness > SWIM_DEAD || v[x].timer > d.tmask ||
        (x && v[x].id == v[x - 1].id)) {
      set_error(sim, "swim_set_members: member %zu (id %u) is invalid (range, self, liveness, duplicate)", x, v[x].id);
      return SWIM_EINVAL;
    }
  std::vector<uint32_t> nb(d.cap, SWIM_NO_MEMBER), inc(d.cap, 0), last(d.cap, 0);
  std::vector<uint8_t> st(d.cap, SWIM_VACANT);
  for (size_t x = 0; x < n; ++x) {
    // the countdown only exists while Suspect; a Suspect member given without one is armed with S
    const uint32_t timer = v[x].liveness != SWIM_SUSPECT ? 0u : v[x].timer ? v[x].timer : d.S_arm;
    nb[x] = v[x].id; st[x] = (uint8_t)(v[x].liveness | (timer << 2)); inc[x] = v[x].incarnation;
    last[x] = (uint32_t)v[x].last_change;
  }
  const size_t base = (size_t)(node - d.first) * d.cap;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(d.nbr + base, nb.data(), d.cap * 4, cudaMemcpyHostToDevice));
  CUDA_TRY(sim, cudaMemcpy(d.vst + base, st.data(), d.cap, cudaMemcpyHostToDevice));
  CUDA_TRY(sim, cudaMemcpy(d.vinc + base, inc.data(), d.cap * 4, cudaMemcpyHostToDevice));
  CUDA_TRY(sim, cudaMemcpy(d.vlast + base, last.data(), d.cap * 4, cudaMemcpyHostToDevice));
  sim->edges_dirty = true;
  sim->tdead_dirty = true;
  sim->view_set = true;
  return SWIM_OK;
}

// kRandomMembers (Core.hs:69-74)
extern "C" int swim_k_random_members(swim_sim_t *sim, uint32_t node, uint32_t n, const swim_member_t *ex, size_t n_ex,
                                     swim_member_t *out, size_t cap, size_t *n_out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!out || !n_out || (!ex && n_ex)) return SWIM_EINVAL;
  std::vector<swim_member_t> row;
  if ((rc = fetch_row(sim, node, row))) return rc;
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_KRANDOM; a.node = node; a.n = n; a.call = (uint32_t)sim->scalar_calls++;
  for (size_t s = 0; s < row.size(); ++s) // rows are compact: member s sits in slot s
    for (size_t e = 0; e < n_ex; ++e)
      if (member_eq(row[s], ex[e])) a.excl[s >> 5] |= 1u << (s & 31); // `notElem m excludes`
  if ((rc = run_scalar(sim, a))) return rc;
  if (a.n_out > cap) return SWIM_ECAP;
  for (uint32_t x = 0; x < a.n_out; ++x) out[x] = row[a.slots[x]];
  *n_out = a.n_out;
  return SWIM_OK;
}

// removeDeadNodes (Core.hs:65-67)
extern "C" int swim_remove_dead_nodes(swim_sim_t *sim, uint32_t node) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_REMOVE_DEAD; a.node = node;
  if ((rc = run_scalar(sim, a))) return rc;
  sim->edges_dirty = true;
  sim->tdead_dirty = true;
  return SWIM_OK;
}

extern "C" int swim_next_seqno(swim_sim_t *sim, uint32_t node, uint32_t *out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!out) return SWIM_EINVAL;
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_NEXT_SEQNO; a.node = node;
  if ((rc = run_scalar(sim, a))) return rc;
  *out = a.value;
  return SWIM_OK;
}

extern "C" int swim_next_incarnation(swim_sim_t *sim, uint32_t node, uint32_t *out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!out) return SWIM_EINVAL;
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_NEXT_INC; a.node = node;
  if ((rc = run_scalar(sim, a))) return rc;
  *out = a.value;
  return SWIM_OK;
}

extern "C" int swim_suspect_node(swim_sim_t *sim, uint32_t node, const swim_message_t *msg, swim_message_t *out, int *has_out) {
  return apply_message(sim, node, SWIM_MSG_SUSPECT, msg, out, has_out);
}
extern "C" int swim_dead_node(swim_sim_t *sim, uint32_t node, const swim_message_t *msg, swim_message_t *out, int *has_out) {
  return apply_message(sim, node, SWIM_MSG_DEAD, msg, out, has_out);
}
extern "C" int swim_alive_node(swim_sim_t *sim, uint32_t node, const swim_message_t *msg, swim_message_t *out, int *has_out) {
  return apply_message(sim, node, SWIM_MSG_ALIVE, msg, out, has_out);
}

// disseminate, Broadcast branch (Core.hs:131,136-138)
extern "C" int swim_broadcast(swim_sim_t *sim, uint32_t node, const swim_message_t *msg) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!msg) return SWIM_EINVAL;
  if (msg->kind != SWIM_MSG_SUSPECT && msg->kind != SWIM_MSG_ALIVE && msg->kind != SWIM_MSG_DEAD) {
    set_error(sim, "swim_broadcast: Ping / IndirectPing / Ack are sent directly, never enqueued (Core.hs:124-126)");
    return SWIM_EINVAL;
  }
  if (msg->incarnation < 0 || msg->incarnation > 0xFFFFFFFFll) { set_error(sim, "incarnation does not fit u32"); return SWIM_ERANGE; }
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_ENQUEUE; a.node = node;
  a.rec = make_uint4(msg->node, (uint32_t)msg->incarnation, msg->kind == SWIM_MSG_DEAD ? msg->dead_from : 0u, msg->kind);
  return run_scalar(sim, a);
}

extern "C" int swim_get_broadcasts(swim_sim_t *sim, uint32_t node, swim_message_t *out, size_t cap, size_t *n_out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!out || !n_out) return SWIM_EINVAL;
  const SimDev &d = sim->dev;
  const uint32_t l = node - d.first;
  uint8_t cnt = 0;
  std::vector<uint4> recs(d.B);
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(&cnt, d.pb_cnt + l, 1, cudaMemcpyDeviceToHost));
  CUDA_TRY(sim, cudaMemcpy(recs.data(), d.pb + (size_t)l * d.B, d.B * sizeof(uint4), cudaMemcpyDeviceToHost));
  if (cnt > cap) return SWIM_ECAP;
  for (uint32_t q = 0; q < cnt; ++q) msg_of_rec(sim, recs[q], &out[q]);
  *n_out = cnt;
  return SWIM_OK;
}

extern "C" int swim_tick_timers(swim_sim_t *sim, uint32_t node, uint32_t *n_expired) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_TICK_TIMERS; a.node = node;
  rc = run_scalar(sim, a);
  if (rc) return rc;
  if (n_expired) *n_expired = a.value;
  return SWIM_OK;
}

extern "C" int swim_take_broadcasts(swim_sim_t *sim, uint32_t node, swim_message_t *out, size_t cap, size_t *n_out) {
  int rc = swim_get_broadcasts(sim, node, out, cap, n_out);
  if (rc) return rc;
  ScalarArgs a;
  memset(&a, 0, sizeof a);
  a.op = OP_SPEND; a.node = node;
  return run_scalar(sim, a);
}

// `process` (Core.hs:89-117)
extern "C" int swim_handle_message(swim_sim_t *sim, uint32_t node, uint32_t sender_addr, uint16_t sender_port,
                                   const swim_message_t *msg, swim_gossip_t *out, size_t cap, size_t *n_out) {
  int rc = check_node(sim, node);
  if (rc) return rc;
  if (!msg || !out || !n_out || cap < 1) return SWIM_EINVAL;
  *n_out = 0;
  memset(out, 0, sizeof *out);
  switch (msg->kind) {
    case SWIM_MSG_ACK: // invokeAckHandler; emits nothing (Core.hs:92-94)
      return SWIM_OK;
    case SWIM_MSG_PING:
      if (msg->node != node) return SWIM_OK; // not for us: ignore (Core.hs:100-101)
      out->is_direct = 1; out->dest_addr = sender_addr; out->dest_port = sender_port;
      out->msg.kind = SWIM_MSG_ACK; out->msg.seq_no = msg->seq_no; out->msg.payload_len = 0; // Core.hs:99
      *n_out = 1;
      return SWIM_OK;
    case SWIM_MSG_INDIRECT_PING: { // [Q4] seq := nextIncarnation (Core.hs:105-108; pinned by Spec.hs:166-174)
      uint32_t next = 0;
      if ((rc = swim_next_incarnation(sim, node, &next))) return rc;
      out->is_direct = 1; out->dest_addr = msg->target; out->dest_port = msg->port;
      out->msg.kind = SWIM_MSG_PING; out->msg.seq_no = next; out->msg.node = msg->node;
      *n_out = 1;
      return SWIM_OK;
    }
    case SWIM_MSG_SUSPECT: case SWIM_MSG_DEAD: case SWIM_MSG_ALIVE: {
      int has = 0;
      if ((rc = apply_message(sim, node, msg->kind, msg, &out->msg, &has))) return rc;
      if (has) { out->is_direct = 0; *n_out = 1; } // maybeBroadcast (Core.hs:119-121)
      return SWIM_OK;
    }
  }
  set_error(sim, "swim_handle_message: unknown message kind %u", msg->kind);
  return SWIM_EINVAL;
}
