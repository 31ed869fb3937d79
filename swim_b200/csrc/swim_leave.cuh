// swim_leave.cuh — graceful leaves between steps (DESIGN.md §2.8), on the device. Compiled as part of swim_sim.cu's
// translation unit, after swim_join.cuh (whose scratch, scan and sort helpers and call skeleton it uses).
//
// memberlist's Leave: the departing process broadcasts Dead about itself (From = itself) and waits for the gossip to
// spread before it stops. Here the wait is condensed into the call: every leaver goes down as a CRASH at the current
// round does, and each member of its row that it holds Alive or Suspect and that is up receives Dead(self_inc, L, from L)
// as one injected datagram. The merge is event_kernel's SWIM_EV_INJECT path itself, fed with a list built here: one
// event per (recipient, leaver), grouped by recipient with its leavers in ascending id (a stable sort by recipient of
// directions produced in leaver order). No membership changes, so the mail graph is kept.
#pragma once

#include "swim_join.cuh"

namespace {

// One thread per listed id: mark[id] = 1 when the process is up (a repeated id marks the same word).
__global__ void __launch_bounds__(kGT) leave_mark_kernel(SimDev d, const uint32_t *ids, uint32_t np, uint32_t *mark) {
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x)
    if (d.alive[ids[k]]) mark[ids[k]] = 1u;
}

// One thread per node: the marked nodes, ascending, into lv[pos[i]]; each goes down as a CRASH at `round` does
// (alive, last_crash) and is never brought back by the seeded churn (back_at = 0). *n_local += the leavers this shard
// owns. The crashed-member bitmaps are re-derived before the next round (tdead_dirty), not marked here.
__global__ void __launch_bounds__(kGT) leave_depart_kernel(SimDev d, uint32_t round, const uint32_t *mark, const u64 *pos,
                                                           uint32_t *lv, u64 *n_local) {
  uint32_t mine = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < d.N; i += gridDim.x * blockDim.x) {
    if (!mark[i]) continue;
    lv[pos[i]] = i;
    d.alive[i] = 0;
    d.last_crash[i] = round;
    d.back_at[i] = 0;
    mine += i - d.first < d.n;
  }
  mine = __reduce_add_sync(kFull, mine);
  if ((threadIdx.x & 31) == 0 && mine) atomicAdd(n_local, (u64)mine);
}

// One warp per leaver k (global id lv[k], its row in nbr / vst by global id): a member m of the row whose slot is Alive
// or Suspect, that is up (after every departure) and local, is one direction k -> m, counted at m (cnt) and keyed by m
// at position k * cap + slot (SWIM_NO_MEMBER otherwise), so a sort by key keeps each recipient's leavers ascending.
__global__ void __launch_bounds__(kGT) leave_edges_kernel(SimDev d, const uint32_t *lv, uint32_t nl, const uint32_t *nbr,
                                                          const uint8_t *vst, uint32_t *cnt, uint32_t *key) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t k = warp; k < nl; k += nwarps) {
    const size_t row = (size_t)lv[k] * d.cap;
    for (uint32_t s = lane; s < d.cap; s += 32) {
      const uint32_t m = nbr[row + s], live = vst[row + s] & 3u;
      const bool to = (live == SWIM_ALIVE || live == SWIM_SUSPECT) && d.alive[m] && m - d.first < d.n;
      if (to) atomicAdd(&cnt[m - d.first], 1u);
      key[(size_t)k * d.cap + s] = to ? m : SWIM_NO_MEMBER;
    }
  }
}

// Event p of the sorted directions: recipient rcv[p] receives Dead(self_inc, L, from L) of leaver L = lv[who[p]], as a
// SWIM_EV_INJECT datagram.
__global__ void __launch_bounds__(kGT) leave_events_kernel(const uint32_t *rcv, const uint32_t *who, size_t E, const uint32_t *lv,
                                                           const uint32_t *self_inc, DevEvent *ev) {
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < E; p += (size_t)gridDim.x * blockDim.x) {
    const uint32_t L = lv[who[p]];
    ev[p].node = rcv[p];
    ev[p].kind = SWIM_EV_INJECT;
    ev[p].rec = make_rec(L, self_inc[L], L, SWIM_MSG_DEAD);
  }
}

// event_kernel<W> on `n_ev` events at the current round (a plain launch: between steps nothing is chained).
int leave_inject(swim_sim *sim, const DevEvent *ev, uint32_t n_ev) {
  SimDev d = sim->dev;
  d.round = sim->round;
  const int g = (int)std::min<size_t>((n_ev + kWarpsPerBlock - 1) / kWarpsPerBlock, (size_t)sim->sm_count * 4);
  switch (d.cap / 32) {
    case 1: SWIM_LAUNCH(event_kernel<1>, g, kThreads, sim->stream, d, ev, n_ev, (const uint32_t *)nullptr); break;
    case 2: SWIM_LAUNCH(event_kernel<2>, g, kThreads, sim->stream, d, ev, n_ev, (const uint32_t *)nullptr); break;
    case 4: SWIM_LAUNCH(event_kernel<4>, g, kThreads, sim->stream, d, ev, n_ev, (const uint32_t *)nullptr); break;
    default: SWIM_LAUNCH(event_kernel<8>, g, kThreads, sim->stream, d, ev, n_ev, (const uint32_t *)nullptr); break;
  }
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

// The whole call on one rank, from the uploaded ids. `gsnap` (sharded): the gathered global snapshot, from which the
// leavers' rows and incarnations are read by global id; null: this shard's own rows (a single shard holds every row, and a
// leaver's row does not change during the merge: only up recipients are written). h = {leavers owned here, records
// delivered to this shard's recipients}.
int leave_local(swim_sim *sim, Scratch &s, const uint32_t *ids, uint32_t np, const PpSnap *gsnap, u64 h[2]) {
  const SimDev &d = sim->dev;
  const size_t n = d.n, N = d.N;
  uint32_t *mark, *cnt;
  u64 *pos, *seg, *res, nl = 0, E = 0;
  SCRATCH(s, mark, N);
  SCRATCH(s, pos, N + 1);
  SCRATCH(s, cnt, n);
  SCRATCH(s, seg, n + 1);
  SCRATCH(s, res, 1);
  GRAPH_TRY(sim, cudaMemsetAsync(mark, 0, N * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(cnt, 0, n * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(res, 0, 8, sim->stream));
  SWIM_LAUNCH(leave_mark_kernel, grid_of(sim, (np + kGT - 1) / kGT), kGT, sim->stream, d, ids, np, mark);
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  int rc;
  if ((rc = scan_total(sim, s, mark, N, pos, &nl))) return rc;
  if (nl) {
    uint32_t *lv, *key;
    SCRATCH(s, lv, nl);
    SCRATCH(s, key, nl * d.cap);
    SWIM_LAUNCH(leave_depart_kernel, grid_of(sim, (N + kGT - 1) / kGT), kGT, sim->stream, d, sim->round, (const uint32_t *)mark,
                (const u64 *)pos, lv, res);
    SWIM_LAUNCH(leave_edges_kernel, row_grid(sim, nl), kGT, sim->stream, d, (const uint32_t *)lv, (uint32_t)nl,
                gsnap ? gsnap->nbr : (const uint32_t *)d.nbr, gsnap ? gsnap->vst : (const uint8_t *)d.vst, cnt, key);
    sim->launches += 2;
    GRAPH_TRY(sim, cudaGetLastError());
    if ((rc = scan_total(sim, s, cnt, n, seg, &E))) return rc;
    if (E) {
      const uint32_t *rcv, *who;
      DevEvent *ev;
      if ((rc = sort_by_key(sim, s, key, nl * d.cap, d.cap, E, d.N, &rcv, &who))) return rc;
      SCRATCH(s, ev, E);
      SWIM_LAUNCH(leave_events_kernel, grid_of(sim, (E + kGT - 1) / kGT), kGT, sim->stream, rcv, who, (size_t)E,
                  (const uint32_t *)lv, gsnap ? gsnap->self_inc : (const uint32_t *)d.self_inc, ev);
      ++sim->launches;
      GRAPH_TRY(sim, cudaGetLastError());
      // (event_kernel counts in 32 bits; a recipient's run may span two launches, which run in stream order)
      for (u64 p = 0; p < E; p += 0x40000000ull)
        if ((rc = leave_inject(sim, ev + p, (uint32_t)std::min<u64>(E - p, 0x40000000ull)))) return rc;
    }
  }
  GRAPH_TRY(sim, cudaMemcpyAsync(h, res, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  h[1] = E;
  return SWIM_OK;
}

} // namespace

extern "C" int swim_sim_leave(swim_sim_t *sim, const uint32_t *nodes, size_t n, uint64_t *n_left, uint64_t *n_delivered) {
  if (!sim || (!nodes && n)) return SWIM_EINVAL;
  int rc;
  if ((rc = between_steps_check(sim, "swim_sim_leave"))) return rc;
  const SimDev &d = sim->dev;
  if (n > 0x7FFFFFFFull) { set_error(sim, "swim_sim_leave: %zu ids in one call (at most 2^31 - 1)", n); return SWIM_EINVAL; }
  for (size_t x = 0; x < n; ++x)
    if (nodes[x] >= d.N) { set_error(sim, "swim_sim_leave: id %zu (%u) >= N = %u", x, nodes[x], d.N); return SWIM_EINVAL; }
  u64 h[2] = {0, 0};
  if (n) { // no membership changes (edited stays 0): alive[] and rows changed, so only the per-node state is re-derived
    const uint32_t np = (uint32_t)n;
    rc = between_steps(sim, [&](Scratch &s, const PpSnap *gsnap, u64 *) -> int {
      uint32_t *ids;
      SCRATCH(s, ids, np);
      GRAPH_TRY(sim, cudaMemcpyAsync(ids, nodes, (size_t)np * 4, cudaMemcpyHostToDevice, sim->stream));
      return leave_local(sim, s, ids, np, gsnap, h);
    });
    if (rc) return rc;
  }
  if (n_left) *n_left = h[0];
  if (n_delivered) *n_delivered = h[1];
  return SWIM_OK;
}
