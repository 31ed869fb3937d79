// swim_join.cuh — seed joins between steps (DESIGN.md §2.7), on the device. Compiled as part of swim_sim.cu's
// translation unit, after swim_pushpull.cuh (whose merge, scan and call skeleton it uses).
//
// memberlist's Join(joinHosts): each pair (joiner j, seed s) is one full-state exchange between j and s, whether or not
// either lists the other. The exchange is push-pull's: both states are read from a snapshot, and each receiver merges
// its senders in ascending id through push_pull_kernel. Only the choice of who talks to whom differs: the pair list
// replaces the Philox partner draw, so the receiver -> sender lists are built from the pairs (both directions of every
// exchange, counted per receiver, sorted by (receiver, sender)). A receiver named by several pairs of the same sender
// gets that sender once: push_pull_kernel skips a repeated sender. With SWIM_JOIN_FRESH the up joiners first lose their
// rows and piggyback buffers, so what they send is Alive(self) alone.
#pragma once

#include "swim_pushpull.cuh"

namespace {

static_assert(sizeof(swim_join_t) == sizeof(uint2), "swim_join_t is uploaded as uint2 {node, seed}");

// SWIM_JOIN_FRESH: one warp per pair. The first warp that claims an up local joiner empties its row (every slot
// vacant, as remove_dead_kernel leaves a freed slot) and its piggyback buffer; later pairs of the same joiner find it
// claimed. *vacated += the occupied slots emptied.
__global__ void __launch_bounds__(kGT) join_reset_kernel(SimDev d, const uint2 *pr, uint32_t np, uint32_t *claim, u64 *vacated) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t gone = 0;
  for (uint32_t k = warp; k < np; k += nwarps) {
    const uint32_t j = pr[k].x, l = j - d.first;
    if (l >= d.n || !d.alive[j]) continue;
    uint32_t won = 0;
    if (lane == 0) won = atomicExch(&claim[l], 1u) == 0u;
    if (!__shfl_sync(kFull, won, 0)) continue;
    for (uint32_t s = lane; s < d.cap; s += 32) {
      const size_t x = (size_t)l * d.cap + s;
      gone += (d.vst[x] & 3u) != SWIM_VACANT;
      d.nbr[x] = SWIM_NO_MEMBER; d.vst[x] = SWIM_VACANT; d.vinc[x] = 0; d.vlast[x] = 0;
    }
    if (lane == 0) d.pb_cnt[l] = 0;
  }
  gone = __reduce_add_sync(kFull, gone);
  if (lane == 0 && gone) atomicAdd(vacated, (u64)gone);
}

// One thread per pair k = (j, s). Both up: an exchange, with direction 2k (s's state to j) and 2k + 1 (j's state to s).
// A direction whose receiver is local is counted at its receiver (cnt) and keyed by its sender (skey, SWIM_NO_MEMBER
// otherwise); rcv[2k + dir] = its receiver. *n_ex += the exchanges whose joiner is local.
__global__ void __launch_bounds__(kGT) join_edges_kernel(SimDev d, const uint2 *pr, uint32_t np, uint32_t *cnt, uint32_t *skey,
                                                         uint32_t *rcv, u64 *n_ex) {
  uint32_t ex = 0;
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x) {
    const uint32_t j = pr[k].x, s = pr[k].y;
    const bool both = d.alive[j] && d.alive[s];
    ex += both && j - d.first < d.n;
#pragma unroll
    for (int dir = 0; dir < 2; ++dir) {
      const uint32_t r = dir ? s : j, from = dir ? j : s;
      const bool mine = both && r - d.first < d.n;
      if (mine) atomicAdd(&cnt[r - d.first], 1u);
      skey[2 * (size_t)k + dir] = mine ? from : SWIM_NO_MEMBER;
      rcv[2 * (size_t)k + dir] = r;
    }
  }
  ex = __reduce_add_sync(kFull, ex);
  if ((threadIdx.x & 31) == 0 && ex) atomicAdd(n_ex, (u64)ex);
}

// out[p] = src[idx[p]]: the values that travel with a radix sort's keys (which hands back positions only)
__global__ void __launch_bounds__(kGT) join_take_kernel(const uint32_t *idx, const uint32_t *src, size_t n, uint32_t *out) {
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < n; p += (size_t)gridDim.x * blockDim.x) out[p] = src[idx[p]];
}

// SWIM_JOIN_FRESH on this shard's joiners. *vacated = the occupied slots emptied.
int join_reset(swim_sim *sim, Scratch &s, const uint2 *pr, uint32_t np, u64 *vacated) {
  const SimDev &d = sim->dev;
  uint32_t *claim;
  u64 *res;
  SCRATCH(s, claim, d.n);
  SCRATCH(s, res, 1);
  GRAPH_TRY(sim, cudaMemsetAsync(claim, 0, (size_t)d.n * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(res, 0, 8, sim->stream));
  SWIM_LAUNCH(join_reset_kernel, row_grid(sim, np), kGT, sim->stream, d, pr, np, claim, res);
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  GRAPH_TRY(sim, cudaMemcpyAsync(vacated, res, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  return SWIM_OK;
}

// The exchanges on this shard's receivers, from the snapshot `gsnap` (sharded: the gathered global one; null: this
// shard's rows, copied here). h = {inserted, dropped on a full row, exchanges whose joiner is local}.
int join_local(swim_sim *sim, Scratch &s, const uint2 *pr, uint32_t np, const PpSnap *gsnap, u64 h[3]) {
  const SimDev &d = sim->dev;
  const size_t n = d.n, nd = 2 * (size_t)np;
  uint32_t *cnt, *part, *skey, *rcv;
  u64 *seg, *res, E = 0;
  SCRATCH(s, cnt, n);
  SCRATCH(s, part, n);
  SCRATCH(s, seg, n + 1);
  SCRATCH(s, res, 3);
  SCRATCH(s, skey, nd);
  SCRATCH(s, rcv, nd);
  GRAPH_TRY(sim, cudaMemsetAsync(cnt, 0, n * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(part, 0xFF, n * 4, sim->stream)); // no partner draw: every sender is in the lists
  GRAPH_TRY(sim, cudaMemsetAsync(res, 0, 3 * 8, sim->stream));
  SWIM_LAUNCH(join_edges_kernel, grid_of(sim, (np + kGT - 1) / kGT), kGT, sim->stream, d, pr, np, cnt, skey, rcv, res + 2);
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  int rc;
  if ((rc = scan_total(sim, s, cnt, n, seg, &E))) return rc;
  if (E) {
    // (receiver, sender) order: a stable sort of the directions by sender, then a stable sort of that by receiver
    const uint32_t *k1, *v1, *k2, *v2;
    uint32_t *key2, *chooser;
    SCRATCH(s, key2, E);
    SCRATCH(s, chooser, E);
    const int g = grid_of(sim, (E + kGT - 1) / kGT);
    if ((rc = sort_by_key(sim, s, skey, nd, 1, E, d.N, &k1, &v1))) return rc;
    SWIM_LAUNCH(join_take_kernel, g, kGT, sim->stream, v1, (const uint32_t *)rcv, (size_t)E, key2);
    ++sim->launches;
    if ((rc = sort_by_key(sim, s, key2, E, 1, E, d.N, &k2, &v2))) return rc;
    SWIM_LAUNCH(join_take_kernel, g, kGT, sim->stream, v2, k1, (size_t)E, chooser);
    ++sim->launches;
    GRAPH_TRY(sim, cudaGetLastError());
    if ((rc = pp_merge(sim, s, gsnap, part, seg, chooser, res))) return rc;
  }
  GRAPH_TRY(sim, cudaMemcpyAsync(h, res, 3 * sizeof(u64), cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  return SWIM_OK;
}

} // namespace

extern "C" int swim_sim_join(swim_sim_t *sim, const swim_join_t *joins, size_t n, uint32_t flags, uint64_t *n_exchanges,
                             uint64_t *n_inserted, uint64_t *n_full) {
  if (!sim || (!joins && n)) return SWIM_EINVAL;
  int rc;
  if ((rc = between_steps_check(sim, "swim_sim_join"))) return rc;
  const SimDev &d = sim->dev;
  if (flags & ~(uint32_t)SWIM_JOIN_FRESH) { set_error(sim, "swim_sim_join: unknown flags 0x%x", flags); return SWIM_EINVAL; }
  if (n > 0x7FFFFFFFull) { set_error(sim, "swim_sim_join: %zu pairs in one call (at most 2^31 - 1)", n); return SWIM_EINVAL; }
  for (size_t x = 0; x < n; ++x)
    if (joins[x].node >= d.N || joins[x].seed >= d.N || joins[x].node == joins[x].seed) {
      set_error(sim, "swim_sim_join: pair %zu (node %u, seed %u) is invalid (id >= N, or node == seed)", x, joins[x].node,
                joins[x].seed);
      return SWIM_EINVAL;
    }
  u64 h[3] = {0, 0, 0}, vacated = 0;
  if (n) {
    const uint32_t np = (uint32_t)n;
    uint2 *pr = nullptr;
    rc = between_steps(
        sim,
        [&](Scratch &s, const PpSnap *gsnap, u64 *edited) { // members inserted or removed
          const int rc = join_local(sim, s, pr, np, gsnap, h);
          *edited = h[0] + vacated;
          return rc;
        },
        [&](Scratch &s) -> int { // the upload, and SWIM_JOIN_FRESH's resets
          SCRATCH(s, pr, np);
          GRAPH_TRY(sim, cudaMemcpyAsync(pr, joins, (size_t)np * sizeof(uint2), cudaMemcpyHostToDevice, sim->stream));
          return flags & SWIM_JOIN_FRESH ? join_reset(sim, s, pr, np, &vacated) : SWIM_OK;
        });
    if (rc) return rc;
  }
  if (n_exchanges) *n_exchanges = h[2];
  if (n_inserted) *n_inserted = h[0];
  if (n_full) *n_full = h[1];
  return SWIM_OK;
}
