// swim_pushpull.cuh — the push-pull state exchange between steps (DESIGN.md §2.6), on the device.
// Compiled as part of swim_sim.cu's translation unit, after swim_graph.cuh (whose scan, sort, scratch and row-insert
// helpers it uses).
//
// memberlist's periodic anti-entropy: every up node picks one random Alive member of its view, and if that partner is up
// the two swap their full member state. Each side merges what it receives through the receive path's state machine
// (row_apply), and a merge inserts the Alive members it did not list — the only way a bulk run learns unknown members.
// Everything that is sent is read from a snapshot taken before any row changes, so the result does not depend on the
// order in which warps run. On a sharded handle the call is a collective: the snapshot is every rank's rows gathered
// into global-id order, every rank draws the partners of all N nodes from it (the draws are a function of the snapshot,
// alive[] and the round, so all ranks agree without exchanging them), and each rank merges into its own receivers.
#pragma once

#include <cstddef>
#include <type_traits>

#include "swim_graph.cuh"

namespace {

// One thread per node i of rows [0, rows) of (nbr, vst), which start at global id 0: this shard's own rows on a single
// shard, the gathered global snapshot on several. The partner p_i = the floor(x L / 2^32)-th Alive slot (ascending),
// x = word 0 of Philox block (round, i, P_PUSHPULL, 0); p_i = SWIM_NO_MEMBER unless i and p_i are both up. For the
// local nodes i: part[i - first] = p_i. For the local partners p_i: cnt[p_i - first] counts p_i's choosers, and
// key[i] = p_i (SWIM_NO_MEMBER otherwise; key = null on a single shard, where part is that array).
__global__ void __launch_bounds__(kGT) pp_pick_kernel(SimDev d, uint32_t round, const uint32_t *nbr, const uint8_t *vst,
                                                      uint32_t rows, uint32_t *part, uint32_t *key, uint32_t *cnt, u64 *n_ex) {
  uint32_t ex = 0;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < rows; i += gridDim.x * blockDim.x) {
    uint32_t p = SWIM_NO_MEMBER;
    if (d.alive[i]) {
      const uint8_t *st = vst + (size_t)i * d.cap;
      uint32_t L = 0;
      for (uint32_t s = 0; s < d.cap; ++s) L += (st[s] & 3u) == SWIM_ALIVE;
      if (L) {
        uint32_t k = bounded(philox4x32_10(make_uint4(round, i, P_PUSHPULL, 0), d.key0, d.key1).x, L), s = 0;
        for (;; ++s)
          if ((st[s] & 3u) == SWIM_ALIVE && k-- == 0) break;
        p = nbr[(size_t)i * d.cap + s];
        if (!d.alive[p]) p = SWIM_NO_MEMBER;
      }
    }
    const bool to_me = p != SWIM_NO_MEMBER && p - d.first < d.n;
    if (to_me) atomicAdd(&cnt[p - d.first], 1u);
    if (i - d.first < d.n) {
      part[i - d.first] = p;
      ex += p != SWIM_NO_MEMBER;
    }
    if (key) key[i] = to_me ? p : SWIM_NO_MEMBER;
  }
  ex = __reduce_add_sync(kFull, ex);
  if ((threadIdx.x & 31) == 0 && ex) atomicAdd(n_ex, (u64)ex);
}

// The senders' state as the snapshot holds it, by global id.
struct PpSnap {
  const uint32_t *nbr, *vinc, *self_inc;
  const uint8_t *vst;
};

// One warp per local receiver j (global id first + j): senders {part[j]} ∪ choosers(j) in ascending id, each once; record by record through
// row_apply (net), insertion of unknown Alive members, re-broadcast of every `Just`. res = {inserted, dropped on a full row}.
template <int W>
__global__ void __launch_bounds__(kThreads) push_pull_kernel(SimDev d, uint32_t round, PpSnap snap, const uint32_t *part,
                                                             const u64 *seg, const uint32_t *chooser, u64 *res) {
  SWIM_SHARED_2D(uint4, s_pb, kWarpsPerBlock, 32);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t warp = blockIdx.x * kWarpsPerBlock + wib, nwarps = gridDim.x * kWarpsPerBlock;
  Ctr c; c.clear();
  PbStage pbs; pbs.s = s_pb[wib];
  uint32_t inserted = 0, full = 0;
  for (uint32_t j = warp; j < d.n; j += nwarps) {
    uint32_t pull = part[j];
    u64 x = seg[j];
    const u64 x1 = seg[j + 1];
    if (pull == SWIM_NO_MEMBER && x == x1) continue; // (a crashed node neither chooses nor is chosen)
    Row<W> row;
    row_load<W>(row, d, j, lane);
    pb_load(pbs, d, j, lane);
    uint32_t last[W], td[W], used = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      last[w] = d.vlast[(size_t)j * d.cap + 32 * w + lane];
      td[w] = d.meta[(size_t)j * W + w].z;
      used += __popc(__ballot_sync(kFull, (row.st[w] & 3u) != SWIM_VACANT));
    }
    uint32_t self_inc = d.self_inc[j];
    const uint32_t self_inc0 = self_inc;
    bool grew = false;
    for (uint32_t prev = SWIM_NO_MEMBER;;) {
      const uint32_t ch = x < x1 ? chooser[x] : SWIM_NO_MEMBER;
      uint32_t s;
      if (pull != SWIM_NO_MEMBER && pull <= ch) { s = pull; pull = SWIM_NO_MEMBER; if (ch == s) ++x; }
      else if (ch != SWIM_NO_MEMBER) { s = ch; ++x; }
      else break;
      if (s == prev) continue; // a join's chooser list may repeat a sender (duplicated pairs): it is merged once
      prev = s;
      // the sender's row, lane-owned like the receiver's
      uint32_t snb[W], sst[W], sinc[W];
      int nocc = 0; // occupied slots (vacancies are last)
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const size_t y = (size_t)s * d.cap + 32 * w + lane;
        snb[w] = snap.nbr[y]; sst[w] = snap.vst[y] & 3u; sinc[w] = snap.vinc[y];
        nocc += __popc(__ballot_sync(kFull, sst[w] != SWIM_VACANT));
      }
      // record -1: Alive(self_inc, s); then one per occupied slot, in slot order
      for (int q = -1; q < nocc; ++q) {
        uint4 rec;
        if (q < 0) {
          rec = make_rec(s, snap.self_inc[s], 0, SWIM_MSG_ALIVE);
        } else {
          uint32_t m = 0, lv = 0, vi = 0;
#pragma unroll
          for (int w = 0; w < W; ++w) {
            const uint32_t a = __shfl_sync(kFull, snb[w], q & 31), b = __shfl_sync(kFull, sst[w], q & 31),
                           e = __shfl_sync(kFull, sinc[w], q & 31);
            if (w == (q >> 5)) { m = a; lv = b; vi = e; }
          }
          rec = make_rec(m, vi, lv == SWIM_DEAD ? s : 0u,
                         lv == SWIM_ALIVE ? SWIM_MSG_ALIVE : lv == SWIM_SUSPECT ? SWIM_MSG_SUSPECT : SWIM_MSG_DEAD);
        }
        uint4 rb;
        const int v = row_apply<W>(row, d, d.first + j, self_inc, rec, rb, lane, c.v[SWIM_CTR_REFUTES]);
        if (v == 2) { // an Alive member j does not list: addNewMember (Core.hs:206-216), as swim_alive_node inserts
          if (used == d.cap) { ++full; continue; }
          uint32_t pos = 0;
#pragma unroll
          for (int w = 0; w < W; ++w) {
            pos += __popc(__ballot_sync(kFull, (row.st[w] & 3u) != SWIM_VACANT && row.nb[w] < rec.x));
            if (row.touched >> w & 1u) last[w] = round; // slots change places: lastChange moves with them
          }
          row.touched = 0;
          insert_slot<W>(row.nb, row.st, row.inc, last, pos, rec.x, rec.y, round, lane);
          ++used;
          ++inserted;
          grew = true;
          rb = rec;
        } else if (v != 1) {
          continue;
        }
        pb_enqueue(pbs, d, rb, lane, c.v[SWIM_CTR_PB_DROPPED]);
        if (lane == 0) ++c.v[SWIM_CTR_RECS_APPLIED];
      }
    }
    if (grew) { // slots moved: the whole row is written (the per-node records are re-derived before the next round)
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const size_t y = (size_t)j * d.cap + 32 * w + lane;
        if (row.touched >> w & 1u) last[w] = round;
        d.nbr[y] = row.nb[w]; d.vst[y] = (uint8_t)row.st[w]; d.vinc[y] = row.inc[w]; d.vlast[y] = last[w];
      }
    } else {
      row_store<W>(row, d, j, lane, round, td);
    }
    pb_store(pbs, d, j, lane);
    if (lane == 0 && self_inc != self_inc0) d.self_inc[j] = self_inc;
  }
  if (lane == 0 && (inserted || full)) { atomicAdd(&res[0], (u64)inserted); atomicAdd(&res[1], (u64)full); }
  c.flush(d.ctr, lane);
}

} // namespace

namespace {
// A snapshot of `rows` rows by global id and their incarnations, in scratch: on a single shard (`copy`) copies of its
// rows taken on the stream before any row changes, sharded the buffers that every rank's rows are gathered into.
int pp_snapshot(swim_sim *sim, Scratch &s, size_t rows, bool copy, PpSnap *snap) {
  const SimDev &d = sim->dev;
  const size_t slots = rows * d.cap;
  uint32_t *nb, *vi, *si;
  uint8_t *vs;
  SCRATCH(s, nb, slots);
  SCRATCH(s, vi, slots);
  SCRATCH(s, si, rows);
  SCRATCH(s, vs, slots);
  if (copy) {
    GRAPH_TRY(sim, cudaMemcpyAsync(nb, d.nbr, slots * 4, cudaMemcpyDeviceToDevice, sim->stream));
    GRAPH_TRY(sim, cudaMemcpyAsync(vi, d.vinc, slots * 4, cudaMemcpyDeviceToDevice, sim->stream));
    GRAPH_TRY(sim, cudaMemcpyAsync(si, d.self_inc, rows * 4, cudaMemcpyDeviceToDevice, sim->stream));
    GRAPH_TRY(sim, cudaMemcpyAsync(vs, d.vst, slots, cudaMemcpyDeviceToDevice, sim->stream));
  }
  snap->nbr = nb; snap->vinc = vi; snap->self_inc = si; snap->vst = vs;
  return SWIM_OK;
}

// push_pull_kernel at the handle's row width: every local receiver j merges {part[j]} and chooser[seg[j] .. seg[j + 1]),
// from `gsnap` (sharded: the gathered global snapshot) or, on a single shard, from a snapshot of its rows taken here.
int pp_merge(swim_sim *sim, Scratch &s, const PpSnap *gsnap, const uint32_t *part, const u64 *seg, const uint32_t *chooser,
             u64 *res) {
  const SimDev &d = sim->dev;
  PpSnap snap;
  int rc;
  if (gsnap) snap = *gsnap;
  else if ((rc = pp_snapshot(sim, s, d.n, true, &snap))) return rc;
  const int g = grid_of(sim, (d.n + kWarpsPerBlock - 1) / kWarpsPerBlock);
  switch (d.cap / 32) {
    case 1: SWIM_LAUNCH(push_pull_kernel<1>, g, kThreads, sim->stream, d, sim->round, snap, part, seg, chooser, res); break;
    case 2: SWIM_LAUNCH(push_pull_kernel<2>, g, kThreads, sim->stream, d, sim->round, snap, part, seg, chooser, res); break;
    case 4: SWIM_LAUNCH(push_pull_kernel<4>, g, kThreads, sim->stream, d, sim->round, snap, part, seg, chooser, res); break;
    default: SWIM_LAUNCH(push_pull_kernel<8>, g, kThreads, sim->stream, d, sim->round, snap, part, seg, chooser, res); break;
  }
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

// Counts to positions: out[0..n] = the exclusive scan of in[0..n), and *total = out[n] on the host (the stream is
// synchronised, so device-to-host copies queued before this call have landed too).
int scan_total(swim_sim *sim, Scratch &s, const uint32_t *in, size_t n, u64 *out, u64 *total) {
  int rc;
  if ((rc = scan_u32(sim, s, in, n, out))) return rc;
  GRAPH_TRY(sim, cudaMemcpyAsync(total, out + n, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  return SWIM_OK;
}

// The exchange on this shard's receivers. Sharded: `gsnap` is the gathered global snapshot. h = {inserted, dropped on a
// full row, exchanges} of this shard.
int push_pull_local(swim_sim *sim, Scratch &s, const PpSnap *gsnap, u64 h[3]) {
  const SimDev &d = sim->dev;
  const size_t n = d.n;
  const uint32_t rows = gsnap ? d.N : d.n; // the rows the partners are drawn from
  uint32_t *part, *cnt, *key = nullptr;
  u64 *seg, *res, E = 0, ex = 0;
  SCRATCH(s, part, n);
  SCRATCH(s, cnt, n);
  SCRATCH(s, seg, n + 1);
  SCRATCH(s, res, 3);
  if (gsnap) SCRATCH(s, key, rows);
  GRAPH_TRY(sim, cudaMemsetAsync(cnt, 0, n * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(res, 0, 3 * 8, sim->stream));
  const uint32_t *pn = gsnap ? gsnap->nbr : d.nbr;
  const uint8_t *pv = gsnap ? gsnap->vst : d.vst;
  SWIM_LAUNCH(pp_pick_kernel, grid_of(sim, (rows + kGT - 1) / kGT), kGT, sim->stream, d, sim->round, pn, pv, rows, part, key,
              cnt, res + 2);
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  GRAPH_TRY(sim, cudaMemcpyAsync(&ex, res + 2, 8, cudaMemcpyDeviceToHost, sim->stream));
  int rc;
  if ((rc = scan_total(sim, s, cnt, n, seg, &E))) return rc;
  if (E || ex) { // (sharded, a shard's nodes may pull from partners elsewhere while none of its own is chosen)
    // the choosers of every local node, ascending: a stable sort of the partner array by partner
    const uint32_t *skey, *chooser = nullptr;
    if (E && (rc = sort_by_key(sim, s, key ? key : part, rows, 1, E, d.N, &skey, &chooser))) return rc;
    if ((rc = pp_merge(sim, s, gsnap, part, seg, chooser, res))) return rc;
  }
  GRAPH_TRY(sim, cudaMemcpyAsync(h, res, 3 * sizeof(u64), cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  return SWIM_OK;
}

// The entry check of the collective calls between steps (push-pull, joins, leaves), in this order: a sharded handle
// must be connected to its peers, a view installed, and no earlier step failed part-way.
int between_steps_check(swim_sim *sim, const char *api) {
  if (sim->dev.world != 1 && !sim->connected) {
    set_error(sim, "%s: world > 1 needs swim_sim_ipc_connect or swim_sim_connect (every rank makes the call)", api);
    return SWIM_ESTATE;
  }
  if (!sim->view_set) { set_error(sim, "%s: no view installed", api); return SWIM_ESTATE; }
  if (sim->failed) { set_error(sim, "%s: an earlier step failed part-way; the handle's device state is undefined", api); return SWIM_ESTATE; }
  return SWIM_OK;
}

// The body of a call between steps on one rank: `pre(s)` (optional), then `local(s, gsnap, &edited)` on this shard's
// nodes, with gsnap = null on a single shard (the call reads this shard's rows). Sharded, a collective: barrier (every
// rank's earlier calls are done); `pre` and a barrier (every rank's is done before anyone copies a row); the gather of
// the global snapshot into gsnap; barrier (nobody changes a row or alive[] before every rank has its copy); `local`; and
// a last barrier that sums `edited`, so that every rank marks the view changed, and rebuilds at the next step, exactly
// when some rank changed a membership. The scratch is freed before that barrier: a peer that shares this device may
// start its round kernels right after it, and cudaFree would wait for them while they wait for this rank.
template <typename Local, typename Pre>
int between_steps_body(swim_sim *sim, Local &local, Pre &pre, u64 *edited) {
  const SimDev &d = sim->dev;
  const bool sharded = d.world > 1;
  int rc;
  {
    Scratch s(sim);
    PpSnap snap;
    if (sharded && ((rc = pp_snapshot(sim, s, (size_t)d.world * d.per, false, &snap)) || (rc = coll_barrier(sim)))) return rc;
    if constexpr (!std::is_same<Pre, std::nullptr_t>::value)
      if ((rc = pre(s)) || (sharded && (rc = coll_barrier(sim)))) return rc;
    if (sharded && ((rc = coll_gather(sim, kCollNbr, (void *)snap.nbr)) || (rc = coll_gather(sim, kCollVst, (void *)snap.vst)) ||
                    (rc = coll_gather(sim, kCollVinc, (void *)snap.vinc)) ||
                    (rc = coll_gather(sim, kCollSelfInc, (void *)snap.self_inc)) || (rc = coll_barrier(sim))))
      return rc;
    if ((rc = local(s, sharded ? &snap : nullptr, edited))) return rc;
  }
  return sharded ? coll_barrier(sim, *edited, edited) : SWIM_OK;
}

// A call between steps, body and ending: after an error a sharded handle is failed (the ranks are no longer in step);
// otherwise the mail graph is rebuilt by the next step if memberships changed, and in any case the crashed-member
// bitmaps and per-node records are re-derived before the next round.
template <typename Local, typename Pre = std::nullptr_t>
int between_steps(swim_sim *sim, Local local, Pre pre = nullptr) {
  cudaSetDevice(sim->device);
  u64 edited = 0;
  const int rc = between_steps_body(sim, local, pre, &edited);
  if (rc) {
    if (sim->dev.world != 1) sim->failed = true;
    return rc;
  }
  if (edited) mark_edited(sim);
  else sim->tdead_dirty = true;
  return SWIM_OK;
}
} // namespace

extern "C" int swim_sim_push_pull(swim_sim_t *sim, uint64_t *n_exchanges, uint64_t *n_inserted, uint64_t *n_full) {
  if (!sim) return SWIM_EINVAL;
  int rc;
  if ((rc = between_steps_check(sim, "swim_sim_push_pull"))) return rc;
  u64 h[3] = {0, 0, 0};
  rc = between_steps(sim, [&](Scratch &s, const PpSnap *gsnap, u64 *edited) {
    const int rc = push_pull_local(sim, s, gsnap, h);
    *edited = h[0];
    return rc;
  });
  if (rc) return rc;
  if (n_exchanges) *n_exchanges = h[2];
  if (n_inserted) *n_inserted = h[0];
  if (n_full) *n_full = h[1];
  return SWIM_OK;
}
