// swim_graph.cuh — the mail graph of a view, built on the device, and the bulk membership edits that change it.
// Compiled as part of swim_sim.cu's translation unit (included there once).
//
// Everything K1b and K2 use to address mail (the in-edge index in_off / in_src / ridx), the observer lists event_kernel
// uses (obs_off / obs_slot) and the membership filters of all N rows are functions of the global id matrix alone.
// build_graph derives them from a copy of that matrix in device memory: swim_sim_set_view (after one upload),
// swim_sim_set_view_device (the caller's device buffer) and the first step after a membership change (the rows in
// SimDev::nbr, single shard). The edges are taken in (sender, slot) order and sorted by receiver with a stable LSD
// radix sort, so every receiver's senders come out ascending whatever its in-degree.
#pragma once
#include <algorithm>
#include <vector>

#include "swim_host.h"

using namespace swim;

namespace {

#define GRAPH_TRY(sim, call)                                                                      \
  do {                                                                                            \
    cudaError_t e_ = (call);                                                                      \
    if (e_ != cudaSuccess) {                                                                      \
      set_error(sim, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return SWIM_ECUDA;                                                                          \
    }                                                                                             \
  } while (0)

using u64 = unsigned long long;
constexpr int kGT = 256;                 // threads per CTA of the build kernels: one per radix digit
constexpr int kGW = kGT / 32;
constexpr int kItems = 16;               // elements per thread of one scan chunk / radix tile
constexpr uint32_t kTile = kGT * kItems;

// Device scratch of one call: freed when the call returns, on every path.
struct Scratch {
  swim_sim *sim;
  std::vector<void *> p;
  explicit Scratch(swim_sim *s) : sim(s) {}
  ~Scratch() {
    if (!p.empty()) cudaStreamSynchronize(sim->stream);
    for (void *q : p) cudaFree(q);
  }
  template <typename T>
  bool get(T **x, size_t count) {
    void *q = nullptr;
    if (cudaMalloc(&q, (count ? count : 1) * sizeof(T)) != cudaSuccess) return false;
    p.push_back(q);
    *x = (T *)q;
    return true;
  }
};
#define SCRATCH(s, x, count)                                                                                \
  do {                                                                                                      \
    if (!(s).get(&(x), (count))) {                                                                          \
      set_error(sim, "out of device memory for %s (%zu elements)", #x, (size_t)(count));                    \
      return SWIM_ENOMEM;                                                                                   \
    }                                                                                                       \
  } while (0)

// 64-bit atomic min / max of the validation pass (with -DSWIM_EMU, where the runtime is a CPU stub: the GCC builtins)
__device__ __forceinline__ void atomic_min_u64(u64 *p, u64 v) {
#ifdef SWIM_EMU
  u64 old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v < old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
#else
  atomicMin(p, v);
#endif
}
__device__ __forceinline__ void atomic_max_u64(u64 *p, u64 v) {
#ifdef SWIM_EMU
  u64 old = __atomic_load_n(p, __ATOMIC_SEQ_CST);
  while (v > old && !__atomic_compare_exchange_n(p, &old, v, false, __ATOMIC_SEQ_CST, __ATOMIC_SEQ_CST)) {}
#else
  atomicMax(p, v);
#endif
}

int grid_of(const swim_sim *sim, size_t ctas) { return (int)std::max<size_t>(1, std::min<size_t>(ctas, (size_t)sim->sm_count * 8)); }

// ------------------------------------------------------------------ scan
// Exclusive scan of one value per thread over the CTA; *total = the CTA's sum.
__device__ u64 cta_scan(u64 v, u64 *s_w, u64 *total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  u64 inc = v;
  for (int o = 1; o < 32; o <<= 1) {
    const u64 t = __shfl_sync(kFull, inc, (lane - o) & 31);
    if (lane >= o) inc += t;
  }
  if (lane == 31) s_w[wid] = inc;
  __syncthreads();
  u64 before = 0, all = 0;
  for (int w = 0; w < kGW; ++w) {
    const u64 x = s_w[w];
    if (w < wid) before += x;
    all += x;
  }
  __syncthreads(); // s_w is free for the next scan
  *total = all;
  return before + inc - v;
}

__global__ void __launch_bounds__(kGT) chunk_sum_kernel(const uint32_t *in, size_t n, u64 *part, size_t nchunks) {
  SWIM_SHARED_1D(u64, s_w, kGW);
  for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
    u64 v = 0;
    for (int k = 0; k < kItems; ++k) {
      const size_t i = c * kTile + (size_t)k * kGT + threadIdx.x;
      if (i < n) v += in[i];
    }
    u64 tot;
    cta_scan(v, s_w, &tot);
    if (threadIdx.x == 0) part[c] = tot;
  }
}

// one CTA: the chunk sums become the chunks' first positions; part[nchunks] = the total
__global__ void __launch_bounds__(kGT) part_scan_kernel(u64 *part, size_t nchunks) {
  SWIM_SHARED_1D(u64, s_w, kGW);
  u64 carry = 0;
  for (size_t b = 0; b < nchunks; b += kGT) {
    const size_t i = b + threadIdx.x;
    u64 tot;
    const u64 e = cta_scan(i < nchunks ? part[i] : 0, s_w, &tot);
    if (i < nchunks) part[i] = carry + e;
    carry += tot;
  }
  if (threadIdx.x == 0) part[nchunks] = carry;
}

__global__ void __launch_bounds__(kGT) chunk_scan_kernel(const uint32_t *in, size_t n, const u64 *part, size_t nchunks, u64 *out) {
  SWIM_SHARED_1D(u64, s_w, kGW);
  for (size_t c = blockIdx.x; c < nchunks; c += gridDim.x) {
    u64 carry = part[c];
    for (int k = 0; k < kItems; ++k) {
      const size_t i = c * kTile + (size_t)k * kGT + threadIdx.x;
      u64 tot;
      const u64 e = cta_scan(i < n ? in[i] : 0, s_w, &tot);
      if (i < n) out[i] = carry + e;
      carry += tot;
    }
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) out[n] = part[nchunks];
}

// out[0..n] = exclusive prefix sums of in[0..n), out[n] = the total
int scan_u32(swim_sim *sim, Scratch &s, const uint32_t *in, size_t n, u64 *out) {
  const size_t nc = (n + kTile - 1) / kTile;
  u64 *part;
  SCRATCH(s, part, nc + 1);
  const int g = grid_of(sim, nc);
  SWIM_LAUNCH(chunk_sum_kernel, g, kGT, sim->stream, in, n, part, nc);
  SWIM_LAUNCH(part_scan_kernel, 1, kGT, sim->stream, part, nc);
  SWIM_LAUNCH(chunk_scan_kernel, g, kGT, sim->stream, in, n, (const u64 *)part, nc, out);
  sim->launches += 3;
  GRAPH_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

// ------------------------------------------------------------------ stable radix sort by receiver
// Digit counts of every tile, digit-major (hist[d * T + t]), so that one exclusive scan gives each (digit, tile) its first
// output position. Keys equal to SWIM_NO_MEMBER (vacant slots of the id matrix) are left out.
__global__ void __launch_bounds__(kGT) radix_hist_kernel(const uint32_t *key, size_t n, uint32_t shift, uint32_t *hist, uint32_t T) {
  SWIM_SHARED_1D(uint32_t, s_h, kGT);
  for (uint32_t t = blockIdx.x; t < T; t += gridDim.x) {
    s_h[threadIdx.x] = 0;
    __syncthreads();
    for (int k = 0; k < kItems; ++k) {
      const size_t i = (size_t)t * kTile + (size_t)k * kGT + threadIdx.x;
      if (i >= n) continue;
      const uint32_t x = key[i];
      if (x != SWIM_NO_MEMBER) atomicAdd(&s_h[(x >> shift) & 255u], 1u);
    }
    __syncthreads();
    hist[(size_t)threadIdx.x * T + t] = s_h[threadIdx.x];
    __syncthreads();
  }
}

// One stable pass: the tile's elements are ranked 256 at a time in input order (warp: a ballot per digit bit gives the
// lanes with the same digit; CTA: thread d keeps the running count of digit d over the warps and rounds). vin == null:
// the input is the id matrix itself and an element's value is its row (the sender).
__global__ void __launch_bounds__(kGT) radix_scatter_kernel(const uint32_t *kin, const uint32_t *vin, uint32_t cap, size_t n,
                                                            uint32_t shift, const u64 *off, uint32_t T, uint32_t *kout,
                                                            uint32_t *vout) {
  SWIM_SHARED_2D(uint32_t, s_cnt, kGW, kGT);
  SWIM_SHARED_2D(uint32_t, s_off, kGW, kGT);
  SWIM_SHARED_1D(u64, s_base, kGT);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const unsigned below = (1u << lane) - 1u;
  for (uint32_t t = blockIdx.x; t < T; t += gridDim.x) {
    s_base[threadIdx.x] = off[(size_t)threadIdx.x * T + t];
    for (int w = 0; w < kGW; ++w) s_cnt[w][threadIdx.x] = 0;
    uint32_t run = 0; // elements of digit threadIdx.x placed so far in this tile
    __syncthreads();
    for (int k = 0; k < kItems; ++k) {
      const size_t i = (size_t)t * kTile + (size_t)k * kGT + threadIdx.x;
      const uint32_t key = i < n ? kin[i] : SWIM_NO_MEMBER;
      const bool valid = key != SWIM_NO_MEMBER;
      const uint32_t dg = (key >> shift) & 255u;
      unsigned peers = __ballot_sync(kFull, valid);
      for (int b = 0; b < 8; ++b) {
        const unsigned bb = __ballot_sync(kFull, dg >> b & 1u);
        peers &= (dg >> b & 1u) ? bb : ~bb;
      }
      const uint32_t rank = __popc(peers & below);
      if (valid && rank == 0) s_cnt[wid][dg] = __popc(peers);
      __syncthreads();
      for (int w = 0; w < kGW; ++w) {
        const uint32_t c = s_cnt[w][threadIdx.x];
        s_off[w][threadIdx.x] = run;
        run += c;
        s_cnt[w][threadIdx.x] = 0;
      }
      __syncthreads();
      if (valid) {
        const u64 p = s_base[dg] + s_off[wid][dg] + rank;
        kout[p] = key;
        vout[p] = vin ? vin[i] : (uint32_t)(i / cap);
      }
    }
    __syncthreads(); // the tile's reads of s_base / s_off are done
  }
}

// ------------------------------------------------------------------ the graph
// Validation and degrees in one pass over the id matrix: deg[m] = senders listing m, ldeg[m] = this shard's rows listing
// m (sharded only); bad[0] = first local slot that breaks "ascending ids != self, vacancies last" (check_local),
// bad[1] = 1 + the last entry of any row holding an id >= N.
__global__ void __launch_bounds__(kGT) view_check_kernel(const uint32_t *nbr, uint32_t N, uint32_t cap, uint32_t first, uint32_t n,
                                                         int check_local, uint32_t *deg, uint32_t *ldeg, u64 *bad) {
  const size_t total = (size_t)N * cap;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (size_t)gridDim.x * blockDim.x) {
    const uint32_t m = nbr[x];
    if (m == SWIM_NO_MEMBER) continue;
    const uint32_t i = (uint32_t)(x / cap), s = (uint32_t)(x % cap);
    const bool mine = i - first < n;
    if (m >= N) {
      atomic_max_u64(&bad[1], (u64)x + 1);
    } else {
      atomicAdd(&deg[m], 1u);
      if (ldeg && mine) atomicAdd(&ldeg[m], 1u);
    }
    if (check_local && mine) {
      const uint32_t prev = s ? nbr[x - 1] : 0u;
      if ((s && prev == SWIM_NO_MEMBER) || m >= N || m == i || (s && m <= prev)) atomic_min_u64(&bad[0], (u64)(x - (size_t)first * cap));
    }
  }
}

__global__ void __launch_bounds__(kGT) init_vst_kernel(const uint32_t *nbr, size_t slots, uint8_t *vst) {
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < slots; x += (size_t)gridDim.x * blockDim.x)
    vst[x] = nbr[x] == SWIM_NO_MEMBER ? SWIM_VACANT : SWIM_ALIVE;
}

// Edge p of the sorted list (receiver key[p], sender val[p]): its place in the local receiver's in-list, the local
// sender's ridx entry (the index in the receiver's in-list, counted from the receiver's shard's first in-edge) and the
// local sender's observer entry. seg = first sorted position of every receiver; oseg (sharded) = first observer entry of
// every member among this shard's rows, which form one contiguous run of each receiver's ascending senders.
__global__ void __launch_bounds__(kGT) emit_kernel(const uint32_t *nbr, const uint32_t *key, const uint32_t *val, size_t E_all,
                                                   const u64 *seg, const u64 *oseg, uint32_t first, uint32_t n, uint32_t per,
                                                   uint32_t cap, uint32_t *in_src, uint32_t *ridx, uint32_t *obs_slot) {
  const u64 base = seg[first];
  for (size_t p = (size_t)blockIdx.x * blockDim.x + threadIdx.x; p < E_all; p += (size_t)gridDim.x * blockDim.x) {
    const uint32_t j = key[p], i = val[p];
    if (j - first < n) in_src[p - base] = i;
    if (i - first >= n) continue;
    const uint32_t *row = nbr + (size_t)i * cap; // ascending, vacancies (the largest value) last: the slot holding j
    uint32_t lo = 0, hi = cap;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (row[mid] < j) lo = mid + 1; else hi = mid;
    }
    const uint32_t x = (i - first) * cap + lo;
    ridx[x] = (uint32_t)(p - seg[(size_t)(j / per) * per]);
    if (!oseg) {
      obs_slot[p] = x;
    } else {
      u64 a = seg[j], b = seg[(size_t)j + 1];
      while (a < b) {
        const u64 mid = (a + b) >> 1;
        if (val[mid] < first) a = mid + 1; else b = mid;
      }
      obs_slot[oseg[j] + (p - a)] = x;
    }
  }
}

__global__ void __launch_bounds__(kGT) offsets_kernel(const u64 *seg, const u64 *oseg, uint32_t N, uint32_t first, uint32_t n,
                                                      uint32_t *in_off, uint32_t *obs_off) {
  for (size_t m = (size_t)blockIdx.x * blockDim.x + threadIdx.x; m <= N; m += (size_t)gridDim.x * blockDim.x) {
    obs_off[m] = (uint32_t)(oseg ? oseg[m] : seg[m]);
    if (m <= n) in_off[m] = (uint32_t)(seg[first + m] - seg[first]);
  }
}

// membership filters of all N rows, one warp per row (bloom_pos, shared with the senders' test in swim_device.cuh)
__global__ void __launch_bounds__(kGT) bloom_kernel(const uint32_t *nbr, uint32_t N, uint32_t cap, uint32_t *bloom) {
  SWIM_SHARED_2D(uint32_t, s_bf, kGW, SWIM_MAX_VIEW / 2);
  const int lane = threadIdx.x & 31;
  uint32_t *bf = s_bf[threadIdx.x >> 5];
  const uint32_t words = cap / 2, bits = 16 * cap;
  for (uint32_t i = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; i < N; i += (gridDim.x * blockDim.x) >> 5) {
    for (uint32_t k = lane; k < words; k += 32) bf[k] = 0;
    __syncwarp();
    for (uint32_t s = lane; s < cap; s += 32) {
      const uint32_t m = nbr[(size_t)i * cap + s];
      if (m == SWIM_NO_MEMBER) continue;
      for (int which = 0; which < 2; ++which) {
        const uint32_t pos = bloom_pos(m, which, bits);
        atomicOr(&bf[pos >> 5], 1u << (pos & 31));
      }
    }
    __syncwarp();
    for (uint32_t k = lane; k < words; k += 32) bloom[(size_t)i * words + k] = bf[k];
    __syncwarp();
  }
}

// The mail graph of the global id matrix `nbr` (device memory, [N * cap]). With `api` (swim_sim_set_view /
// _set_view_device) the local rows are validated first and then installed, every member Alive at incarnation 0.
int build_graph(swim_sim *sim, const uint32_t *nbr, const char *api) {
  SimDev &d = sim->dev;
  const uint32_t N = d.N, cap = d.cap;
  const size_t slots = (size_t)N * cap, lslots = (size_t)d.n * cap;
  const bool sharded = d.world > 1;
  Scratch s(sim);
  uint32_t *deg, *ldeg = nullptr;
  u64 *bad, *seg, *oseg = nullptr;
  SCRATCH(s, deg, N);
  SCRATCH(s, bad, 2);
  if (sharded) SCRATCH(s, ldeg, N);
  GRAPH_TRY(sim, cudaMemsetAsync(deg, 0, (size_t)N * 4, sim->stream));
  if (ldeg) GRAPH_TRY(sim, cudaMemsetAsync(ldeg, 0, (size_t)N * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(bad, 0xFF, 8, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(bad + 1, 0, 8, sim->stream));
  SWIM_LAUNCH(view_check_kernel, grid_of(sim, (slots + kGT - 1) / kGT), kGT, sim->stream, nbr, N, cap, d.first, d.n,
              api ? 1 : 0, deg, ldeg, bad);
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  u64 hb[2];
  GRAPH_TRY(sim, cudaMemcpyAsync(hb, bad, sizeof hb, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  if (api && hb[0] != ~0ull) {
    set_error(sim, "%s: row %u slot %u is not a sorted set of ids != self", api, d.first + (uint32_t)(hb[0] / cap),
              (uint32_t)(hb[0] % cap));
    return SWIM_EINVAL;
  }
  if (api) {
    if (nbr + (size_t)d.first * cap != d.nbr)
      GRAPH_TRY(sim, cudaMemcpyAsync(d.nbr, nbr + (size_t)d.first * cap, lslots * 4, cudaMemcpyDeviceToDevice, sim->stream));
    SWIM_LAUNCH(init_vst_kernel, grid_of(sim, (lslots + kGT - 1) / kGT), kGT, sim->stream, (const uint32_t *)d.nbr, lslots, d.vst);
    ++sim->launches;
    GRAPH_TRY(sim, cudaGetLastError());
    GRAPH_TRY(sim, cudaMemsetAsync(d.vinc, 0, lslots * 4, sim->stream));
    GRAPH_TRY(sim, cudaMemsetAsync(d.vlast, 0, lslots * 4, sim->stream));
  }
  if (hb[1]) {
    const size_t x = (size_t)(hb[1] - 1);
    uint32_t v = 0;
    GRAPH_TRY(sim, cudaMemcpy(&v, nbr + x, 4, cudaMemcpyDeviceToHost));
    set_error(sim, "view matrix entry %zu holds id %u >= N (%u)", x, v, N);
    return SWIM_EINVAL;
  }
  SCRATCH(s, seg, (size_t)N + 1);
  int rc;
  if ((rc = scan_u32(sim, s, deg, N, seg))) return rc;
  u64 h_first = 0, h_end = 0, E_all = 0;
  GRAPH_TRY(sim, cudaMemcpyAsync(&h_first, seg + d.first, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaMemcpyAsync(&h_end, seg + d.first + d.n, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaMemcpyAsync(&E_all, seg + N, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  const u64 E = h_end - h_first; // in-edges of this shard's receivers
  if (E > 0xFFFFFFFFull) { set_error(sim, "in-edge count %llu exceeds 2^32", E); return SWIM_ERANGE; }
  if (sharded) {
    SCRATCH(s, oseg, (size_t)N + 1);
    if ((rc = scan_u32(sim, s, ldeg, N, oseg))) return rc;
  }
  // sort every edge of the matrix by receiver (stable: senders stay ascending)
  const uint32_t *key = nullptr, *val = nullptr;
  if (E_all) {
    uint32_t *kb[2], *vb[2], *hist;
    u64 *off;
    for (int b = 0; b < 2; ++b) { SCRATCH(s, kb[b], E_all); SCRATCH(s, vb[b], E_all); }
    const uint32_t T0 = (uint32_t)((slots + kTile - 1) / kTile);
    SCRATCH(s, hist, (size_t)256 * T0);
    SCRATCH(s, off, (size_t)256 * T0 + 1);
    const uint32_t bits = 32 - __builtin_clz(N - 1); // N >= 2 here: a row never lists its own id
    const uint32_t *kin = nbr, *vin = nullptr;
    size_t cnt = slots;
    for (uint32_t pass = 0; pass * 8 < bits; ++pass) {
      const uint32_t T = (uint32_t)((cnt + kTile - 1) / kTile), g = (uint32_t)grid_of(sim, T);
      SWIM_LAUNCH(radix_hist_kernel, g, kGT, sim->stream, kin, cnt, pass * 8, hist, T);
      ++sim->launches;
      if ((rc = scan_u32(sim, s, hist, (size_t)256 * T, off))) return rc;
      SWIM_LAUNCH(radix_scatter_kernel, g, kGT, sim->stream, kin, vin, cap, cnt, pass * 8, (const u64 *)off, T, kb[pass & 1], vb[pass & 1]);
      ++sim->launches;
      GRAPH_TRY(sim, cudaGetLastError());
      kin = kb[pass & 1];
      vin = vb[pass & 1];
      cnt = E_all;
    }
    key = kin;
    val = vin;
  }
  // the new index replaces the old one
  if (sim->d_in_src) { cudaFree(sim->d_in_src); sim->d_in_src = nullptr; }
  if (sim->d_eflag) { cudaFree(sim->d_eflag); sim->d_eflag = nullptr; }
  if (sim->d_bloom) { cudaFree(sim->d_bloom); sim->d_bloom = nullptr; }
  const size_t Ea = E ? (size_t)E : 1;
  const size_t estride = (Ea + 255) & ~(size_t)255; // parity stride of the mail flags
  d.estride = (uint32_t)estride;
  GRAPH_TRY(sim, cudaMalloc((void **)&sim->d_in_src, Ea * 4));
  GRAPH_TRY(sim, cudaMalloc((void **)&sim->d_eflag, 2 * estride));
  GRAPH_TRY(sim, cudaMalloc((void **)&sim->d_bloom, slots / 2 * 4));
  GRAPH_TRY(sim, cudaMemsetAsync(sim->d_eflag, 0, 2 * estride, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(d.ridx, 0, lslots * 4, sim->stream));
  GRAPH_TRY(sim, cudaMemsetAsync(d.obs_slot, 0, lslots * 4, sim->stream));
  d.in_src = sim->d_in_src;
  d.eflag = sim->d_eflag;
  d.bloom = sim->d_bloom;
  if (E_all)
    SWIM_LAUNCH(emit_kernel, grid_of(sim, (E_all + kGT - 1) / kGT), kGT, sim->stream, nbr, key, val, (size_t)E_all,
                (const u64 *)seg, (const u64 *)oseg, d.first, d.n, d.per, cap, sim->d_in_src, d.ridx, d.obs_slot);
  SWIM_LAUNCH(offsets_kernel, grid_of(sim, ((size_t)N + kGT) / kGT), kGT, sim->stream, (const u64 *)seg, (const u64 *)oseg, N,
              d.first, d.n, d.in_off, d.obs_off);
  SWIM_LAUNCH(bloom_kernel, grid_of(sim, ((size_t)N + kGW - 1) / kGW), kGT, sim->stream, nbr, N, cap, sim->d_bloom);
  sim->launches += E_all ? 3 : 2;
  GRAPH_TRY(sim, cudaGetLastError());
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  sim->tdead_dirty = true;
  ++sim->view_epoch;
  sim->n_edges = E;
  return swim::dist_alloc_edges(sim);
}

int install_view(swim_sim *sim, const uint32_t *nbr_dev, const char *api) {
  int rc = build_graph(sim, nbr_dev, api);
  if (rc) return rc;
  sim->view_set = true;
  sim->edges_dirty = false;
  return SWIM_OK;
}

// ------------------------------------------------------------------ bulk membership edits (one warp per row)
// removeDeadNodes (Core.hs:65-67) on every local row: Dead entries at least min_age rounds old leave, the rest keep
// their order and move to the front, exactly as the scalar call compacts a row.
template <int W>
__global__ void __launch_bounds__(kGT) remove_dead_kernel(SimDev d, uint32_t round, uint32_t min_age, u64 *n_removed) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t removed = 0;
  for (uint32_t l = warp; l < d.n; l += nwarps) {
    const size_t base = (size_t)l * d.cap + lane;
    uint32_t nb[W], inc[W], last[W];
    uint8_t st[W];
    bool keep[W], drop_any = false;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const size_t x = base + 32 * w;
      nb[w] = d.nbr[x]; st[w] = d.vst[x]; inc[w] = d.vinc[x]; last[w] = d.vlast[x];
      const uint32_t live = st[w] & 3u;
      const bool drop = live == SWIM_DEAD && round - last[w] >= min_age;
      keep[w] = live != SWIM_VACANT && !drop;
      drop_any |= drop;
    }
    const unsigned dm = __ballot_sync(kFull, drop_any);
    if (!dm) continue;
    uint32_t used = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const unsigned km = __ballot_sync(kFull, keep[w]);
      if (keep[w]) {
        const size_t y = (size_t)l * d.cap + used + __popc(km & ((1u << lane) - 1u));
        d.nbr[y] = nb[w]; d.vst[y] = st[w]; d.vinc[y] = inc[w]; d.vlast[y] = last[w];
      }
      used += __popc(km);
    }
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const uint32_t s = 32 * w + lane;
      if (s >= used) {
        const size_t x = base + 32 * w;
        d.nbr[x] = SWIM_NO_MEMBER; d.vst[x] = SWIM_VACANT; d.vinc[x] = 0; d.vlast[x] = 0;
      }
    }
    uint32_t gone = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) gone += __popc(__ballot_sync(kFull, (st[w] & 3u) != SWIM_VACANT && !keep[w]));
    removed += gone;
  }
  if (lane == 0 && removed) atomicAdd(n_removed, (u64)removed);
}

// addNewMember (Core.hs:206-216) for the observers of the adds: adds[grp[g] .. grp[g + 1]) are one observer's, in the
// order given. A listed member is left alone; an unlisted one is inserted in id order as Alive with the add's
// incarnation and lastChange = round; an add to a full row is dropped. res = {added, dropped on a full row}.
template <int W>
__global__ void __launch_bounds__(kGT) add_members_kernel(SimDev d, uint32_t round, const uint4 *adds, const uint32_t *grp,
                                                          uint32_t ngroups, u64 *res) {
  const int lane = threadIdx.x & 31;
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = (gridDim.x * blockDim.x) >> 5;
  uint32_t added = 0, full = 0;
  for (uint32_t g = warp; g < ngroups; g += nwarps) {
    const uint32_t a0 = grp[g], a1 = grp[g + 1];
    const size_t base = (size_t)(adds[a0].x - d.first) * d.cap + lane;
    uint32_t nb[W], st[W], inc[W], last[W], used = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const size_t x = base + 32 * w;
      nb[w] = d.nbr[x]; st[w] = d.vst[x]; inc[w] = d.vinc[x]; last[w] = d.vlast[x];
      used += __popc(__ballot_sync(kFull, (st[w] & 3u) != SWIM_VACANT));
    }
    bool changed = false;
    for (uint32_t a = a0; a < a1; ++a) {
      const uint4 ad = adds[a];
      const uint32_t m = ad.y;
      uint32_t hit = 0, pos = 0;
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const bool present = (st[w] & 3u) != SWIM_VACANT;
        hit |= __ballot_sync(kFull, present && nb[w] == m);
        pos += __popc(__ballot_sync(kFull, present && nb[w] < m));
      }
      if (hit) continue;
      if (used == d.cap) { ++full; continue; }
      // slots >= pos move up by one (the last slot is vacant: used < cap), the new member takes slot pos. After the
      // rotation lane l holds lane l - 1 of the same word; lane 0 takes lane 31 of the word before.
      uint32_t up_nb[W], up_st[W], up_inc[W], up_last[W];
      const int src = (lane + 31) & 31;
#pragma unroll
      for (int w = 0; w < W; ++w) {
        up_nb[w] = __shfl_sync(kFull, nb[w], src); up_st[w] = __shfl_sync(kFull, st[w], src);
        up_inc[w] = __shfl_sync(kFull, inc[w], src); up_last[w] = __shfl_sync(kFull, last[w], src);
      }
      if (lane == 0) {
#pragma unroll
        for (int w = W - 1; w >= 1; --w) {
          up_nb[w] = up_nb[w - 1]; up_st[w] = up_st[w - 1]; up_inc[w] = up_inc[w - 1]; up_last[w] = up_last[w - 1];
        }
      }
#pragma unroll
      for (int w = 0; w < W; ++w) {
        const uint32_t s = 32 * w + lane;
        if (s == pos) { nb[w] = m; st[w] = SWIM_ALIVE; inc[w] = ad.z; last[w] = round; }
        else if (s > pos) { nb[w] = up_nb[w]; st[w] = up_st[w]; inc[w] = up_inc[w]; last[w] = up_last[w]; }
      }
      ++used;
      ++added;
      changed = true;
    }
    if (!changed) continue;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const size_t x = base + 32 * w;
      d.nbr[x] = nb[w]; d.vst[x] = (uint8_t)st[w]; d.vinc[x] = inc[w]; d.vlast[x] = last[w];
    }
  }
  if (lane == 0 && (added || full)) { atomicAdd(&res[0], (u64)added); atomicAdd(&res[1], (u64)full); }
}

// after a bulk edit: the rows changed on the device; the mail graph is rebuilt by the next step, the last round's
// envelopes no longer match the rows and the checkpoint belongs to the old view
void mark_edited(swim_sim *sim) {
  sim->edges_dirty = true;
  sim->tdead_dirty = true;
  sim->rows_edited = true;
  sim->ckpt_valid = false;
}

int edit_preamble(swim_sim *sim, const char *api) {
  if (sim->dev.world != 1) { set_error(sim, "%s: view membership changes are single-shard only", api); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  return SWIM_OK;
}

int row_grid(const swim_sim *sim, size_t rows) { return grid_of(sim, (rows + kGW - 1) / kGW); }

} // namespace

// Rebuild the mail graph from the device rows (after membership changes), in place: no host copy.
namespace swim {
int rebuild_edges_from_device(swim_sim *sim) {
  SimDev &d = sim->dev;
  if (d.world != 1) { set_error(sim, "view membership changes are single-shard only"); return SWIM_ESTATE; }
  int rc = build_graph(sim, d.nbr, nullptr);
  if (rc) return rc;
  sim->edges_dirty = false;
  return SWIM_OK;
}
} // namespace swim

extern "C" int swim_sim_set_view(swim_sim_t *sim, const uint32_t *nbr) {
  if (!sim || !nbr) return SWIM_EINVAL;
  const SimDev &d = sim->dev;
  if (d.p2p) { set_error(sim, "swim_sim_set_view: peers already mapped this rank's arrays (set the view before swim_sim_ipc_connect)"); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  Scratch s(sim);
  uint32_t *m;
  const size_t slots = (size_t)d.N * d.cap;
  SCRATCH(s, m, slots);
  GRAPH_TRY(sim, cudaMemcpyAsync(m, nbr, slots * 4, cudaMemcpyHostToDevice, sim->stream));
  return install_view(sim, m, "swim_sim_set_view");
}

extern "C" int swim_sim_set_view_device(swim_sim_t *sim, const uint32_t *nbr_global_dev) {
  if (!sim || !nbr_global_dev) return SWIM_EINVAL;
  if (sim->dev.p2p) { set_error(sim, "swim_sim_set_view_device: peers already mapped this rank's arrays (set the view before swim_sim_ipc_connect)"); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  return install_view(sim, nbr_global_dev, "swim_sim_set_view_device");
}

extern "C" int swim_sim_remove_dead_nodes(swim_sim_t *sim, uint32_t min_age, uint64_t *n_removed) {
  if (!sim) return SWIM_EINVAL;
  int rc = edit_preamble(sim, "swim_sim_remove_dead_nodes");
  if (rc) return rc;
  const SimDev &d = sim->dev;
  Scratch s(sim);
  u64 *cnt, h = 0;
  SCRATCH(s, cnt, 1);
  GRAPH_TRY(sim, cudaMemsetAsync(cnt, 0, 8, sim->stream));
  const int g = row_grid(sim, d.n);
  switch (d.cap / 32) {
    case 1: SWIM_LAUNCH(remove_dead_kernel<1>, g, kGT, sim->stream, d, sim->round, min_age, cnt); break;
    case 2: SWIM_LAUNCH(remove_dead_kernel<2>, g, kGT, sim->stream, d, sim->round, min_age, cnt); break;
    case 4: SWIM_LAUNCH(remove_dead_kernel<4>, g, kGT, sim->stream, d, sim->round, min_age, cnt); break;
    default: SWIM_LAUNCH(remove_dead_kernel<8>, g, kGT, sim->stream, d, sim->round, min_age, cnt); break;
  }
  GRAPH_TRY(sim, cudaGetLastError());
  ++sim->launches;
  GRAPH_TRY(sim, cudaMemcpyAsync(&h, cnt, 8, cudaMemcpyDeviceToHost, sim->stream));
  GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
  mark_edited(sim);
  if (n_removed) *n_removed = h;
  return SWIM_OK;
}

extern "C" int swim_sim_add_members(swim_sim_t *sim, const swim_member_add_t *adds, size_t n, uint64_t *n_added, uint64_t *n_full) {
  if (!sim || (!adds && n)) return SWIM_EINVAL;
  int rc = edit_preamble(sim, "swim_sim_add_members");
  if (rc) return rc;
  const SimDev &d = sim->dev;
  if (n > 0xFFFFFFFFull) { set_error(sim, "swim_sim_add_members: %zu adds in one call (at most 2^32 - 1)", n); return SWIM_EINVAL; }
  for (size_t x = 0; x < n; ++x)
    if (adds[x].observer >= d.N || adds[x].member >= d.N || adds[x].member == adds[x].observer) {
      set_error(sim, "swim_sim_add_members: add %zu (observer %u, member %u) is invalid (id >= N, or member == observer)", x,
                adds[x].observer, adds[x].member);
      return SWIM_EINVAL;
    }
  u64 h[2] = {0, 0};
  if (n) {
    // one group per observer, its adds in the order given
    std::vector<uint32_t> order(n);
    for (size_t x = 0; x < n; ++x) order[x] = (uint32_t)x;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return adds[a].observer < adds[b].observer; });
    std::vector<uint4> sorted(n);
    std::vector<uint32_t> grp;
    for (size_t x = 0; x < n; ++x) {
      const swim_member_add_t &a = adds[order[x]];
      sorted[x] = make_uint4(a.observer, a.member, a.incarnation, 0u);
      if (x == 0 || a.observer != adds[order[x - 1]].observer) grp.push_back((uint32_t)x);
    }
    const uint32_t ngroups = (uint32_t)grp.size();
    grp.push_back((uint32_t)n);
    Scratch s(sim);
    uint4 *d_adds;
    uint32_t *d_grp;
    u64 *res;
    SCRATCH(s, d_adds, n);
    SCRATCH(s, d_grp, grp.size());
    SCRATCH(s, res, 2);
    GRAPH_TRY(sim, cudaMemcpyAsync(d_adds, sorted.data(), n * sizeof(uint4), cudaMemcpyHostToDevice, sim->stream));
    GRAPH_TRY(sim, cudaMemcpyAsync(d_grp, grp.data(), grp.size() * 4, cudaMemcpyHostToDevice, sim->stream));
    GRAPH_TRY(sim, cudaMemsetAsync(res, 0, 16, sim->stream));
    const int g = row_grid(sim, ngroups);
    const uint4 *ca = d_adds;
    const uint32_t *cg = d_grp;
    switch (d.cap / 32) {
      case 1: SWIM_LAUNCH(add_members_kernel<1>, g, kGT, sim->stream, d, sim->round, ca, cg, ngroups, res); break;
      case 2: SWIM_LAUNCH(add_members_kernel<2>, g, kGT, sim->stream, d, sim->round, ca, cg, ngroups, res); break;
      case 4: SWIM_LAUNCH(add_members_kernel<4>, g, kGT, sim->stream, d, sim->round, ca, cg, ngroups, res); break;
      default: SWIM_LAUNCH(add_members_kernel<8>, g, kGT, sim->stream, d, sim->round, ca, cg, ngroups, res); break;
    }
    GRAPH_TRY(sim, cudaGetLastError());
    ++sim->launches;
    GRAPH_TRY(sim, cudaMemcpyAsync(h, res, sizeof h, cudaMemcpyDeviceToHost, sim->stream));
    GRAPH_TRY(sim, cudaStreamSynchronize(sim->stream));
    mark_edited(sim);
    if (h[0]) sim->view_set = true;
  }
  if (n_added) *n_added = h[0];
  if (n_full) *n_full = h[1];
  return SWIM_OK;
}
