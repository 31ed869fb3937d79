// swim_topology.cuh — the synthetic view graphs of swim_topology_generate (swim_topology.cpp), generated on the device.
// Compiled as part of swim_sim.cu's translation unit (included there once, after swim_graph.cuh, whose scratch, radix
// sort and install_view it uses).
//
// swim_sim_generate_view writes the global [N * cap] id matrix into device scratch and installs it exactly as
// swim_sim_set_view_device does. Every kind is bit-identical to the host generator, which is the statement these
// kernels are tested against:
//   complete, ring   one thread per slot, the sorted row computed in place;
//   random           one thread per row running the host's rejection loop on the same Philox counters, then the rows
//                    sorted (topo_rows_kernel);
//   symmetric        per cycle: Philox keys, a stable radix sort of (key, id) with the ids ascending (so ties come out
//                    by id), and predecessor / successor scattered into slots 2c / 2c + 1; then every row sorted with
//                    duplicates removed and padded (topo_rows_kernel).
#pragma once
#include "swim_host.h"

using namespace swim;

namespace {

// kind 0: row i = every id but i, ascending
__global__ void __launch_bounds__(kGT) topo_complete_kernel(uint32_t N, uint32_t cap, uint32_t *out) {
  const size_t total = (size_t)N * cap;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (size_t)gridDim.x * blockDim.x) {
    const uint32_t i = (uint32_t)(x / cap), s = (uint32_t)(x % cap);
    out[x] = s + 1 < N ? (s < i ? s : s + 1) : SWIM_NO_MEMBER;
  }
}

// kind 2: row i = i - back .. i - 1, i + 1 .. i + fwd (mod N), ascending. That list (offsets in that order) wraps past
// N - 1 or below 0 at most once (degree <= N - 1), so its sorted form is a rotation of it, starting at the wrap.
__global__ void __launch_bounds__(kGT) topo_ring_kernel(uint32_t N, uint32_t cap, uint32_t degree, uint32_t *out) {
  const uint32_t back = degree / 2, fwd = degree - back;
  const size_t total = (size_t)N * cap;
  for (size_t x = (size_t)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (size_t)gridDim.x * blockDim.x) {
    const uint32_t i = (uint32_t)(x / cap), s = (uint32_t)(x % cap);
    uint32_t v = SWIM_NO_MEMBER;
    if (s < degree) {
      const uint32_t start = i < back ? back - i : (uint64_t)i + fwd >= N ? N - 1 - i + back : 0u;
      const uint32_t k = (start + s) % degree;
      // offset k - back (below i) or k - back + 1 (above i), taken mod N
      const uint64_t o = k < back ? (uint64_t)N - (back - k) : (uint64_t)(k - back + 1);
      v = (uint32_t)(((uint64_t)i + o) % N);
    }
    out[x] = v;
  }
}

// kind 1: degree distinct ids != i by rejection sampling on Philox (i, attempt block, P_TOPO, 0), in draw order; the
// rest of the row vacant. topo_rows_kernel sorts the rows afterwards.
__global__ void __launch_bounds__(kGT) topo_random_kernel(uint32_t N, uint32_t cap, uint32_t degree, uint32_t k0, uint32_t k1,
                                                          uint32_t *out) {
  for (size_t ii = (size_t)blockIdx.x * blockDim.x + threadIdx.x; ii < N; ii += (size_t)gridDim.x * blockDim.x) {
    const uint32_t i = (uint32_t)ii;
    uint32_t *row = out + ii * cap;
    uint32_t cnt = 0, block = 0;
    while (cnt < degree) {
      const uint4 y = philox4x32_10(make_uint4(i, block++, P_TOPO, 0u), k0, k1);
      for (int w = 0; w < 4 && cnt < degree; ++w) {
        uint32_t id = bounded(word_of(y, w), N - 1);
        if (id >= i) ++id; // skip self
        bool dup = false;
        for (uint32_t z = 0; z < cnt; ++z) dup |= row[z] == id;
        if (!dup) row[cnt++] = id;
      }
    }
    for (uint32_t s = cnt; s < cap; ++s) row[s] = SWIM_NO_MEMBER;
  }
}

// kind 3, cycle c: key[i] = word i & 3 of Philox (c, i >> 2, P_TOPOSYM, 0), one block per four nodes
__global__ void __launch_bounds__(kGT) topo_keys_kernel(uint32_t N, uint32_t c, uint32_t k0, uint32_t k1, uint32_t *key) {
  const size_t groups = ((size_t)N + 3) / 4;
  for (size_t g = (size_t)blockIdx.x * blockDim.x + threadIdx.x; g < groups; g += (size_t)gridDim.x * blockDim.x) {
    const uint4 y = philox4x32_10(make_uint4(c, (uint32_t)g, P_TOPOSYM, 0u), k0, k1);
    for (int j = 0; j < 4; ++j) {
      const size_t i = 4 * g + j;
      if (i < N) key[i] = word_of(y, j);
    }
  }
}

// kind 3, cycle c: node order[t] takes order[t - 1] (slot 2c) and order[t + 1] (slot 2c + 1), cyclically
__global__ void __launch_bounds__(kGT) topo_cycle_kernel(const uint32_t *order, uint32_t N, uint32_t cap, uint32_t c, uint32_t *out) {
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < N; t += (size_t)gridDim.x * blockDim.x) {
    uint32_t *row = out + (size_t)order[t] * cap + 2 * c;
    row[0] = order[t ? t - 1 : N - 1];
    row[1] = order[t + 1 < N ? t + 1 : 0];
  }
}

// One warp per row (lane owns slots 32 w + lane): the row's ids ascending, each once, SWIM_NO_MEMBER after them. A
// repeated id keeps its first slot; an id's place is the number of distinct ids below it.
template <int W>
__global__ void __launch_bounds__(kGT) topo_rows_kernel(uint32_t N, uint32_t *out) {
  SWIM_SHARED_2D(uint32_t, s_row, kGW, 32 * W);
  constexpr uint32_t cap = 32 * W;
  const int lane = threadIdx.x & 31;
  uint32_t *r = s_row[threadIdx.x >> 5];
  const size_t warp = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5, nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t i = warp; i < N; i += nwarps) {
    uint32_t *row = out + i * cap;
    uint32_t v[W];
#pragma unroll
    for (int w = 0; w < W; ++w) r[32 * w + lane] = row[32 * w + lane];
    __syncwarp();
#pragma unroll
    for (int w = 0; w < W; ++w) {
      const uint32_t s = 32 * w + lane, x = r[s];
      bool first = x != SWIM_NO_MEMBER;
      for (uint32_t t = 0; t < s; ++t) first &= r[t] != x;
      v[w] = first ? x : SWIM_NO_MEMBER;
    }
    __syncwarp();
    uint32_t kept = 0;
#pragma unroll
    for (int w = 0; w < W; ++w) {
      r[32 * w + lane] = v[w];
      kept += __popc(__ballot_sync(kFull, v[w] != SWIM_NO_MEMBER));
    }
    __syncwarp();
#pragma unroll
    for (int w = 0; w < W; ++w) {
      if (v[w] == SWIM_NO_MEMBER) continue;
      uint32_t pos = 0;
      for (uint32_t t = 0; t < cap; ++t) pos += r[t] < v[w];
      row[pos] = v[w];
    }
    for (uint32_t s = kept + lane; s < cap; s += 32) row[s] = SWIM_NO_MEMBER;
    __syncwarp(); // r is free for the next row
  }
}

int sort_rows(swim_sim *sim, uint32_t N, uint32_t cap, uint32_t *m) {
  const int g = grid_of(sim, ((size_t)N + kGW - 1) / kGW);
  switch (cap / 32) {
    case 1: SWIM_LAUNCH(topo_rows_kernel<1>, g, kGT, sim->stream, N, m); break;
    case 2: SWIM_LAUNCH(topo_rows_kernel<2>, g, kGT, sim->stream, N, m); break;
    case 4: SWIM_LAUNCH(topo_rows_kernel<4>, g, kGT, sim->stream, N, m); break;
    default: SWIM_LAUNCH(topo_rows_kernel<8>, g, kGT, sim->stream, N, m); break;
  }
  ++sim->launches;
  GRAPH_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

// swim_topology_generate(kind, N, cap, degree, seed, m) on the handle's stream; the arguments are already checked
int generate_matrix(swim_sim *sim, int kind, uint32_t N, uint32_t cap, uint32_t degree, uint64_t seed, uint32_t *m) {
  const size_t slots = (size_t)N * cap;
  const uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  const int gs = grid_of(sim, (slots + kGT - 1) / kGT), gn = grid_of(sim, ((size_t)N + kGT - 1) / kGT);
  if (kind == SWIM_TOPO_COMPLETE) {
    SWIM_LAUNCH(topo_complete_kernel, gs, kGT, sim->stream, N, cap, m);
    ++sim->launches;
  } else if (kind == SWIM_TOPO_RING) {
    SWIM_LAUNCH(topo_ring_kernel, gs, kGT, sim->stream, N, cap, degree, m);
    ++sim->launches;
  } else if (kind == SWIM_TOPO_RANDOM) {
    SWIM_LAUNCH(topo_random_kernel, gn, kGT, sim->stream, N, cap, degree, k0, k1, m);
    ++sim->launches;
    GRAPH_TRY(sim, cudaGetLastError());
    return sort_rows(sim, N, cap, m);
  } else {
    GRAPH_TRY(sim, cudaMemsetAsync(m, 0xFF, slots * 4, sim->stream));
    for (uint32_t c = 0; c < degree / 2; ++c) {
      Scratch s(sim); // one cycle's keys and sort buffers, freed before the next cycle's
      uint32_t *key;
      SCRATCH(s, key, N);
      SWIM_LAUNCH(topo_keys_kernel, grid_of(sim, ((size_t)N / 4 + kGT) / kGT), kGT, sim->stream, N, c, k0, k1, key);
      ++sim->launches;
      GRAPH_TRY(sim, cudaGetLastError());
      const uint32_t *skey, *order;
      int rc;
      if ((rc = radix_sort(sim, s, key, N, 1, N, 32, false, &skey, &order))) return rc; // value = position = id
      SWIM_LAUNCH(topo_cycle_kernel, gn, kGT, sim->stream, order, N, cap, c, m);
      ++sim->launches;
      GRAPH_TRY(sim, cudaGetLastError());
    }
    return sort_rows(sim, N, cap, m);
  }
  GRAPH_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

} // namespace

extern "C" int swim_sim_generate_view(swim_sim_t *sim, int kind, uint32_t degree, uint64_t seed) {
  if (!sim) return SWIM_EINVAL;
  const SimDev &d = sim->dev;
  const uint32_t asked = degree;
  int rc = swim::topology_params(kind, d.N, d.cap, &degree);
  if (rc) {
    set_error(sim, "swim_sim_generate_view: kind %d with degree %u does not fit N = %u, view_cap = %u", kind, asked, d.N, d.cap);
    return rc;
  }
  if (d.p2p) { set_error(sim, "swim_sim_generate_view: peers already mapped this rank's arrays (set the view before swim_sim_ipc_connect)"); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  Scratch s(sim);
  uint32_t *m;
  SCRATCH(s, m, (size_t)d.N * d.cap);
  if ((rc = generate_matrix(sim, kind, d.N, d.cap, degree, seed, m))) return rc;
  return install_view(sim, m, "swim_sim_generate_view");
}
