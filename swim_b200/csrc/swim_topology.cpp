// swim_topology.cpp — synthetic view graphs for the BASELINE configs (host side, no device).
// The reference has no topology notion: every process knows whatever `storeMembers` holds
// (Types.hs:55). A row here is one node's member map keys in ascending order (Core.hs:77).
#include <algorithm>
#include <cstdint>
#include <vector>

#include "../../include/swim.h"

namespace swim {
// (declared in swim_host.h: swim_sim_generate_view checks its arguments here too)
int topology_params(int kind, uint32_t N, uint32_t cap, uint32_t *degree) {
  if (N == 0 || cap == 0 || cap % 32 || cap > SWIM_MAX_VIEW) return SWIM_EINVAL;
  if (kind == SWIM_TOPO_COMPLETE) *degree = N - 1;
  if (kind == SWIM_TOPO_SYMMETRIC && (N < 3 || *degree < 2 || *degree % 2)) return SWIM_EINVAL;
  if (*degree > cap || *degree > N - 1) return SWIM_ECAP;
  if (kind != SWIM_TOPO_COMPLETE && kind != SWIM_TOPO_RANDOM && kind != SWIM_TOPO_RING && kind != SWIM_TOPO_SYMMETRIC)
    return SWIM_EINVAL;
  return SWIM_OK;
}
} // namespace swim

namespace {
struct Philox {
  uint32_t k0, k1;
  void operator()(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t out[4]) const {
    uint32_t a = k0, b = k1;
    for (int r = 0; r < 10; ++r) {
      uint64_t p0 = 0xD2511F53ull * c0, p1 = 0xCD9E8D57ull * c2;
      uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ a, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ b;
      c1 = (uint32_t)p1; c3 = (uint32_t)p0; c0 = n0; c2 = n2;
      a += 0x9E3779B9u; b += 0xBB67AE85u;
    }
    out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
  }
};

// Symmetric random views: the union of degree / 2 random Hamiltonian cycles. Cycle c visits the nodes in the order of
// (key_c(i), i), key_c(i) = word i & 3 of Philox(ctr = (c, i >> 2, P_TOPOSYM = 11, 0)); each node takes its predecessor
// and successor on every cycle, and its row is their distinct values, ascending. Written for clarity, not speed: this
// is the statement the device generator (swim_topology.cuh) is tested against.
void symmetric_rows(const Philox &rng, uint32_t N, uint32_t cap, uint32_t degree, uint32_t *out) {
  const uint32_t cycles = degree / 2;
#pragma omp parallel for schedule(dynamic, 1)
  for (int64_t cc = 0; cc < (int64_t)cycles; ++cc) {
    const uint32_t c = (uint32_t)cc;
    std::vector<uint64_t> order(N);
    for (uint32_t i = 0; i < N; ++i) {
      uint32_t w[4];
      rng(c, i >> 2, 11u, 0u, w);
      order[i] = (uint64_t)w[i & 3] << 32 | i;
    }
    std::sort(order.begin(), order.end());
    for (uint32_t t = 0; t < N; ++t) {
      const uint32_t i = (uint32_t)order[t];
      uint32_t *row = out + (size_t)i * cap;
      row[2 * c] = (uint32_t)order[(t + N - 1) % N];
      row[2 * c + 1] = (uint32_t)order[(t + 1) % N];
    }
  }
#pragma omp parallel for schedule(static)
  for (int64_t ii = 0; ii < (int64_t)N; ++ii) {
    uint32_t *row = out + (size_t)ii * cap;
    std::sort(row, row + degree);
    const uint32_t cnt = (uint32_t)(std::unique(row, row + degree) - row);
    for (uint32_t s = cnt; s < cap; ++s) row[s] = SWIM_NO_MEMBER;
  }
}
} // namespace

extern "C" int swim_topology_generate(int kind, uint32_t N, uint32_t cap, uint32_t degree, uint64_t seed,
                                      uint32_t *out) {
  if (!out) return SWIM_EINVAL;
  const int rc = swim::topology_params(kind, N, cap, &degree);
  if (rc) return rc;
  const Philox rng{(uint32_t)seed, (uint32_t)(seed >> 32)};
  if (kind == SWIM_TOPO_SYMMETRIC) {
    symmetric_rows(rng, N, cap, degree, out);
    return SWIM_OK;
  }
#pragma omp parallel for schedule(static)
  for (int64_t ii = 0; ii < (int64_t)N; ++ii) {
    const uint32_t i = (uint32_t)ii;
    uint32_t *row = out + (size_t)i * cap;
    uint32_t cnt = 0;
    if (kind == SWIM_TOPO_COMPLETE) {
      for (uint32_t j = 0; j < N; ++j)
        if (j != i) row[cnt++] = j;
    } else if (kind == SWIM_TOPO_RING) {
      // i±1 .. ±degree/2 (an odd degree takes one more successor)
      const uint32_t back = degree / 2, fwd = degree - back;
      for (uint32_t o = 1; o <= back; ++o) row[cnt++] = (uint32_t)(((uint64_t)i + N - o) % N);
      for (uint32_t o = 1; o <= fwd; ++o) row[cnt++] = (uint32_t)(((uint64_t)i + o) % N);
      std::sort(row, row + cnt);
    } else {
      // uniform random distinct ids != i: rejection sampling on Philox(ctr = (i, block, P_TOPO=3, 0))
      uint32_t block = 0;
      while (cnt < degree) {
        uint32_t w[4];
        rng(i, block++, 3u, 0u, w);
        for (int x = 0; x < 4 && cnt < degree; ++x) {
          uint32_t id = (uint32_t)(((uint64_t)w[x] * (N - 1)) >> 32);
          if (id >= i) ++id; // skip self
          bool dup = false;
          for (uint32_t y = 0; y < cnt; ++y) dup |= row[y] == id;
          if (!dup) row[cnt++] = id;
        }
      }
      std::sort(row, row + cnt);
    }
    for (; cnt < cap; ++cnt) row[cnt] = SWIM_NO_MEMBER;
  }
  return SWIM_OK;
}
