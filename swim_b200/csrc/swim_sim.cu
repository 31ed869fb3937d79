// swim_sim.cu — host side of the C ABI (include/swim.h): handle, HBM layout, round driver.
// Replaces the process wiring of Core.main (reference Core.hs:272-287): instead of three
// conduits and a ticker thread per OS process, one handle owns N stores in HBM and
// swim_sim_step runs the protocol period for all of them.
#include <algorithm>
#include <chrono>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "swim_device.cuh"
#include "swim_host.h"

using namespace swim;

namespace swim {
thread_local std::string g_last_error;

void set_error(swim_sim *sim, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_last_error = buf;
  if (sim) sim->last_error = buf;
}
} // namespace swim

#define CUDA_TRY(sim, call)                                                             \
  do {                                                                                  \
    cudaError_t e_ = (call);                                                            \
    if (e_ != cudaSuccess) {                                                            \
      set_error(sim, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return e_ == cudaErrorNoDevice || e_ == cudaErrorInsufficientDriver ? SWIM_ENODEV : SWIM_ECUDA; \
    }                                                                                   \
  } while (0)

extern "C" uint32_t swim_abi_version(void) { return SWIM_ABI_VERSION; }

extern "C" const char *swim_strerror(int code) {
  switch (code) {
    case SWIM_OK: return "ok";
    case SWIM_EINVAL: return "invalid argument";
    case SWIM_ENOMEM: return "out of memory";
    case SWIM_ECUDA: return "CUDA error";
    case SWIM_ERANGE: return "value out of range";
    case SWIM_EDECODE: return "decode error";
    case SWIM_ENODEV: return "no CUDA device (swim-b200 has no CPU fallback)";
    case SWIM_ENCCL: return "NCCL error";
    case SWIM_ECAP: return "capacity exceeded";
    case SWIM_ESTATE: return "invalid state";
  }
  return "unknown error";
}

extern "C" const char *swim_last_error(const swim_sim_t *sim) {
  return sim ? sim->last_error.c_str() : g_last_error.c_str();
}

extern "C" int swim_config_default(swim_config_t *cfg) {
  if (!cfg) return SWIM_EINVAL;
  memset(cfg, 0, sizeof *cfg);
  cfg->abi_version = SWIM_ABI_VERSION;
  cfg->n_nodes = 32;
  cfg->view_cap = 32;
  cfg->k_indirect = 3; // reference default numToGossip = 10 (Util.hs:48); BASELINE configs use k = 3
  cfg->fanout = 4;
  cfg->pb_cap = 8;
  cfg->suspicion_rounds = 5;
  cfg->retransmit = 8;
  cfg->loss_ppm = 0;
  cfg->seed = 0x5EED0001ull;
  cfg->rank = 0;
  cfg->world = 1;
  cfg->device = -1;
  cfg->base_port = 4000;
  cfg->churn_ppm = 0;
  cfg->rejoin_min = 10; // BASELINE config C5: rejoin after U[10, 50] rounds
  cfg->rejoin_max = 50;
  cfg->probes_per_round = 1;
  cfg->suspicion_max = 0;
  return SWIM_OK;
}

static int validate(const swim_config_t *c) {
  if (!c || c->abi_version != SWIM_ABI_VERSION) return SWIM_EINVAL;
  if (c->n_nodes == 0 || c->world == 0 || c->world > SWIM_MAX_WORLD || c->rank >= c->world) return SWIM_EINVAL;
  if (c->view_cap != 32 && c->view_cap != 64 && c->view_cap != 128 && c->view_cap != 256) return SWIM_EINVAL;
  if (c->k_indirect > SWIM_MAX_K || c->fanout < 1 || c->fanout > 1 + c->k_indirect) return SWIM_EINVAL;
  if (c->pb_cap < 1 || c->pb_cap > SWIM_MAX_PB) return SWIM_EINVAL;
  if (c->suspicion_rounds < 1 || c->suspicion_rounds > SWIM_MAX_TIMER) return SWIM_EINVAL;
  if (c->retransmit < 1 || c->retransmit > 255 || c->loss_ppm > 1000000u) return SWIM_EINVAL;
  if (c->flags & ~SWIM_F__ALL) return SWIM_EINVAL;
  if (c->churn_ppm > 1000000u || (c->churn_ppm && (c->rejoin_min < 1 || c->rejoin_max < c->rejoin_min))) return SWIM_EINVAL;
  if (c->probes_per_round < 1 || c->probes_per_round > SWIM_MAX_PROBES) return SWIM_EINVAL;
  if (c->suspicion_max && (c->suspicion_max < c->suspicion_rounds || c->suspicion_max > SWIM_MAX_TIMER_LIFEGUARD)) return SWIM_EINVAL;
  return SWIM_OK;
}

namespace swim {
uint32_t shard_first(uint32_t N, uint32_t world, uint32_t rank) {
  uint64_t per = ((uint64_t)N + world - 1) / world, f = per * rank;
  return (uint32_t)(f > N ? N : f);
}
} // namespace swim

template <typename T>
static int dalloc(swim_sim *sim, T **p, size_t count, int fill) {
  if (count == 0) count = 1;
  CUDA_TRY(sim, cudaMalloc((void **)p, count * sizeof(T)));
  CUDA_TRY(sim, cudaMemset(*p, fill, count * sizeof(T)));
  sim->allocs.push_back((void *)*p);
  return SWIM_OK;
}

template <int W>
static void prepare_kernels(swim_sim *sim); // grid sizes + kernel preload, defined with the round driver

// suspicion countdown parameters: fixed timeout, or Lifeguard's timeout(c) = max - (max - min) log(c + 1) / log(K + 1) with
// K = 3 confirmations, the logarithms in 1/256ths (0, .5, log 3 / log 4, 1) so that host, device and oracle agree exactly
static void set_suspicion_params(SimDev &d, const swim_config_t *cfg) {
  d.lg = cfg->suspicion_max ? 1u : 0u;
  d.S_arm = cfg->suspicion_max ? cfg->suspicion_max : cfg->suspicion_rounds;
  d.tmask = d.lg ? SWIM_MAX_TIMER_LIFEGUARD : SWIM_MAX_TIMER;
  for (int c = 0; c < 4; ++c) d.lg_delta[c] = 0;
  if (d.lg) {
    static const uint32_t frac[4] = {0, 128, 203, 256};
    uint32_t T[4];
    for (int c = 0; c < 4; ++c) T[c] = cfg->suspicion_max - ((cfg->suspicion_max - cfg->suspicion_rounds) * frac[c] + 128) / 256;
    for (int c = 1; c < 4; ++c) d.lg_delta[c] = T[c - 1] - T[c];
  }
}

// device-generated crash / rejoin events of one round (churn_kernel): expected 2 N p of them, room for 4x + slack
static int alloc_churn_list(swim_sim *sim) {
  SimDev &d = sim->dev;
  if (!d.churn_ppm) return SWIM_OK;
  const uint32_t want = (uint32_t)std::min<uint64_t>((uint64_t)d.N * 2, (uint64_t)d.N * d.churn_ppm / 1000000ull * 8 + 4096);
  if (d.churn_ev && want <= d.churn_cap) return SWIM_OK;
  int r;
  if ((r = dalloc(sim, &d.churn_ev, want, 0))) return r; // (an outgrown list stays in `allocs` until destroy)
  d.churn_cap = want;
  if (!d.churn_cnt && (r = dalloc(sim, &d.churn_cnt, 4, 0))) return r;
  return SWIM_OK;
}

extern "C" int swim_sim_create(const swim_config_t *cfg, swim_sim_t **out) {
  if (!out) return SWIM_EINVAL;
  *out = nullptr;
  int rc = validate(cfg);
  if (rc) { set_error(nullptr, "swim_sim_create: invalid config"); return rc; }
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    set_error(nullptr, "swim_sim_create: no CUDA device (%s); swim-b200 has no CPU fallback",
              e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
    return SWIM_ENODEV;
  }
  swim_sim *sim = new (std::nothrow) swim_sim();
  if (!sim) return SWIM_ENOMEM;
  sim->cfg = *cfg;
  sim->opt_split = getenv("SWIM_SPLIT") != nullptr;
  // sharded runs with the fused exchange: one fused kernel per event-free stretch (the last CTA of a grid barrier does the cross-GPU handshake)
  // or the split launch sequence with peer_barrier_kernel; SWIM_ROUND_KERNEL=0|1 overrides the default
  if (const char *rk = getenv("SWIM_ROUND_KERNEL")) sim->opt_round_kernel = atoi(rk) != 0;
  sim->opt_one_round = getenv("SWIM_ONE_ROUND_PER_LAUNCH") != nullptr;
  // rounds decided per batched quiet scan of round_kernel (1..8; 0 or 1 turns batching off)
  if (const char *xm = getenv("SWIM_XMODE")) sim->opt_xmode = atoi(xm) != 0 ? 1 : 0;
  if (const char *qb = getenv("SWIM_QUIET_BATCH")) sim->opt_quiet_batch = (uint32_t)std::min(8l, std::max(0l, strtol(qb, nullptr, 10)));
  if (cfg->device >= 0) {
    rc = [&]() { CUDA_TRY(sim, cudaSetDevice(cfg->device)); return SWIM_OK; }();
    if (rc) { g_last_error = sim->last_error; delete sim; return rc; }
  }
  cudaGetDevice(&sim->device);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, sim->device);
  sim->sm_count = prop.multiProcessorCount;
  SimDev &d = sim->dev;
  memset(&d, 0, sizeof d);
  d.N = cfg->n_nodes; d.cap = cfg->view_cap; d.k = cfg->k_indirect; d.fanout = cfg->fanout;
  d.P = cfg->probes_per_round;
  d.B = cfg->pb_cap; d.S = cfg->suspicion_rounds; d.T = cfg->retransmit; d.loss_ppm = cfg->loss_ppm;
  d.flags = cfg->flags;
  set_suspicion_params(d, cfg);
  d.churn_ppm = cfg->churn_ppm; d.rejoin_min = cfg->rejoin_min; d.rejoin_span = cfg->rejoin_max - cfg->rejoin_min + 1;
  d.key0 = (uint32_t)cfg->seed; d.key1 = (uint32_t)(cfg->seed >> 32);
  d.world = cfg->world; d.rank = cfg->rank;
  d.per = (uint32_t)(((uint64_t)d.N + d.world - 1) / d.world);
  d.first = shard_first(d.N, d.world, d.rank);
  d.n = shard_first(d.N, d.world, d.rank + 1) - d.first;
  const size_t n = d.n, slots = n * d.cap;
  rc = [&]() -> int {
    int r;
    CUDA_TRY(sim, cudaStreamCreateWithFlags(&sim->own_stream, cudaStreamNonBlocking));
    sim->stream = sim->own_stream;
    CUDA_TRY(sim, cudaEventCreate(&sim->ev_start));
    CUDA_TRY(sim, cudaEventCreate(&sim->ev_stop));
    CUDA_TRY(sim, cudaEventCreateWithFlags(&sim->ev_upload, cudaEventDisableTiming));
    if ((r = dalloc(sim, &d.alive, d.N, 1))) return r;       // every node up
    if ((r = dalloc(sim, &d.back_at, d.N, 0))) return r;     // churn: no rejoin scheduled
    if ((r = dalloc(sim, &d.last_crash, d.N, 0))) return r;
    if ((r = dalloc(sim, &d.last_rejoin, d.N, 0))) return r;
    if ((r = alloc_churn_list(sim))) return r;
    if ((r = dalloc(sim, &d.self_inc, n, 0))) return r;      // Util.hs:80
    if ((r = dalloc(sim, &d.seqno, n, 0))) return r;         // Util.hs:79
    if ((r = dalloc(sim, &d.nbr, slots, 0xFF))) return r;    // Util.hs:78 empty member map
    if ((r = dalloc(sim, &d.vst, slots, 0))) return r;
    CUDA_TRY(sim, cudaMemset(d.vst, SWIM_VACANT, slots ? slots : 1));
    if ((r = dalloc(sim, &d.vinc, slots, 0))) return r;
    if ((r = dalloc(sim, &d.vlast, slots, 0))) return r;
    if ((r = dalloc(sim, &d.pb, n * d.B, 0))) return r;
    if ((r = dalloc(sim, &d.pb_cnt, n, 0))) return r;
    if ((r = dalloc(sim, &d.out, 2 * (size_t)d.per * d.B, 0))) return r; // [parity][per*B]
    if ((r = dalloc(sim, &d.out_cnt, 2 * (size_t)d.per, 0))) return r;
    if ((r = dalloc(sim, &d.claim, n, 0))) return r;
    if ((r = dalloc(sim, &d.xcnt, SWIM_MAX_WORLD, 0))) return r;
    d.rcap = d.per * d.fanout; // a source rank can list at most per*fanout receivers per round
    if (d.world > 1) {
      if ((r = dalloc(sim, &d.rlr, 2 * (size_t)d.world * d.rcap, 0))) return r;
      if ((r = dalloc(sim, &d.rcnt, 2 * (size_t)d.world, 0))) return r;
    }
    if ((r = dalloc(sim, &d.ridx, slots, 0))) return r;
    if ((r = dalloc(sim, &d.in_off, n + 1, 0))) return r;
    if ((r = dalloc(sim, &d.meta, slots / 32, 0))) return r;
    if ((r = dalloc(sim, &d.nsum, n, 0))) return r;
    if ((r = dalloc(sim, &d.obs_off, (size_t)d.N + 1, 0))) return r;
    if ((r = dalloc(sim, &d.obs_slot, slots, 0))) return r;
    if ((r = dalloc(sim, &d.wl, 2 * n, 0))) return r; // [parity]
    if ((r = dalloc(sim, &d.wl_cnt, 4, 0))) return r;
    if ((r = dalloc(sim, &d.ncand, 4, 0))) return r;
    d.mbw = (d.per + 31) / 32;
    if ((r = dalloc(sim, &d.mailbits, 3 * (size_t)d.mbw, 0))) return r;
    if ((r = dalloc(sim, &d.workbits, 3 * (size_t)d.mbw, 0))) return r;
    if ((r = dalloc(sim, &d.wl_n, 4, 0))) return r;
    if ((r = dalloc(sim, &d.rl, 2 * n * d.fanout, 0xFF))) return r; // [parity] recipient slots, empty = 0xFFFFFFFF
    if ((r = dalloc(sim, &d.cl, 2 * n * d.fanout, 0xFF))) return r; // [parity] delivered slots, compact
    // {digest, mismatch count} scratch and the counters share one block: swim_sim_observe reads both back in one copy
    if ((r = dalloc(sim, &sim->d_scratch, 2 + SWIM_CTR__COUNT, 0))) return r;
    d.ctr = sim->d_scratch + 2;
    if ((r = dalloc(sim, &sim->d_bar, SWIM_MAX_WORLD, 0))) return r;
    // watchdog word of the in-kernel waits: pinned host memory mapped into the device, so swim_sim_sync reads it
    // without a copy (it is written only when a wait gives up)
    CUDA_TRY(sim, cudaHostAlloc((void **)&sim->h_bar_err, sizeof(uint32_t), cudaHostAllocMapped));
    *sim->h_bar_err = 0;
    CUDA_TRY(sim, cudaHostGetDevicePointer((void **)&d.bar_err, sim->h_bar_err, 0));
    CUDA_TRY(sim, cudaHostAlloc((void **)&sim->h_observe, (SWIM_CTR__COUNT + 2) * sizeof(unsigned long long), cudaHostAllocDefault));
    CUDA_TRY(sim, cudaHostAlloc((void **)&sim->h_obs, (SWIM_CTR__COUNT + 4) * sizeof(unsigned long long), cudaHostAllocMapped));
    memset(sim->h_obs, 0, (SWIM_CTR__COUNT + 4) * sizeof(unsigned long long));
    CUDA_TRY(sim, cudaHostGetDevicePointer((void **)&sim->d_obs, sim->h_obs, 0));
    if ((r = dalloc(sim, &sim->d_obs_acc, 2, 0))) return r;
    if ((r = dalloc(sim, &sim->d_obs_done, 2, 0))) return r;
    if ((r = dalloc(sim, &d.gbar, 4, 0))) return r;
    if ((r = dalloc(sim, &d.qm, 4, 0))) return r;
    if ((r = dalloc(sim, &sim->d_coll, 1, 0))) return r; // barrier words of the collectives between steps
    return SWIM_OK;
  }();
  if (rc) { g_last_error = sim->last_error; swim_sim_destroy(sim); return rc; }
  switch (d.cap / 32) {
    case 1: prepare_kernels<1>(sim); break;
    case 2: prepare_kernels<2>(sim); break;
    case 4: prepare_kernels<4>(sim); break;
    default: prepare_kernels<8>(sim); break;
  }
  *out = sim;
  return SWIM_OK;
}

extern "C" void swim_sim_destroy(swim_sim_t *sim) {
  if (!sim) return;
  cudaSetDevice(sim->device);
  if (sim->own_stream) cudaStreamSynchronize(sim->own_stream);
  swim::dist_teardown(sim);
  for (void *p : sim->allocs) cudaFree(p);
  if (sim->d_in_src) cudaFree(sim->d_in_src);
  if (sim->d_eflag) cudaFree(sim->d_eflag);
  if (sim->d_bloom) cudaFree(sim->d_bloom);
  if (sim->d_events) cudaFree(sim->d_events);
  if (sim->dev.tl) cudaFree(sim->dev.tl);
  if (sim->h_events) cudaFreeHost(sim->h_events);
  if (sim->ev_upload) cudaEventDestroy(sim->ev_upload);
  for (auto &c : sim->ckpt_arrays) cudaFree(c.first);
  if (sim->d_eslot) { cudaFree(sim->d_eslot); sim->d_eslot = nullptr; }
  for (cudaEvent_t e : sim->prof_events) cudaEventDestroy(e);
  if (sim->h_bar_err) cudaFreeHost(sim->h_bar_err);
  if (sim->h_observe) cudaFreeHost(sim->h_observe);
  if (sim->h_obs) cudaFreeHost(sim->h_obs);
  if (sim->ev_start) cudaEventDestroy(sim->ev_start);
  if (sim->ev_stop) cudaEventDestroy(sim->ev_stop);
  if (sim->own_stream) cudaStreamDestroy(sim->own_stream);
  delete sim;
}

extern "C" int swim_sim_local_range(const swim_sim_t *sim, uint32_t *first, uint32_t *count) {
  if (!sim || !first || !count) return SWIM_EINVAL;
  *first = sim->dev.first;
  *count = sim->dev.n;
  return SWIM_OK;
}

// swim_sim_set_view / _set_view_device, the device-side mail-graph build and the bulk membership edits
#include "swim_graph.cuh"
// swim_sim_push_pull: the state exchange between steps
#include "swim_pushpull.cuh"
// swim_sim_join: seed joins between steps
#include "swim_join.cuh"
// swim_sim_leave: graceful leaves between steps
#include "swim_leave.cuh"
// swim_sim_generate_view: the synthetic view graphs generated on the device
#include "swim_topology.cuh"

// ------------------------------------------------------------------ events
extern "C" int swim_sim_inject(swim_sim_t *sim, const swim_event_t *ev, size_t n) {
  if (!sim || (!ev && n)) return SWIM_EINVAL;
  for (size_t x = 0; x < n; ++x) {
    if (ev[x].round <= sim->round || ev[x].node >= sim->dev.N || ev[x].kind > SWIM_EV_INJECT) {
      set_error(sim, "swim_sim_inject: event %zu invalid (round %u <= %u, node %u, kind %u)", x, ev[x].round,
                sim->round, ev[x].node, ev[x].kind);
      return SWIM_EINVAL;
    }
    if (ev[x].kind == SWIM_EV_INJECT) {
      const swim_message_t &m = ev[x].msg;
      if (m.kind != SWIM_MSG_SUSPECT && m.kind != SWIM_MSG_ALIVE && m.kind != SWIM_MSG_DEAD) {
        set_error(sim, "swim_sim_inject: only Suspect/Alive/Dead can be injected");
        return SWIM_EINVAL;
      }
      if (m.incarnation < 0 || m.incarnation > 0xFFFFFFFFll) return SWIM_ERANGE;
    }
  }
  // the queue stays sorted by round (stable: same-round events keep the order they were given in): only the new batch
  // is sorted, then merged in
  const auto by_round = [](const swim_event_t &a, const swim_event_t &b) { return a.round < b.round; };
  const size_t old_n = sim->events.size();
  sim->events.insert(sim->events.end(), ev, ev + n);
  std::stable_sort(sim->events.begin() + old_n, sim->events.end(), by_round);
  std::inplace_merge(sim->events.begin(), sim->events.begin() + old_n, sim->events.end(), by_round);
  return SWIM_OK;
}

// ------------------------------------------------------------------ round driver
static int grid_for(const swim_sim *sim, size_t warps_needed) {
  size_t blocks = (warps_needed + kWarpsPerBlock - 1) / kWarpsPerBlock;
  size_t cap = (size_t)sim->sm_count * (2048 / kThreads);
  if (blocks < 1) blocks = 1;
  return (int)std::min(blocks, cap);
}

// one resident wave of a persistent kernel: SMs x (CTAs the occupancy calculator allows per SM)
template <typename K>
static int wave_grid(const swim_sim *sim, K kernel, size_t warps_needed) {
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kThreads, 0) != cudaSuccess || per_sm < 1) per_sm = 1;
  size_t blocks = (warps_needed + kWarpsPerBlock - 1) / kWarpsPerBlock;
  if (blocks < 1) blocks = 1;
  return (int)std::min(blocks, (size_t)sim->sm_count * per_sm);
}

// launch with programmatic stream serialization (see pdl_wait / pdl_launch in swim_device.cuh)
template <typename K, typename... Args>
static cudaError_t launch_pdl_ex(K kernel, int grid, int block, cudaStream_t stream, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)block);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}
template <typename K>
static cudaError_t launch_pdl(K kernel, int grid, cudaStream_t stream, const SimDev &d) {
  return launch_pdl_ex(kernel, grid, kThreads, stream, d);
}

// Once per handle, at create: the one-wave grid sizes (occupancy queries), and every kernel of the bulk path is loaded
// now — with lazy module loading the first launch of a kernel pays its load, and for event_kernel that first launch
// would sit in the middle of a timed swim_sim_step call.
template <int W>
static void prepare_kernels(swim_sim *sim) {
  const SimDev &d = sim->dev;
  sim->grids[0] = wave_grid(sim, tick_scan_kernel<W>, ((size_t)d.n + 128 * kScanGroups) / (128 * kScanGroups) + 1);
  sim->grids[1] = wave_grid(sim, tick_work_kernel<W>, (size_t)d.n);
  sim->grids[2] = wave_grid(sim, recv_kernel<W>, (size_t)d.n);
  // (both instances of a round kernel: the grid must be co-resident whichever one a launch takes)
  sim->grids[4] = std::min(wave_grid(sim, round_kernel<W, false>, (size_t)d.n), wave_grid(sim, round_kernel<W, true>, (size_t)d.n));
  sim->grids[5] = std::min(wave_grid(sim, round_kernel_x<W, false>, (size_t)d.n), wave_grid(sim, round_kernel_x<W, true>, (size_t)d.n));
#ifndef SWIM_EMU
  cudaFuncAttributes a;
  cudaFuncGetAttributes(&a, event_kernel<W>);
  cudaFuncGetAttributes(&a, churn_kernel);
  cudaFuncGetAttributes(&a, derive_meta_kernel);
  cudaFuncGetAttributes(&a, digest_kernel);
  cudaFuncGetAttributes(&a, mismatch_kernel);
  cudaFuncGetAttributes(&a, observe_kernel);
  cudaFuncGetAttributes(&a, peer_barrier_kernel);
  cudaGetLastError();
#endif
}

template <int W>
static int run_rounds(swim_sim *sim, uint32_t rounds) {
  SimDev &d = sim->dev;
  const int grid = sim->grids[0], wgrid = sim->grids[1], rgrid = sim->grids[2];
  if (sim->tdead_dirty) {
    SWIM_LAUNCH(derive_meta_kernel, grid_for(sim, d.n), kThreads, sim->stream, d);
    ++sim->launches;
    sim->tdead_dirty = false;
  }
  // The events that fall inside this call leave the queue now (a failure further down must not replay them) and go to
  // the device through a pinned staging buffer: one asynchronous copy on the handle's stream, no synchronisation. Each
  // round's events are grouped by node (stable), which is what event_kernel's run ownership needs; events of different
  // nodes commute (a crash / rejoin touches alive[node] and the observers' crashed-member bits, an injected datagram its
  // own node's store), so only the per-node order is part of the semantics (DESIGN.md 2.2, phase E).
  size_t n_ev = 0;
  while (n_ev < sim->events.size() && sim->events[n_ev].round <= sim->round + rounds) ++n_ev;
  std::vector<uint32_t> ev_round; // round of staged event x
  if (n_ev) {
    if (n_ev > sim->d_events_cap) {
      CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
      if (sim->d_events) { cudaFree(sim->d_events); sim->d_events = nullptr; }
      if (sim->h_events) { cudaFreeHost(sim->h_events); sim->h_events = nullptr; }
      sim->d_events_cap = sim->h_events_cap = 0;
      const size_t cap = n_ev * 2 + 1024;
      CUDA_TRY(sim, cudaMalloc((void **)&sim->d_events, cap * sizeof(DevEvent)));
      CUDA_TRY(sim, cudaHostAlloc((void **)&sim->h_events, cap * sizeof(DevEvent), cudaHostAllocDefault));
      sim->d_events_cap = sim->h_events_cap = cap;
    } else {
      CUDA_TRY(sim, cudaEventSynchronize(sim->ev_upload)); // the previous call's copy has left the staging buffer (long ago)
    }
    std::vector<uint32_t> order(n_ev);
    for (size_t x = 0; x < n_ev; ++x) order[x] = (uint32_t)x;
    std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
      const swim_event_t &ea = sim->events[a], &eb = sim->events[b];
      return ea.round != eb.round ? ea.round < eb.round : ea.node < eb.node;
    });
    DevEvent *dev = (DevEvent *)sim->h_events;
    ev_round.resize(n_ev);
    for (size_t x = 0; x < n_ev; ++x) {
      const swim_event_t &e = sim->events[order[x]];
      ev_round[x] = e.round;
      dev[x].node = e.node;
      dev[x].kind = e.kind;
      dev[x].rec = make_uint4(e.msg.node, (uint32_t)e.msg.incarnation,
                              e.msg.kind == SWIM_MSG_DEAD ? e.msg.dead_from : 0u, e.msg.kind);
    }
    sim->events.erase(sim->events.begin(), sim->events.begin() + n_ev);
    CUDA_TRY(sim, cudaMemcpyAsync(sim->d_events, dev, n_ev * sizeof(DevEvent), cudaMemcpyHostToDevice, sim->stream));
    CUDA_TRY(sim, cudaEventRecord(sim->ev_upload, sim->stream));
  }
  size_t ev_pos = 0;
  // Default: one kernel per round. The split sequence (K1a, K1b, [exchange], K2 as separate launches) serves
  // per-kernel profiling, the staged NCCL exchange and SWIM_SPLIT=1.
  // Sharded runs with the fused exchange: round_kernel too (grid_barrier<true>: the last CTA to arrive at the barrier after
  // K1b — or at the scan barrier of a round without work — does the cross-GPU handshake, one thread per peer);
  // SWIM_ROUND_KERNEL=0 selects the split sequence + peer_barrier_kernel instead.
  const bool single_kernel = !sim->profile && !sim->opt_split &&
                             (d.world == 1 || (d.p2p && sim->opt_round_kernel));
  const int kgrid = sim->grids[4];
  const bool multi_round_off = sim->opt_one_round;
  // Event and churn kernels join the programmatic-serialization chain of the round kernels on a single shard only. A kernel
  // launched that way may become resident (and then sit in griddepcontrol.wait, holding its CTA slots) as soon as its
  // predecessor has started, so an unbroken chain lets a whole queue of future kernels pile up on the device. A shard's
  // round kernel waits ON THE DEVICE for its peers; when several ranks share one GPU (tests/test_gpu_shards_one_device.py)
  // the piled-up future kernels of one rank can take the slots another rank's current kernel still needs — a plain launch
  // here bounds the pile, as it did before.
  const bool chain_events = d.world == 1;
  for (uint32_t r = 0; r < rounds; ++r) {
    d.round = ++sim->round;
    size_t ev_end = ev_pos;
    while (ev_end < n_ev && ev_round[ev_end] == d.round) ++ev_end;
    if (d.churn_ppm) { // phase C: seeded churn of this round, generated and applied on the device
      int mk = prof_begin(sim, 0);
      // the list counter has two slots (round parity): churn_kernel of round r fills slot r & 1 and clears the other one
      // for round r + 1, so the chain churn -> events -> round kernel needs no memset between its launches and stays
      // programmatically serialised; only a jump of the round counter (load, set_round, first use) clears both here
      if (sim->churn_last_round + 1 != d.round) CUDA_TRY(sim, cudaMemsetAsync(d.churn_cnt, 0, 16, sim->stream));
      sim->churn_last_round = d.round;
      const uint32_t *cnt_r = d.churn_cnt + (d.round & 1u);
      if (chain_events) {
        CUDA_TRY(sim, launch_pdl_ex(churn_kernel, sim->sm_count * 8, 256, sim->stream, d));
        CUDA_TRY(sim, launch_pdl_ex(event_kernel<W>, sim->sm_count * 4, kThreads, sim->stream, d, (const DevEvent *)d.churn_ev, 0u, cnt_r));
      } else {
        SWIM_LAUNCH(churn_kernel, sim->sm_count * 8, 256, sim->stream, d);
        SWIM_LAUNCH(event_kernel<W>, sim->sm_count * 4, kThreads, sim->stream, d, (const DevEvent *)d.churn_ev, 0u, cnt_r);
      }
      prof_end(sim, mk);
      sim->launches += 2;
    }
    if (ev_end > ev_pos) {
      const uint32_t cnt = (uint32_t)(ev_end - ev_pos);
      const int eg = (int)std::min<size_t>((cnt + kWarpsPerBlock - 1) / kWarpsPerBlock, (size_t)sim->sm_count * 4);
      int mk = prof_begin(sim, 0);
      if (chain_events)
        CUDA_TRY(sim, launch_pdl_ex(event_kernel<W>, eg, kThreads, sim->stream, d, (const DevEvent *)sim->d_events + ev_pos, cnt,
                                    (const uint32_t *)nullptr));
      else
        SWIM_LAUNCH(event_kernel<W>, eg, kThreads, sim->stream, d, (const DevEvent *)sim->d_events + ev_pos, cnt, (const uint32_t *)nullptr);
      prof_end(sim, mk);
      ++sim->launches;
      ev_pos = ev_end;
    }
    if (single_kernel) { // K1a + K1b + K2 in one launch (grid barriers inside), for every round up to the next event
      uint32_t nr = rounds - r;
      if (ev_pos < n_ev) nr = std::min<uint32_t>(nr, ev_round[ev_pos] - d.round);
      if (multi_round_off || d.churn_ppm) nr = 1; // churn: events every round
      nr = std::min<uint32_t>(nr, 65536u); // (per-launch event counts are carried in 32 bits up to the final flush)
      d.nrounds = nr;
      d.qbatch = sim->opt_quiet_batch;
      d.fused = 1;
      // round_kernel_x (one grid barrier per round) pays a scan + barrier of its own at the start of every launch and gains
      // one barrier and one tail per busy round: it wins on long, lightly loaded event-free stretches of C3 and not on short
      // launches (a burst, or one round per call as in the end-to-end loop); the threshold has not been re-tuned on the
      // H100. Default ("auto"): launches of at least kXModeMinRounds rounds on a single
      // shard; SWIM_XMODE=1 / 0 forces it on (sharded runs included) / off.
      constexpr uint32_t kXModeMinRounds = 32;
      const bool use_x = sim->opt_xmode == 1 || (sim->opt_xmode < 0 && d.world == 1 && nr >= kXModeMinRounds);
      const bool sharded = d.world > 1 && d.p2p; // (otherwise a single shard: single_kernel rules out the staged exchange)
      if (use_x)
        CUDA_TRY(sim, launch_pdl(sharded ? round_kernel_x<W, true> : round_kernel_x<W, false>, sim->grids[5], sim->stream, d));
      else
        CUDA_TRY(sim, launch_pdl(sharded ? round_kernel<W, true> : round_kernel<W, false>, kgrid, sim->stream, d));
      d.fused = 0;
      ++sim->launches;
      sim->round += nr - 1;
      r += nr - 1;
      continue;
    }
    int mk = prof_begin(sim, 1);
    CUDA_TRY(sim, launch_pdl(tick_scan_kernel<W>, grid, sim->stream, d));
    prof_end(sim, mk);
    mk = prof_begin(sim, 4);
    CUDA_TRY(sim, launch_pdl(tick_work_kernel<W>, wgrid, sim->stream, d));
    prof_end(sim, mk);
    sim->launches += 2;
    if (d.world > 1) {
      mk = prof_begin(sim, 2);
      if (d.p2p) { // fused exchange: the data already sits in the peers' memory; synchronise the GPUs
        CUDA_TRY(sim, launch_pdl(peer_barrier_kernel, 1, sim->stream, d)); // keeps the PDL chain K1b -> barrier -> K2
        ++sim->launches;
      } else {     // staged exchange: envelopes moved by NCCL, flags raised by deliver_kernel
        int rc = swim::dist_exchange(sim);
        if (rc) return rc;
      }
      prof_end(sim, mk);
    }
    mk = prof_begin(sim, 3);
    CUDA_TRY(sim, launch_pdl(recv_kernel<W>, rgrid, sim->stream, d));
    prof_end(sim, mk);
    ++sim->launches;
    if (sim->profile) sim->prof_ms[5] += 1;
  }
  CUDA_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

// timed: bracket the call's kernels with the two events swim_sim_last_step_ms reads. swim_sim_step_observe — the per-round
// call of a study loop — goes without them: two stream operations and two API calls less per round, and nothing between
// the round kernel and the observe kernel that is chained behind it.
static int step_async_impl(swim_sim_t *sim, uint32_t rounds, bool timed) {
  if (!sim) return SWIM_EINVAL;
  if (!sim->view_set) { set_error(sim, "swim_sim_step: no view installed (swim_sim_set_view / swim_set_members)"); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  if (sim->edges_dirty || sim->bulk_dirty) {
    int rc = swim::rebuild_edges_from_device(sim);
    if (rc) return rc;
  }
  if (sim->dev.world > 1 && !sim->connected) { set_error(sim, "swim_sim_step: world > 1 needs swim_sim_ipc_connect or swim_sim_connect"); return SWIM_ESTATE; }
  if (sim->failed) { set_error(sim, "swim_sim_step: an earlier step failed part-way; the handle's device state is undefined"); return SWIM_ESTATE; }
  swim::refresh_peer_tables(sim);
  if (timed) CUDA_TRY(sim, cudaEventRecord(sim->ev_start, sim->stream));
  int rc;
  switch (sim->dev.cap / 32) {
    case 1: rc = run_rounds<1>(sim, rounds); break;
    case 2: rc = run_rounds<2>(sim, rounds); break;
    case 4: rc = run_rounds<4>(sim, rounds); break;
    default: rc = run_rounds<8>(sim, rounds); break;
  }
  if (rc) { sim->failed = true; return rc; } // rounds and events were consumed: no retry on this handle
  if (timed) CUDA_TRY(sim, cudaEventRecord(sim->ev_stop, sim->stream));
  sim->timed = timed;
  sim->rows_edited = false;
  return SWIM_OK;
}

extern "C" int swim_sim_step_async(swim_sim_t *sim, uint32_t rounds) { return step_async_impl(sim, rounds, true); }

extern "C" int swim_sim_sync(swim_sim_t *sim) {
  if (!sim) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  const uint32_t err = *(volatile uint32_t *)sim->h_bar_err;
  if (err) {
    set_error(sim, err == 1 ? "a cross-GPU wait timed out (a peer rank stopped stepping)"
                   : err == 3 ? "the device-side churn event list overflowed (churn_ppm too high for its capacity)"
                              : "an in-kernel grid barrier timed out");
    sim->failed = true; // the rounds of that launch ran without their barriers: the device state is undefined
    return SWIM_ESTATE;
  }
  return SWIM_OK;
}

extern "C" int swim_sim_step(swim_sim_t *sim, uint32_t rounds) {
  int rc = swim_sim_step_async(sim, rounds);
  if (rc) return rc;
  return swim_sim_sync(sim);
}

extern "C" int swim_sim_set_stream(swim_sim_t *sim, void *cuda_stream) {
  if (!sim) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  sim->stream = cuda_stream ? (cudaStream_t)cuda_stream : sim->own_stream;
  return SWIM_OK;
}

extern "C" int swim_sim_last_step_ms(const swim_sim_t *sim, float *ms) {
  if (!sim || !ms) return SWIM_EINVAL;
  if (!sim->timed) return SWIM_ESTATE;
  cudaError_t e = cudaEventElapsedTime(ms, sim->ev_start, sim->ev_stop);
  return e == cudaSuccess ? SWIM_OK : SWIM_ECUDA;
}

// Everything on the device that is stamped with a round number or holds one round's transient mail: after the round
// counter moves backwards (swim_sim_set_round on a handle that has stepped, swim_sim_load) a stale stamp would equal a
// round that is about to run again — recv_pass would take a receiver as "already claimed" and drop its mail.
static int reset_round_state(swim_sim *sim) {
  SimDev &d = sim->dev;
  const size_t n = d.n ? d.n : 1;
  CUDA_TRY(sim, cudaMemsetAsync(d.claim, 0, n * 4, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.wl_cnt, 0, 16, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.ncand, 0, 16, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.mailbits, 0, 3 * (size_t)d.mbw * 4, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.workbits, 0, 3 * (size_t)d.mbw * 4, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.wl_n, 0, 16, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.qm, 0, 16, sim->stream));
  CUDA_TRY(sim, cudaMemsetAsync(d.gbar, 0, 4, sim->stream)); // arrival count; the generation word keeps counting
  CUDA_TRY(sim, cudaMemsetAsync(d.xcnt, 0, SWIM_MAX_WORLD * 4, sim->stream));
  if (sim->d_eflag) CUDA_TRY(sim, cudaMemsetAsync(sim->d_eflag, 0, 2 * (size_t)d.estride, sim->stream));
  if (d.world > 1 && d.rcnt) CUDA_TRY(sim, cudaMemsetAsync(d.rcnt, 0, 2 * (size_t)d.world * 4, sim->stream));
  // cross-GPU barrier words: "peer q has published round r" — every peer stands at sim->round now (the caller holds
  // all ranks between steps while round counters move)
  uint32_t bar[SWIM_MAX_WORLD];
  for (uint32_t q = 0; q < SWIM_MAX_WORLD; ++q) bar[q] = sim->round;
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(sim->d_bar, bar, sizeof bar, cudaMemcpyHostToDevice));
  return SWIM_OK;
}

extern "C" int swim_sim_set_round(swim_sim_t *sim, uint32_t round) {
  if (!sim) return SWIM_EINVAL;
  if (!sim->events.empty() && sim->events.front().round <= round) {
    set_error(sim, "swim_sim_set_round: an event is pending at round %u <= %u", sim->events.front().round, round);
    return SWIM_EINVAL;
  }
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  sim->round = round;
  sim->tdead_dirty = true; // the per-node records are rebuilt (mail stamps included) before the next round
  return reset_round_state(sim);
}

extern "C" int swim_sim_set_params(swim_sim_t *sim, const swim_config_t *cfg) {
  if (!sim || !cfg) return SWIM_EINVAL;
  int rc = validate(cfg);
  if (rc) { set_error(sim, "swim_sim_set_params: invalid config"); return rc; }
  swim_config_t a = *cfg, b = sim->cfg; // everything but the protocol scalars must match the handle
  a.suspicion_rounds = b.suspicion_rounds; a.suspicion_max = b.suspicion_max; a.retransmit = b.retransmit;
  a.loss_ppm = b.loss_ppm; a.flags = b.flags; a.churn_ppm = b.churn_ppm; a.rejoin_min = b.rejoin_min;
  a.rejoin_max = b.rejoin_max; a.seed = b.seed; a._reserved = b._reserved;
  if (memcmp(&a, &b, sizeof a) != 0) { set_error(sim, "swim_sim_set_params: only suspicion_rounds, suspicion_max, retransmit, loss_ppm, flags, churn_ppm, rejoin_min/max and seed may change"); return SWIM_EINVAL; }
  if ((cfg->flags & SWIM_F_ROUND_ROBIN) && (cfg->view_cap & (cfg->view_cap - 1))) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  sim->cfg = *cfg;
  SimDev &d = sim->dev;
  d.S = cfg->suspicion_rounds; d.T = cfg->retransmit; d.loss_ppm = cfg->loss_ppm; d.flags = cfg->flags;
  d.key0 = (uint32_t)cfg->seed; d.key1 = (uint32_t)(cfg->seed >> 32);
  set_suspicion_params(d, cfg);
  d.churn_ppm = cfg->churn_ppm; d.rejoin_min = cfg->rejoin_min; d.rejoin_span = cfg->rejoin_max - cfg->rejoin_min + 1;
  return alloc_churn_list(sim);
}

// ------------------------------------------------------------------ device-resident checkpoint
static void ckpt_sources(const swim_sim *sim, std::vector<std::pair<void *, size_t>> &v) {
  const SimDev &d = sim->dev;
  const size_t n = d.n, slots = n * d.cap;
  v = {{d.alive, (size_t)d.N}, {d.back_at, (size_t)d.N * 4}, {d.last_crash, (size_t)d.N * 4}, {d.last_rejoin, (size_t)d.N * 4},
       {d.self_inc, n * 4}, {d.seqno, n * 4}, {d.vst, slots}, {d.vinc, slots * 4},
       {d.vlast, slots * 4}, {d.pb, n * d.B * sizeof(uint4)}, {d.pb_cnt, n}, {d.meta, slots / 32 * sizeof(uint4)},
       {d.nsum, n * 4}, {sim->d_scratch, (2 + SWIM_CTR__COUNT) * sizeof(unsigned long long)}};
}

extern "C" int swim_sim_save(swim_sim_t *sim) {
  if (!sim) return SWIM_EINVAL;
  if (!sim->view_set || sim->edges_dirty || sim->bulk_dirty) { set_error(sim, "swim_sim_save: no view installed, or memberships changed since the last step"); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  const SimDev &d = sim->dev;
  if (sim->tdead_dirty) { // the saved per-node records are current
    SWIM_LAUNCH(derive_meta_kernel, grid_for(sim, d.n), kThreads, sim->stream, d);
    ++sim->launches;
    sim->tdead_dirty = false;
  }
  std::vector<std::pair<void *, size_t>> src;
  ckpt_sources(sim, src);
  if (sim->ckpt_arrays.empty()) {
    for (auto &a : src) {
      void *p = nullptr;
      CUDA_TRY(sim, cudaMalloc(&p, a.second ? a.second : 1));
      sim->ckpt_arrays.push_back({p, a.second});
    }
  }
  for (size_t x = 0; x < src.size(); ++x)
    CUDA_TRY(sim, cudaMemcpyAsync(sim->ckpt_arrays[x].first, src[x].first, src[x].second, cudaMemcpyDeviceToDevice, sim->stream));
  sim->ckpt_round = sim->round;
  sim->ckpt_events = sim->events;
  sim->ckpt_epoch = sim->view_epoch;
  sim->ckpt_valid = true;
  return SWIM_OK;
}

extern "C" int swim_sim_load(swim_sim_t *sim) {
  if (!sim) return SWIM_EINVAL;
  if (!sim->ckpt_valid || sim->edges_dirty || sim->bulk_dirty || sim->ckpt_epoch != sim->view_epoch) {
    set_error(sim, "swim_sim_load: no checkpoint of this view (swim_sim_save first; a new view or a membership change drops it)");
    return SWIM_ESTATE;
  }
  cudaSetDevice(sim->device);
  std::vector<std::pair<void *, size_t>> dst;
  ckpt_sources(sim, dst);
  for (size_t x = 0; x < dst.size(); ++x)
    CUDA_TRY(sim, cudaMemcpyAsync(dst[x].first, sim->ckpt_arrays[x].first, dst[x].second, cudaMemcpyDeviceToDevice, sim->stream));
  sim->round = sim->ckpt_round;
  sim->events = sim->ckpt_events;
  sim->tdead_dirty = false;
  sim->failed = false;
  return reset_round_state(sim);
}

extern "C" int swim_sim_round(const swim_sim_t *sim, uint32_t *round) {
  if (!sim || !round) return SWIM_EINVAL;
  *round = sim->round;
  return SWIM_OK;
}

// ------------------------------------------------------------------ per-kernel profiling
namespace swim {
int prof_begin(swim_sim *sim, int phase) {
  if (!sim->profile) return -1;
  if (sim->prof_used + 2 > sim->prof_events.size()) {
    for (int x = 0; x < 2; ++x) {
      cudaEvent_t e;
      if (cudaEventCreate(&e) != cudaSuccess) return -1;
      sim->prof_events.push_back(e);
    }
  }
  const int idx = (int)sim->prof_used;
  sim->prof_used += 2;
  cudaEventRecord(sim->prof_events[idx], sim->stream);
  sim->prof_marks.push_back({phase, idx});
  return idx;
}
void prof_end(swim_sim *sim, int mark) {
  if (mark >= 0) cudaEventRecord(sim->prof_events[mark + 1], sim->stream);
}
int prof_collect(swim_sim *sim) {
  if (sim->prof_marks.empty()) return SWIM_OK;
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  for (auto &m : sim->prof_marks) {
    float ms = 0;
    if (cudaEventElapsedTime(&ms, sim->prof_events[m.second], sim->prof_events[m.second + 1]) == cudaSuccess)
      sim->prof_ms[m.first] += ms;
  }
  sim->prof_marks.clear();
  sim->prof_used = 0;
  return SWIM_OK;
}
} // namespace swim

extern "C" int swim_sim_set_profile(swim_sim_t *sim, int enable) {
  if (!sim) return SWIM_EINVAL;
  int rc = swim::prof_collect(sim);
  if (rc) return rc;
  sim->profile = enable != 0;
  if (enable) for (double &v : sim->prof_ms) v = 0;
  return SWIM_OK;
}

extern "C" int swim_sim_profile_ms(swim_sim_t *sim, double *out, size_t n) {
  if (!sim || !out) return SWIM_EINVAL;
  int rc = swim::prof_collect(sim);
  if (rc) return rc;
  for (size_t x = 0; x < n && x < SWIM_PROFILE_SLOTS; ++x) out[x] = sim->prof_ms[x];
  return SWIM_OK;
}

// Phase timeline of round_kernel (profiling aid; see tl_mark in swim_device.cuh): room for `rounds` rounds starting at
// the next round to run; 0 switches it off. Costs one %globaltimer read + one store by one thread per phase.
extern "C" int swim_sim_set_timeline(swim_sim_t *sim, uint32_t rounds) {
  if (!sim) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  SimDev &d = sim->dev;
  if (d.tl) { cudaFree(d.tl); d.tl = nullptr; }
  d.tl_cap = 0;
  if (!rounds) return SWIM_OK;
  CUDA_TRY(sim, cudaMalloc((void **)&d.tl, (size_t)rounds * 8 * sizeof(unsigned long long)));
  CUDA_TRY(sim, cudaMemset(d.tl, 0, (size_t)rounds * 8 * sizeof(unsigned long long)));
  d.tl_cap = rounds;
  d.tl_round0 = sim->round + 1;
  return SWIM_OK;
}

extern "C" int swim_sim_get_timeline(swim_sim_t *sim, uint64_t *out, size_t rounds) {
  if (!sim || !out) return SWIM_EINVAL;
  const SimDev &d = sim->dev;
  if (!d.tl || rounds > d.tl_cap) { set_error(sim, "swim_sim_get_timeline: not enabled for %zu rounds", rounds); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(out, d.tl, rounds * 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
  return SWIM_OK;
}

// ------------------------------------------------------------------ calibration of the latency floor
// What a round of the fused kernel cannot go below on this machine: the cost of one grid barrier of the resident wave
// (measured with the kernel's own barrier) and the latency of one dependent global load (pointer chase by one thread
// over a footprint beyond L2 for HBM, and well inside it for L2). bench.py turns them into roofline.latency_floor.
namespace {
__global__ void __launch_bounds__(kThreads, kMinBlocks) calib_barrier_kernel(SimDev d, uint32_t reps, unsigned long long *out) {
  barrier_begin(d);
  grid_barrier(d); // everybody is here
  unsigned long long t0 = 0, t1 = 0;
#ifndef SWIM_EMU
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
#endif
  for (uint32_t r = 0; r < reps; ++r) grid_barrier(d);
#ifndef SWIM_EMU
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
#endif
  if (blockIdx.x == 0 && threadIdx.x == 0) out[0] = t1 - t0;
}
__global__ void calib_fill_kernel(uint32_t *next, uint32_t mask) { // full-period LCG over [0, mask]: a single cycle
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i <= mask; i += (size_t)gridDim.x * blockDim.x)
    next[i] = ((uint32_t)i * 1664525u + 1013904223u) & mask;
}
__global__ void calib_chase_kernel(const uint32_t *next, uint32_t hops, unsigned long long *out) {
  uint32_t x = 12345u & 0xFFFFu;
  unsigned long long t0 = 0, t1 = 0;
#ifndef SWIM_EMU
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0));
#endif
  for (uint32_t h = 0; h < hops; ++h) x = __ldcg(next + x);
#ifndef SWIM_EMU
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
#endif
  out[0] = t1 - t0;
  out[1] = x;
}
} // namespace

extern "C" int swim_sim_calibrate(swim_sim_t *sim, double *out, size_t n) {
  if (!sim || !out || n < 4) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  const SimDev &d = sim->dev;
  unsigned long long *d_out = nullptr, h[2];
  uint32_t *next = nullptr;
  const uint32_t big = (1u << 27) - 1, small = (1u << 18) - 1; // 512 MB (beyond L2) and 1 MB (inside it)
  CUDA_TRY(sim, cudaMalloc((void **)&d_out, 16));
  int blocks = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&blocks, calib_barrier_kernel, kThreads, 0) != cudaSuccess || blocks < 1) blocks = 1;
  const int grid = std::min(sim->grids[4], sim->sm_count * blocks); // the fused kernel's wave
  const uint32_t reps = 200;
  SWIM_LAUNCH(calib_barrier_kernel, grid, kThreads, sim->stream, d, reps, d_out);
  CUDA_TRY(sim, cudaMemcpyAsync(h, d_out, 8, cudaMemcpyDeviceToHost, sim->stream));
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  out[0] = (double)h[0] / reps;
  out[3] = (double)grid * kWarpsPerBlock;
  if (cudaMalloc((void **)&next, ((size_t)big + 1) * 4) != cudaSuccess) { cudaFree(d_out); set_error(sim, "swim_sim_calibrate: out of memory"); return SWIM_ENOMEM; }
  for (int pass = 0; pass < 2; ++pass) {
    const uint32_t mask = pass == 0 ? big : small, hops = 4000;
    SWIM_LAUNCH(calib_fill_kernel, sim->sm_count * 8, 256, sim->stream, next, mask);
    if (pass == 1) SWIM_LAUNCH(calib_chase_kernel, 1, 1, sim->stream, next, mask + 1, d_out); // walk the whole cycle once: L2 warm
    SWIM_LAUNCH(calib_chase_kernel, 1, 1, sim->stream, next, hops, d_out);
    CUDA_TRY(sim, cudaMemcpyAsync(h, d_out, 16, cudaMemcpyDeviceToHost, sim->stream));
    CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
    out[1 + pass] = (double)h[0] / hops;
  }
  cudaFree(next);
  cudaFree(d_out);
  CUDA_TRY(sim, cudaGetLastError());
  return SWIM_OK;
}

extern "C" int swim_sim_launch_count(const swim_sim_t *sim, uint64_t *count) {
  if (!sim || !count) return SWIM_EINVAL;
  *count = sim->launches;
  return SWIM_OK;
}

// ------------------------------------------------------------------ bulk state access
static void *array_ptr(const swim_sim *sim, int arr, size_t *bytes) {
  const SimDev &d = sim->dev;
  const size_t n = d.n, slots = n * d.cap;
  switch (arr) {
    case SWIM_ARR_ALIVE: *bytes = d.N; return d.alive;
    case SWIM_ARR_SELF_INC: *bytes = n * 4; return d.self_inc;
    case SWIM_ARR_SEQNO: *bytes = n * 4; return d.seqno;
    case SWIM_ARR_NBR: *bytes = slots * 4; return d.nbr;
    case SWIM_ARR_VST: *bytes = slots; return d.vst;
    case SWIM_ARR_VINC: *bytes = slots * 4; return d.vinc;
    case SWIM_ARR_VLAST: *bytes = slots * 4; return d.vlast;
    case SWIM_ARR_PB: *bytes = n * d.B * sizeof(swim_record_t); return d.pb;
    case SWIM_ARR_PB_CNT: *bytes = n; return d.pb_cnt;
    case SWIM_ARR_BACK_AT: *bytes = (size_t)d.N * 4; return d.back_at;
    case SWIM_ARR_LAST_CRASH: *bytes = (size_t)d.N * 4; return d.last_crash;
    case SWIM_ARR_LAST_REJOIN: *bytes = (size_t)d.N * 4; return d.last_rejoin;
  }
  *bytes = 0;
  return nullptr;
}

extern "C" int swim_sim_array_bytes(const swim_sim_t *sim, int arr, size_t *bytes) {
  if (!sim || !bytes) return SWIM_EINVAL;
  return array_ptr(sim, arr, bytes) ? SWIM_OK : SWIM_EINVAL;
}

extern "C" int swim_sim_get_array(swim_sim_t *sim, int arr, void *buf, size_t bytes) {
  if (!sim || !buf) return SWIM_EINVAL;
  size_t want;
  void *p = array_ptr(sim, arr, &want);
  if (!p || want != bytes) { set_error(sim, "swim_sim_get_array(%d): expected %zu bytes, got %zu", arr, want, bytes); return SWIM_EINVAL; }
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(buf, p, bytes, cudaMemcpyDeviceToHost));
  if (arr == SWIM_ARR_PB) { // entries at or beyond the count are defined to read as zero
    std::vector<uint8_t> cnt(sim->dev.n ? sim->dev.n : 1);
    CUDA_TRY(sim, cudaMemcpy(cnt.data(), sim->dev.pb_cnt, sim->dev.n, cudaMemcpyDeviceToHost));
    swim_record_t *r = (swim_record_t *)buf;
    for (uint32_t l = 0; l < sim->dev.n; ++l)
      for (uint32_t q = cnt[l]; q < sim->dev.B; ++q) memset(&r[(size_t)l * sim->dev.B + q], 0, sizeof *r);
  }
  return SWIM_OK;
}

extern "C" int swim_sim_set_array(swim_sim_t *sim, int arr, const void *buf, size_t bytes) {
  if (!sim || !buf) return SWIM_EINVAL;
  if (arr == SWIM_ARR_NBR) { set_error(sim, "swim_sim_set_array: use swim_sim_set_view for SWIM_ARR_NBR"); return SWIM_EINVAL; }
  size_t want;
  void *p = array_ptr(sim, arr, &want);
  if (!p || want != bytes) { set_error(sim, "swim_sim_set_array(%d): expected %zu bytes, got %zu", arr, want, bytes); return SWIM_EINVAL; }
  if (arr == SWIM_ARR_VST) { // the countdown exists exactly while Suspect: a Suspect entry with timer 0 would wrap on its next tick
    const uint8_t *b = (const uint8_t *)buf;
    const SimDev &d = sim->dev;
    for (size_t x = 0; x < bytes; ++x) {
      const uint32_t live = b[x] & 3u, timer = (b[x] >> 2) & d.tmask;
      if (live == SWIM_SUSPECT ? (timer == 0 || timer > d.S_arm) : (b[x] >> 2) != 0) {
        set_error(sim, "swim_sim_set_array(SWIM_ARR_VST): entry %zu = 0x%02x: a Suspect entry needs a countdown in 1..%u, any other entry none", x, b[x], d.S_arm);
        return SWIM_EINVAL;
      }
    }
  }
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(p, buf, bytes, cudaMemcpyHostToDevice));
  if (arr == SWIM_ARR_ALIVE || arr == SWIM_ARR_VST || arr == SWIM_ARR_PB_CNT) sim->tdead_dirty = true; // meta is derived state
  return SWIM_OK;
}

static int reduce_u64(swim_sim *sim, int which, uint64_t *out) {
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaMemsetAsync(sim->d_scratch, 0, 8, sim->stream));
  const SimDev &d = sim->dev;
  if (which == 0) {
    SWIM_LAUNCH(digest_kernel, grid_for(sim, ((size_t)d.n * d.cap + 31) / 32 / 8 + 1), kThreads, sim->stream, d, sim->d_scratch);
  } else {
    if (sim->tdead_dirty) { // the detector reads the crashed-member bitmaps
      SWIM_LAUNCH(derive_meta_kernel, grid_for(sim, d.n), kThreads, sim->stream, d);
      ++sim->launches;
      sim->tdead_dirty = false;
    }
    SWIM_LAUNCH(mismatch_kernel, grid_for(sim, ((size_t)d.n + 31) / 32), kThreads, sim->stream, d, sim->d_scratch);
  }
  CUDA_TRY(sim, cudaGetLastError());
  ++sim->launches;
  unsigned long long v = 0;
  CUDA_TRY(sim, cudaMemcpyAsync(&v, sim->d_scratch, 8, cudaMemcpyDeviceToHost, sim->stream));
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  *out = v;
  return SWIM_OK;
}

extern "C" int swim_sim_digest(swim_sim_t *sim, uint64_t *digest) {
  if (!sim || !digest) return SWIM_EINVAL;
  return reduce_u64(sim, 0, digest);
}

extern "C" int swim_sim_mismatches(swim_sim_t *sim, uint64_t *count) {
  if (!sim || !count) return SWIM_EINVAL;
  return reduce_u64(sim, 1, count);
}

extern "C" int swim_sim_observe(swim_sim_t *sim, uint64_t *counters, size_t n_counters, uint64_t *digest, uint64_t *mismatches) {
  if (!sim) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  const SimDev &d = sim->dev;
  CUDA_TRY(sim, cudaMemsetAsync(sim->d_scratch, 0, 16, sim->stream));
  if (digest) {
    SWIM_LAUNCH(digest_kernel, grid_for(sim, ((size_t)d.n * d.cap + 31) / 32 / 8 + 1), kThreads, sim->stream, d, sim->d_scratch);
    ++sim->launches;
  }
  if (mismatches) {
    if (sim->tdead_dirty) {
      SWIM_LAUNCH(derive_meta_kernel, grid_for(sim, d.n), kThreads, sim->stream, d);
      ++sim->launches;
      sim->tdead_dirty = false;
    }
    SWIM_LAUNCH(mismatch_kernel, grid_for(sim, ((size_t)d.n + 31) / 32), kThreads, sim->stream, d, sim->d_scratch + 1);
    ++sim->launches;
  }
  CUDA_TRY(sim, cudaGetLastError());
  unsigned long long *h = sim->h_observe;
  CUDA_TRY(sim, cudaMemcpyAsync(h, sim->d_scratch, (2 + SWIM_CTR__COUNT) * sizeof(unsigned long long), cudaMemcpyDeviceToHost, sim->stream));
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  if (digest) *digest = h[0];
  if (mismatches) *mismatches = h[1];
  for (size_t i = 0; counters && i < n_counters && i < SWIM_CTR__COUNT; ++i) counters[i] = h[2 + i];
  return SWIM_OK;
}

// Step and read back in ONE call: `rounds` rounds, then observe_kernel chained behind them writes the cumulative counters
// and the convergence count straight into mapped pinned host memory; the host polls a sequence number there instead of
// synchronising the stream. No memset, no copy-engine operation, no stream synchronisation on the path.
extern "C" int swim_sim_step_observe(swim_sim_t *sim, uint32_t rounds, uint64_t *counters, size_t n_counters, uint64_t *mismatches) {
  if (!sim) return SWIM_EINVAL;
  int rc = step_async_impl(sim, rounds, false);
  if (rc) return rc;
  const SimDev &d = sim->dev;
  if (sim->tdead_dirty) { // (cannot be: the step above rebuilt the per-node records)
    SWIM_LAUNCH(derive_meta_kernel, grid_for(sim, d.n), kThreads, sim->stream, d);
    ++sim->launches;
    sim->tdead_dirty = false;
  }
  const unsigned long long seq = ++sim->obs_seq;
  const int grid = (int)std::max<size_t>(1, std::min<size_t>(((size_t)d.n + kThreads * 8 - 1) / (kThreads * 8), (size_t)sim->sm_count * 2));
  {
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)grid);
    cfg.blockDim = dim3(kThreads);
    cfg.stream = sim->stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    CUDA_TRY(sim, cudaLaunchKernelEx(&cfg, observe_kernel, d, sim->d_obs_acc, sim->d_obs_done,
                                     (volatile unsigned long long *)sim->d_obs, seq));
  }
  ++sim->launches;
  volatile unsigned long long *h = sim->h_obs;
  const auto t0 = std::chrono::steady_clock::now();
  for (unsigned long long spins = 0; h[SWIM_CTR__COUNT + 2] != seq; ++spins) {
#if defined(__x86_64__) && !defined(SWIM_EMU)
    __builtin_ia32_pause();
#endif
    if ((spins & 0x3FFFFull) != 0x3FFFFull) continue;
    // every few hundred microseconds: has the stream finished (or failed) without the report landing? has it taken too long?
    const cudaError_t q = cudaStreamQuery(sim->stream);
    const bool late = std::chrono::steady_clock::now() - t0 > std::chrono::seconds(120);
    if (q != cudaErrorNotReady || late) {
      if (!late) CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
      if (h[SWIM_CTR__COUNT + 2] != seq) {
        set_error(sim, late ? "swim_sim_step_observe: no report from the device after 120 s" : "swim_sim_step_observe: the stream finished without a report");
        sim->failed = true;
        return SWIM_ECUDA;
      }
    }
  }
  if (h[SWIM_CTR__COUNT + 1]) return swim_sim_sync(sim); // a watchdog fired: the usual report
  if (mismatches) *mismatches = h[SWIM_CTR__COUNT];
  for (size_t i = 0; counters && i < n_counters && i < SWIM_CTR__COUNT; ++i) counters[i] = h[i];
  return SWIM_OK;
}

extern "C" int swim_sim_counters(swim_sim_t *sim, uint64_t *out, size_t n) {
  if (!sim || !out) return SWIM_EINVAL;
  cudaSetDevice(sim->device);
  unsigned long long v[SWIM_CTR__COUNT];
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  CUDA_TRY(sim, cudaMemcpy(v, sim->dev.ctr, sizeof v, cudaMemcpyDeviceToHost));
  for (size_t i = 0; i < n && i < SWIM_CTR__COUNT; ++i) out[i] = v[i];
  return SWIM_OK;
}
