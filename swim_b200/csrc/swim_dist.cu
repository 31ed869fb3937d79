// swim_dist.cu — the cross-shard exchange: one all-to-all of piggyback envelopes per round.
//
// This is the UDP hop of the reference (Core.hs:280 sourceSocket / Core.hs:286 sinkToSocket) for
// envelopes whose receiver lives on another GPU. K1b appends such envelopes to per-destination
// buckets; after K1b every rank all-gathers the bucket counts, the counts reach the host (one
// stream synchronisation), a grouped ncclSend/ncclRecv moves exactly the filled part of every
// bucket over NVLink, and `deliver_kernel` turns the received envelopes into in-edge flags so that
// K2 runs unchanged. Receive order stays "ascending global sender id" because it is given by the
// receiver's sorted in-list, not by arrival order.
//
// NCCL is bound lazily (dlopen) so that single-GPU users of the C ABI need only the CUDA driver,
// and so that a Python process that already loaded torch's NCCL shares that copy.
#include <dlfcn.h>
#include <unistd.h>
#include <nccl.h>

#include <algorithm>
#include <chrono>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <thread>
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

struct NcclApi {
  void *handle = nullptr;
  ncclResult_t (*GetUniqueId)(ncclUniqueId *) = nullptr;
  ncclResult_t (*CommInitRank)(ncclComm_t *, int, ncclUniqueId, int) = nullptr;
  ncclResult_t (*CommDestroy)(ncclComm_t) = nullptr;
  ncclResult_t (*AllGather)(const void *, void *, size_t, ncclDataType_t, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Send)(const void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*Recv)(void *, size_t, ncclDataType_t, int, ncclComm_t, cudaStream_t) = nullptr;
  ncclResult_t (*GroupStart)() = nullptr;
  ncclResult_t (*GroupEnd)() = nullptr;
  const char *(*GetErrorString)(ncclResult_t) = nullptr;
};

NcclApi g_nccl;

int load_nccl(swim_sim *sim) {
  if (g_nccl.handle) return SWIM_OK;
  void *h = nullptr;
  if (const char *p = getenv("SWIM_NCCL_LIB")) h = dlopen(p, RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_NOLOAD); // the copy torch already mapped
  if (!h) h = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
  if (!h) h = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
  if (!h) { set_error(sim, "cannot load libnccl.so.2: %s", dlerror()); return SWIM_ENCCL; }
#define BIND(field, name)                                                            \
  *(void **)(&g_nccl.field) = dlsym(h, name);                                        \
  if (!g_nccl.field) { set_error(sim, "libnccl lacks %s", name); return SWIM_ENCCL; }
  BIND(GetUniqueId, "ncclGetUniqueId");
  BIND(CommInitRank, "ncclCommInitRank");
  BIND(CommDestroy, "ncclCommDestroy");
  BIND(AllGather, "ncclAllGather");
  BIND(Send, "ncclSend");
  BIND(Recv, "ncclRecv");
  BIND(GroupStart, "ncclGroupStart");
  BIND(GroupEnd, "ncclGroupEnd");
  BIND(GetErrorString, "ncclGetErrorString");
#undef BIND
  g_nccl.handle = h;
  return SWIM_OK;
}

#define NCCL_TRY(sim, call)                                                                          \
  do {                                                                                               \
    ncclResult_t r_ = (call);                                                                        \
    if (r_ != ncclSuccess) {                                                                         \
      set_error(sim, "%s failed: %s (%s:%d)", #call, g_nccl.GetErrorString(r_), __FILE__, __LINE__); \
      return SWIM_ENCCL;                                                                             \
    }                                                                                                \
  } while (0)

struct Dist {
  ncclComm_t comm = nullptr;
  uint32_t *d_matrix = nullptr; // [world][world+1] all-gathered bucket counts (+ overflow flags)
  uint32_t *h_matrix = nullptr; // pinned
  size_t xrecv_cap = 0;         // envelopes
};

// Received envelopes -> in-edge flags + per-source receiver lists. One thread per envelope; the
// position of an envelope inside its source's block is its slot in that source's list, so no atomics.
struct DeliverArgs {
  uint32_t off[SWIM_MAX_WORLD + 1]; // prefix offsets of the source ranks' blocks inside xrecv
};

__global__ void deliver_kernel(SimDev d, DeliverArgs a, uint32_t total) {
  const uint32_t par = d.round & 1;
  if (blockIdx.x == 0 && threadIdx.x < d.world)
    d.rcnt[par * d.world + threadIdx.x] = a.off[threadIdx.x + 1] - a.off[threadIdx.x];
  for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < total; k += gridDim.x * blockDim.x) {
    const uint4 hdr = d.xrecv[(size_t)k * (1 + d.B)]; // {in-edge index, count, sender id, receiver (local)}
    uint32_t src = 0;
    while (k >= a.off[src + 1]) ++src;
    d.eflag[(size_t)par * d.estride + hdr.x] = 2;
    d.eslot[hdr.x] = k;
    d.rlr[((size_t)par * d.world + src) * d.rcap + (k - a.off[src])] = hdr.w;
  }
}

} // namespace

extern "C" int swim_nccl_unique_id(uint8_t *id) {
  if (!id) return SWIM_EINVAL;
  int rc = load_nccl(nullptr);
  if (rc) return rc;
  static_assert(sizeof(ncclUniqueId) <= SWIM_NCCL_ID_BYTES, "id buffer too small");
  ncclUniqueId u;
  NCCL_TRY(nullptr, g_nccl.GetUniqueId(&u));
  memset(id, 0, SWIM_NCCL_ID_BYTES);
  memcpy(id, &u, sizeof u);
  return SWIM_OK;
}

extern "C" int swim_sim_connect(swim_sim_t *sim, const uint8_t *id) {
  if (!sim || !id) return SWIM_EINVAL;
  SimDev &d = sim->dev;
  if (d.world == 1) { sim->connected = true; return SWIM_OK; }
  if (sim->connected) return SWIM_OK;
  int rc = load_nccl(sim);
  if (rc) return rc;
  cudaSetDevice(sim->device);
  Dist *x = new Dist();
  sim->dist = x;
  ncclUniqueId u;
  memcpy(&u, id, sizeof u);
  NCCL_TRY(sim, g_nccl.CommInitRank(&x->comm, (int)d.world, u, (int)d.rank));
  // bucket capacity: twice the expected densest round (every local node sends `fanout` envelopes,
  // receivers spread evenly over the shards) plus slack; an overflow is reported, never silent
  const size_t per_bucket = 2 * ((size_t)d.n * d.fanout / d.world) + 4096;
  d.xcap = (uint32_t)per_bucket;
  const size_t env = 1 + d.B;
  x->xrecv_cap = per_bucket * (d.world - 1);
  CUDA_TRY(sim, cudaMalloc((void **)&d.xsend, per_bucket * d.world * env * sizeof(uint4)));
  CUDA_TRY(sim, cudaMalloc((void **)&d.xrecv, x->xrecv_cap * env * sizeof(uint4)));
  CUDA_TRY(sim, cudaMalloc((void **)&d.xsend_cnt, (d.world + 1) * sizeof(uint32_t)));
  CUDA_TRY(sim, cudaMemset(d.xsend_cnt, 0, (d.world + 1) * sizeof(uint32_t)));
  CUDA_TRY(sim, cudaMalloc((void **)&x->d_matrix, (size_t)d.world * (d.world + 1) * sizeof(uint32_t)));
  CUDA_TRY(sim, cudaMallocHost((void **)&x->h_matrix, (size_t)d.world * (d.world + 1) * sizeof(uint32_t)));
  sim->allocs.push_back(d.xsend);
  sim->allocs.push_back(d.xrecv);
  sim->allocs.push_back(d.xsend_cnt);
  sim->allocs.push_back(x->d_matrix);
  sim->connected = true;
  return SWIM_OK;
}

// ------------------------------------------------------------------ fused exchange over peer memory
namespace {
// Arrays a rank exports: the round kernels' (eflag .. mailbits) and what the collectives between steps read (nbr .. coll).
// None of them changes size with the view: eflag is the only view-sized array a peer maps, and a sharded rebuild re-maps
// it (coll_remap_eflag); out, out_cnt, rlr, rcnt, bar and mailbits are sized from `per` / `rcap`, nbr, vst, vinc and
// self_inc from the shard's rows.
enum { kXEflag, kXOut, kXOutCnt, kXRlr, kXRcnt, kXBar, kXMailbits, kXNbr, kXVst, kXVinc, kXSelfInc, kXColl, kXCount };
struct IpcBlob {
  uint32_t magic, rank, n, estride;
  cudaIpcMemHandle_t h[kXCount];
  // the exporting process and its raw device pointers: ranks that live in ONE process (several handles, on one device or
  // on peer devices) cannot open each other's IPC handles — they use the pointers as they are
  uint64_t pid;
  int32_t device, _pad;
  uint64_t raw[kXCount];
};
static_assert(sizeof(IpcBlob) <= SWIM_IPC_BLOB_BYTES, "blob too small");
constexpr uint32_t kBlobMagic = 0x53574D4Au; // "SWMJ"
} // namespace

extern "C" int swim_sim_ipc_export(swim_sim_t *sim, uint8_t *blob) {
  if (!sim || !blob) return SWIM_EINVAL;
  if (!sim->view_set) { set_error(sim, "swim_sim_ipc_export: install the view first (swim_sim_set_view)"); return SWIM_ESTATE; }
  cudaSetDevice(sim->device);
  SimDev &d = sim->dev;
  IpcBlob b;
  memset(&b, 0, sizeof b);
  b.magic = kBlobMagic; b.rank = d.rank; b.n = d.n; b.estride = d.estride;
  void *ptrs[kXCount] = {d.eflag, d.out, d.out_cnt, d.rlr, d.rcnt, sim->d_bar, d.mailbits,
                         d.nbr, d.vst, d.vinc, d.self_inc, sim->d_coll};
  for (int x = 0; x < kXCount; ++x) {
    CUDA_TRY(sim, cudaIpcGetMemHandle(&b.h[x], ptrs[x]));
    b.raw[x] = (uint64_t)(uintptr_t)ptrs[x];
  }
  b.pid = (uint64_t)getpid();
  b.device = sim->device;
  memset(blob, 0, SWIM_IPC_BLOB_BYTES);
  memcpy(blob, &b, sizeof b);
  return SWIM_OK;
}

extern "C" int swim_sim_ipc_connect(swim_sim_t *sim, const uint8_t *blobs) {
  if (!sim || !blobs) return SWIM_EINVAL;
  SimDev &d = sim->dev;
  if (d.world == 1) { sim->connected = true; return SWIM_OK; }
  if (d.p2p) return SWIM_OK;
  cudaSetDevice(sim->device);
  for (uint32_t r = 0; r < d.world; ++r) {
    IpcBlob b;
    memcpy(&b, blobs + (size_t)r * SWIM_IPC_BLOB_BYTES, sizeof b);
    if (b.magic != kBlobMagic || b.rank != r) { set_error(sim, "swim_sim_ipc_connect: blob %u is not rank %u's export", r, r); return SWIM_EINVAL; }
    if (r == d.rank) continue;
    void *p[kXCount];
    sim->peer.same_process[r] = b.pid == (uint64_t)getpid();
    if (sim->peer.same_process[r]) { // a rank of this very process: its pointers are valid here as they are
      if (b.device != sim->device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(b.device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) { set_error(sim, "swim_sim_ipc_connect: no peer access to device %d: %s", b.device, cudaGetErrorString(e)); return SWIM_ECUDA; }
        cudaGetLastError();
      }
      for (int x = 0; x < kXCount; ++x) p[x] = (void *)(uintptr_t)b.raw[x];
    } else {
      for (int x = 0; x < kXCount; ++x) {
        CUDA_TRY(sim, cudaIpcOpenMemHandle(&p[x], b.h[x], cudaIpcMemLazyEnablePeerAccess));
        sim->ipc_opened.push_back(p[x]);
      }
    }
    d.eflag_p[r] = (uint8_t *)p[kXEflag]; d.estride_p[r] = b.estride;
    d.out_p[r] = (const uint4 *)p[kXOut]; d.out_cnt_p[r] = (const uint8_t *)p[kXOutCnt];
    d.rlr_p[r] = (uint32_t *)p[kXRlr]; d.rcnt_p[r] = (uint32_t *)p[kXRcnt]; d.bar_p[r] = (uint32_t *)p[kXBar];
    d.mailbits_p[r] = (uint32_t *)p[kXMailbits];
    PeerViews &v = sim->peer;
    v.nbr[r] = (const uint32_t *)p[kXNbr]; v.vst[r] = (const uint8_t *)p[kXVst]; v.vinc[r] = (const uint32_t *)p[kXVinc];
    v.self_inc[r] = (const uint32_t *)p[kXSelfInc]; v.coll[r] = (CollBlock *)p[kXColl];
  }
  d.p2p = 1;
  sim->connected = true;
  return SWIM_OK;
}

namespace swim {

void refresh_peer_tables(swim_sim *sim) { // entry [rank] always aliases this rank's own arrays
  SimDev &d = sim->dev;
  const uint32_t r = d.rank;
  d.eflag_p[r] = d.eflag; d.estride_p[r] = d.estride; d.out_p[r] = d.out; d.out_cnt_p[r] = d.out_cnt;
  d.rlr_p[r] = d.rlr; d.rcnt_p[r] = d.rcnt; d.bar_p[r] = sim->d_bar; d.mailbits_p[r] = d.mailbits;
}

int dist_alloc_edges(swim_sim *sim) { // eslot follows the in-edge count
  SimDev &d = sim->dev;
  if (d.world == 1) return SWIM_OK;
  if (sim->d_eslot) { cudaFree(sim->d_eslot); sim->d_eslot = nullptr; }
  CUDA_TRY(sim, cudaMalloc((void **)&sim->d_eslot, (sim->n_edges ? sim->n_edges : 1) * sizeof(uint32_t)));
  d.eslot = sim->d_eslot;
  return SWIM_OK;
}

int dist_exchange(swim_sim *sim) {
  SimDev &d = sim->dev;
  Dist *x = (Dist *)sim->dist;
  if (!x) { set_error(sim, "multi-shard exchange not connected"); return SWIM_ESTATE; }
  const uint32_t G = d.world, row = G + 1;
  // 1. everybody learns everybody's bucket counts
  NCCL_TRY(sim, g_nccl.AllGather(d.xsend_cnt, x->d_matrix, row, ncclUint32, x->comm, sim->stream));
  CUDA_TRY(sim, cudaMemcpyAsync(x->h_matrix, x->d_matrix, (size_t)G * row * sizeof(uint32_t), cudaMemcpyDeviceToHost, sim->stream));
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  for (uint32_t a = 0; a < G; ++a)
    if (x->h_matrix[a * row + G]) {
      set_error(sim, "round %u: rank %u overflowed an exchange bucket (capacity %u envelopes)", d.round, a, d.xcap);
      return SWIM_ECAP;
    }
  // 2. move exactly the filled part of every bucket
  const size_t env_bytes = (size_t)(1 + d.B) * sizeof(uint4);
  size_t total_recv = 0, any = 0;
  DeliverArgs da;
  memset(&da, 0, sizeof da);
  for (uint32_t a = 0; a < G; ++a)
    for (uint32_t b = 0; b < G; ++b) any += x->h_matrix[a * row + b];
  if (any) {
    NCCL_TRY(sim, g_nccl.GroupStart());
    for (uint32_t p = 0; p < G; ++p) {
      if (p == d.rank) continue;
      const uint32_t n_send = x->h_matrix[d.rank * row + p], n_recv = x->h_matrix[p * row + d.rank];
      if (n_send)
        NCCL_TRY(sim, g_nccl.Send((const uint8_t *)d.xsend + (size_t)p * d.xcap * env_bytes, n_send * env_bytes, ncclUint8, (int)p, x->comm, sim->stream));
      if (n_recv) {
        if (total_recv + n_recv > x->xrecv_cap || n_recv > d.rcap) { g_nccl.GroupEnd(); set_error(sim, "exchange receive buffer overflow"); return SWIM_ECAP; }
        NCCL_TRY(sim, g_nccl.Recv((uint8_t *)d.xrecv + total_recv * env_bytes, n_recv * env_bytes, ncclUint8, (int)p, x->comm, sim->stream));
        total_recv += n_recv;
      }
      da.off[p + 1] = (uint32_t)total_recv;
    }
    NCCL_TRY(sim, g_nccl.GroupEnd());
    CUDA_TRY(sim, cudaMemsetAsync(d.xsend_cnt, 0, row * sizeof(uint32_t), sim->stream));
  }
  for (uint32_t p = 0; p < G; ++p) // ranks skipped above (self, or nothing exchanged at all) keep their prefix
    if (da.off[p + 1] < da.off[p]) da.off[p + 1] = da.off[p];
  // always launched: it also publishes this round's per-source counts (zeros when nothing arrived)
  const int grid = (int)std::max<size_t>(1, std::min<size_t>((total_recv + 255) / 256, (size_t)sim->sm_count * 8));
  SWIM_LAUNCH(deliver_kernel, grid, 256, sim->stream, d, da, (uint32_t)total_recv);
  ++sim->launches;
  return SWIM_OK;
}

} // namespace swim

// ------------------------------------------------------------------ collectives between steps
// The sharded forms of the bulk membership calls and of the mail-graph rebuild (swim_graph.cuh, swim_pushpull.cuh) need
// three things from the peers while no round runs: a barrier, which may carry one value per rank and return their sum; a
// gather of one per-row array into a [world x per]-row buffer (rank r's rows from row r * per on, so the buffer is
// addressed by global id and only its tail past N is padding); and, after a rebuild reallocated the mail flags, the
// peers' new flag arrays. Over peer memory they use the arrays swim_sim_ipc_connect mapped and a barrier word of their
// own (never the round kernels' words, whose handshake state must stay as it is); on the staged path, NCCL.
namespace {
struct CollPeers {
  CollBlock *b[SWIM_MAX_WORLD];
};

// Thread q stores this rank's value into peer q's block, then (release, system scope) this barrier's generation.
__global__ void coll_publish_kernel(uint32_t world, uint32_t rank, CollPeers p, uint32_t gen, unsigned long long val) {
  const uint32_t q = threadIdx.x;
  if (q < world && q != rank) {
    __threadfence_system(); // this rank's writes before the barrier (its earlier kernels and copies) come first
    p.b[q]->val[gen & 1][rank] = val;
    st_release_sys(&p.b[q]->bar[rank], gen);
  }
}

// Thread q reads (acquire) peer q's generation word in this rank's block and the value q brought with it.
__global__ void coll_poll_kernel(uint32_t world, uint32_t rank, CollBlock *mine, uint32_t gen) {
  const uint32_t q = threadIdx.x;
  if (q < world && q != rank) {
    const uint32_t g = ld_acquire_sys(&mine->bar[q]);
    mine->seen[q] = g;
    if ((int32_t)(g - gen) >= 0) mine->got[q] = *(volatile unsigned long long *)&mine->val[gen & 1][q];
  }
}

// The wait of a barrier over peer memory is the host's, one short poll kernel at a time, and not a kernel spinning on
// the device: ranks that share a device would otherwise dead-lock whenever one of them calls cudaFree (which waits for
// every kernel on the device, the peer's spinning barrier included) before it reaches the barrier. The wait is bounded
// like the round handshake's (about a minute).
constexpr double kCollWaitSeconds = 60.0;
} // namespace

namespace swim {

int coll_barrier(swim_sim *sim, unsigned long long mine, unsigned long long *sum) {
  SimDev &d = sim->dev;
  const uint32_t G = d.world;
  unsigned long long got[SWIM_MAX_WORLD];
  unsigned long long *d_got = (unsigned long long *)((uint8_t *)sim->d_coll + offsetof(CollBlock, got));
  const uint32_t gen = ++sim->coll_gen;
  if (d.p2p) {
    CollPeers p;
    memset(&p, 0, sizeof p);
    for (uint32_t q = 0; q < G; ++q) p.b[q] = sim->peer.coll[q];
    SWIM_LAUNCH(coll_publish_kernel, 1, 32, sim->stream, G, d.rank, p, gen, mine);
    ++sim->launches;
    CUDA_TRY(sim, cudaGetLastError());
    const uint32_t *d_seen = (const uint32_t *)((const uint8_t *)sim->d_coll + offsetof(CollBlock, seen));
    const auto t0 = std::chrono::steady_clock::now();
    for (int poll = 0;; ++poll) {
      uint32_t seen[SWIM_MAX_WORLD];
      SWIM_LAUNCH(coll_poll_kernel, 1, 32, sim->stream, G, d.rank, sim->d_coll, gen);
      ++sim->launches;
      CUDA_TRY(sim, cudaGetLastError());
      CUDA_TRY(sim, cudaMemcpyAsync(seen, d_seen, G * sizeof(uint32_t), cudaMemcpyDeviceToHost, sim->stream));
      CUDA_TRY(sim, cudaMemcpyAsync(got, d_got, G * sizeof(unsigned long long), cudaMemcpyDeviceToHost, sim->stream));
      CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
      bool all = true;
      for (uint32_t q = 0; q < G; ++q) all &= q == d.rank || (int32_t)(seen[q] - gen) >= 0;
      if (all) break;
      if (std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count() > kCollWaitSeconds) {
        set_error(sim, "a barrier between steps timed out (a peer rank did not make the same call)");
        sim->failed = true;
        return SWIM_ESTATE;
      }
      if (poll >= 16) std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
  } else { // staged path: a one-word all-gather is the barrier
    Dist *x = (Dist *)sim->dist;
    if (!x) { set_error(sim, "multi-shard exchange not connected"); return SWIM_ESTATE; }
    unsigned long long *w = d_got;
    CUDA_TRY(sim, cudaMemcpyAsync(w + d.rank, &mine, sizeof mine, cudaMemcpyHostToDevice, sim->stream));
    NCCL_TRY(sim, g_nccl.AllGather(w + d.rank, w, 1, ncclUint64, x->comm, sim->stream));
    CUDA_TRY(sim, cudaMemcpyAsync(got, w, G * sizeof(unsigned long long), cudaMemcpyDeviceToHost, sim->stream));
    CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  }
  got[d.rank] = mine;
  if (sum) {
    *sum = 0;
    for (uint32_t q = 0; q < G; ++q) *sum += got[q];
  }
  return SWIM_OK;
}

int coll_gather(swim_sim *sim, CollArray which, void *out) {
  SimDev &d = sim->dev;
  const size_t rb = which == kCollNbr || which == kCollVinc ? (size_t)d.cap * 4 : which == kCollVst ? d.cap : 4;
  const void *local = which == kCollNbr ? (const void *)d.nbr : which == kCollVst ? (const void *)d.vst
                    : which == kCollVinc ? (const void *)d.vinc : (const void *)d.self_inc;
  uint8_t *o = (uint8_t *)out;
  if (d.n) CUDA_TRY(sim, cudaMemcpyAsync(o + (size_t)d.rank * d.per * rb, local, d.n * rb, cudaMemcpyDeviceToDevice, sim->stream));
  if (d.p2p) {
    const PeerViews &v = sim->peer;
    for (uint32_t r = 0; r < d.world; ++r) {
      const uint32_t f = shard_first(d.N, d.world, r), n = shard_first(d.N, d.world, r + 1) - f;
      if (r == d.rank || !n) continue;
      const void *src = which == kCollNbr ? (const void *)v.nbr[r] : which == kCollVst ? (const void *)v.vst[r]
                      : which == kCollVinc ? (const void *)v.vinc[r] : (const void *)v.self_inc[r];
      CUDA_TRY(sim, cudaMemcpyAsync(o + (size_t)r * d.per * rb, src, n * rb, cudaMemcpyDefault, sim->stream));
    }
  } else {
    Dist *x = (Dist *)sim->dist;
    if (!x) { set_error(sim, "multi-shard exchange not connected"); return SWIM_ESTATE; }
    const size_t part = (size_t)d.per * rb; // (in place: this rank's part of the buffer is its send buffer)
    NCCL_TRY(sim, g_nccl.AllGather(o + d.rank * part, o, part, ncclUint8, x->comm, sim->stream));
  }
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  return SWIM_OK;
}

// After a sharded rebuild over peer memory: every rank's mail flags live in a new array with a new parity stride. Each
// rank publishes its own in its block; after a barrier it maps every peer's (closing the old mapping); after a second
// barrier nobody holds the retired arrays any more, and each rank frees its own. A third barrier follows the free: no
// rank starts its round kernels (which wait for the peers on the device) while a peer that shares its device may still
// be in cudaFree (which waits for every kernel on the device).
int coll_remap_eflag(swim_sim *sim, uint8_t *retired) {
  SimDev &d = sim->dev;
  CollBlock pub;
  memset(&pub, 0, sizeof pub);
  CUDA_TRY(sim, cudaIpcGetMemHandle(&pub.eflag_h, d.eflag));
  pub.eflag_raw = (unsigned long long)(uintptr_t)d.eflag;
  pub.estride = d.estride;
  const size_t off = offsetof(CollBlock, eflag_h), bytes = sizeof(CollBlock) - off;
  CUDA_TRY(sim, cudaMemcpyAsync((uint8_t *)sim->d_coll + off, (const uint8_t *)&pub + off, bytes, cudaMemcpyHostToDevice, sim->stream));
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  int rc;
  if ((rc = coll_barrier(sim))) return rc;
  for (uint32_t r = 0; r < d.world; ++r) {
    if (r == d.rank) continue;
    CollBlock b;
    CUDA_TRY(sim, cudaMemcpy((uint8_t *)&b + off, (const uint8_t *)sim->peer.coll[r] + off, bytes, cudaMemcpyDefault));
    void *p = (void *)(uintptr_t)b.eflag_raw;
    if (!sim->peer.same_process[r]) {
      auto it = std::find(sim->ipc_opened.begin(), sim->ipc_opened.end(), (void *)d.eflag_p[r]);
      if (it != sim->ipc_opened.end()) { cudaIpcCloseMemHandle(*it); sim->ipc_opened.erase(it); }
      CUDA_TRY(sim, cudaIpcOpenMemHandle(&p, b.eflag_h, cudaIpcMemLazyEnablePeerAccess));
      sim->ipc_opened.push_back(p);
    }
    d.eflag_p[r] = (uint8_t *)p;
    d.estride_p[r] = b.estride;
  }
  if ((rc = coll_barrier(sim))) return rc;
  if (retired) CUDA_TRY(sim, cudaFree(retired));
  return coll_barrier(sim);
}

void dist_teardown(swim_sim *sim) {
  for (void *p : sim->ipc_opened) cudaIpcCloseMemHandle(p);
  sim->ipc_opened.clear();
  Dist *x = (Dist *)sim->dist;
  if (!x) return;
  if (x->comm && g_nccl.CommDestroy) g_nccl.CommDestroy(x->comm);
  if (x->h_matrix) cudaFreeHost(x->h_matrix);
  delete x;
  sim->dist = nullptr;
}

} // namespace swim
