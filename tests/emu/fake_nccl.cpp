// tests/emu/fake_nccl.cpp — TEST INFRASTRUCTURE. An in-process stand-in for the nine NCCL entry points that
// swim_b200/csrc/swim_dist.cu binds with dlopen/dlsym (SWIM_NCCL_LIB points at this library), so the STAGED exchange —
// bucket counts all-gathered, envelopes sent/received per peer, deliver_kernel — runs with the ranks as threads of one
// process. Semantics kept: collectives block until every rank of the communicator has called them; point-to-point
// operations issued between ncclGroupStart and ncclGroupEnd complete at ncclGroupEnd; sends are buffered.
//
// One source for two builds. On the SIMT emulator (tests/emu/build_emu.py) the buffers are host memory and the CUDA calls
// below are the emulator header's no-op / memmove. Against the real CUDA runtime (tests/nccl_fixtures.py) the buffers are
// device memory of ranks that share a GPU: the stand-in waits for the caller's stream before it reads a send buffer, and
// moves bytes through host staging with copies on that stream. It links its own copy of the runtime (statically, symbols
// hidden), so all it shares with the library is the primary context that the calling thread has current — through which
// the library's streams and device pointers are valid here too.
#include <cuda_runtime.h>
#include <nccl.h>

#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <cstring>
#include <deque>
#include <map>
#include <mutex>
#include <vector>

namespace {

struct Group {
  std::mutex m;
  std::condition_variable cv;
  int world = 0, joined = 0, left = 0;
  // all-gather
  std::vector<std::vector<uint8_t>> stage;
  int ag_arrived = 0, ag_done = 0;
  uint64_t ag_gen = 0;
  // buffered point-to-point messages: box[src * world + dst]
  std::vector<std::deque<std::vector<uint8_t>>> box;
};

struct Comm { Group *g; int rank; };

struct PendingRecv { void *dst; size_t bytes; int src; Comm *c; cudaStream_t stream; };

std::mutex g_reg_m;
std::map<uint64_t, Group *> g_groups;
std::atomic<uint64_t> g_next_id{0x5157494D00000001ull};
thread_local int tl_group_depth = 0;
thread_local std::vector<PendingRecv> tl_recvs;

// A copy between host staging and a buffer of the caller's, queued on the caller's stream and complete on return: a send
// buffer is read after the work queued before the call (which writes it), and a receive buffer is written before the
// work queued after it. (A plain cudaMemcpy would run on the legacy default stream, and from pageable memory it may
// return before its DMA has landed.)
bool copy(void *dst, const void *src, size_t n, cudaStream_t stream) {
  return cudaMemcpyAsync(dst, src, n, cudaMemcpyDefault, stream) == cudaSuccess && cudaStreamSynchronize(stream) == cudaSuccess;
}

size_t dtype_bytes(ncclDataType_t t) {
  switch ((int)t) {
    case 0: case 1: return 1;       // int8 / uint8
    case 2: case 3: return 4;       // int32 / uint32
    case 4: case 5: return 8;       // int64 / uint64
    case 6: return 2;               // half
    case 7: return 4;               // float
    case 8: return 8;               // double
    default: return 2;
  }
}

bool finish_recvs() {
  bool ok = true;
  for (PendingRecv &r : tl_recvs) {
    Group *g = r.c->g;
    std::unique_lock<std::mutex> lk(g->m);
    auto &q = g->box[(size_t)r.src * g->world + r.c->rank];
    g->cv.wait(lk, [&] { return !q.empty(); });
    std::vector<uint8_t> msg = std::move(q.front());
    q.pop_front();
    lk.unlock();
    ok &= copy(r.dst, msg.data(), msg.size() < r.bytes ? msg.size() : r.bytes, r.stream);
  }
  tl_recvs.clear();
  return ok;
}

} // namespace

#define API extern "C" __attribute__((visibility("default")))

API const char *ncclGetErrorString(ncclResult_t r) { return r == ncclSuccess ? "no error" : "fake NCCL error"; }

API ncclResult_t ncclGetUniqueId(ncclUniqueId *id) {
  memset(id, 0, sizeof *id);
  const uint64_t v = g_next_id.fetch_add(1);
  memcpy(id->internal, &v, sizeof v);
  return ncclSuccess;
}

API ncclResult_t ncclCommInitRank(ncclComm_t *comm, int nranks, ncclUniqueId id, int rank) {
  uint64_t key;
  memcpy(&key, id.internal, sizeof key);
  Group *g;
  {
    std::lock_guard<std::mutex> lk(g_reg_m);
    Group *&slot = g_groups[key];
    if (!slot) {
      slot = new Group();
      slot->world = nranks;
      slot->stage.resize(nranks);
      slot->box.resize((size_t)nranks * nranks);
    }
    g = slot;
  }
  {
    std::unique_lock<std::mutex> lk(g->m);
    ++g->joined;
    g->cv.notify_all();
    g->cv.wait(lk, [&] { return g->joined >= g->world; }); // a communicator exists once every rank has joined
  }
  *comm = reinterpret_cast<ncclComm_t>(new Comm{g, rank});
  return ncclSuccess;
}

API ncclResult_t ncclCommDestroy(ncclComm_t comm) {
  Comm *c = reinterpret_cast<Comm *>(comm);
  delete c; // the group itself stays registered: a handful of bytes per test
  return ncclSuccess;
}

API ncclResult_t ncclAllGather(const void *send, void *recv, size_t count, ncclDataType_t t, ncclComm_t comm, cudaStream_t stream) {
  Comm *c = reinterpret_cast<Comm *>(comm);
  Group *g = c->g;
  const size_t bytes = count * dtype_bytes(t);
  std::vector<uint8_t> mine(bytes); // read before the lock: the send buffer may be this rank's part of `recv` (in place)
  if (!copy(mine.data(), send, bytes, stream)) return ncclUnhandledCudaError;
  std::vector<uint8_t> all((size_t)g->world * bytes);
  {
    std::unique_lock<std::mutex> lk(g->m);
    g->cv.wait(lk, [&] { return g->ag_done == 0; }); // the previous all-gather has been read by everybody
    g->stage[c->rank] = std::move(mine);
    const uint64_t gen = g->ag_gen;
    if (++g->ag_arrived == g->world) { g->ag_arrived = 0; g->ag_done = g->world; ++g->ag_gen; g->cv.notify_all(); }
    else g->cv.wait(lk, [&] { return g->ag_gen != gen; });
    for (int r = 0; r < g->world; ++r) memcpy(all.data() + (size_t)r * bytes, g->stage[r].data(), bytes);
    if (--g->ag_done == 0) g->cv.notify_all();
  }
  return copy(recv, all.data(), all.size(), stream) ? ncclSuccess : ncclUnhandledCudaError;
}

API ncclResult_t ncclGroupStart() { ++tl_group_depth; return ncclSuccess; }

API ncclResult_t ncclGroupEnd() {
  if (tl_group_depth > 0 && --tl_group_depth == 0 && !finish_recvs()) return ncclUnhandledCudaError;
  return ncclSuccess;
}

API ncclResult_t ncclSend(const void *buf, size_t count, ncclDataType_t t, int peer, ncclComm_t comm, cudaStream_t stream) {
  Comm *c = reinterpret_cast<Comm *>(comm);
  Group *g = c->g;
  std::vector<uint8_t> msg(count * dtype_bytes(t));
  if (!copy(msg.data(), buf, msg.size(), stream)) return ncclUnhandledCudaError;
  {
    std::lock_guard<std::mutex> lk(g->m);
    g->box[(size_t)c->rank * g->world + peer].push_back(std::move(msg));
  }
  g->cv.notify_all();
  return ncclSuccess;
}

API ncclResult_t ncclRecv(void *buf, size_t count, ncclDataType_t t, int peer, ncclComm_t comm, cudaStream_t stream) {
  tl_recvs.push_back(PendingRecv{buf, count * dtype_bytes(t), peer, reinterpret_cast<Comm *>(comm), stream});
  if (tl_group_depth == 0 && !finish_recvs()) return ncclUnhandledCudaError;
  return ncclSuccess;
}
