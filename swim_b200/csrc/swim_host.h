// swim_host.h — the handle behind swim_sim_t (include/swim.h). Host-only bookkeeping plus the
// SimDev block of device pointers handed to every kernel by value.
#pragma once
#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "swim_device.cuh"

struct swim_sim {
  swim_config_t cfg{};
  swim::SimDev dev{};
  int device = 0;
  int sm_count = 148;
  cudaStream_t own_stream = nullptr;
  cudaStream_t stream = nullptr;
  cudaEvent_t ev_start = nullptr, ev_stop = nullptr;
  bool timed = false;
  uint32_t round = 0;
  bool view_set = false;
  bool edges_dirty = false; // scalar or bulk calls changed a row's membership: the mail graph is rebuilt by the next step
  bool rows_edited = false; // a bulk membership edit since the last step: the last round's envelopes no longer match the rows
  bool tdead_dirty = true;  // crashed-member bitmaps must be rebuilt from alive[]
  bool connected = false;   // multi-shard exchange ready
  uint64_t n_edges = 0;
  uint64_t scalar_calls = 0;
  std::vector<void *> allocs;
  uint32_t *d_in_src = nullptr;
  uint8_t *d_eflag = nullptr;
  uint32_t *d_bloom = nullptr; // membership filters of all N rows (rebuilt with the in-edge index)
  uint32_t *d_eslot = nullptr; // exchange-buffer slot per in-edge (world > 1)
  void *d_events = nullptr;
  size_t d_events_cap = 0;
  void *h_events = nullptr;          // pinned staging of the events of one swim_sim_step call (no pageable copies,
  size_t h_events_cap = 0;           //   no synchronisation inside the call)
  cudaEvent_t ev_upload = nullptr;   // recorded after the staging buffer's copy: it may be rewritten once this fired
  bool failed = false;               // a launch failed part-way through a step: the device state is undefined
  // device-resident checkpoint (swim_sim_save / swim_sim_load): one slot per handle
  std::vector<std::pair<void *, size_t>> ckpt_arrays; // (copy, bytes) in the order of ckpt_sources()
  uint32_t ckpt_round = 0;
  uint64_t view_epoch = 0, ckpt_epoch = 0; // build_graph (swim_graph.cuh) counts views; a checkpoint belongs to one
  bool ckpt_valid = false;
  std::vector<swim_event_t> ckpt_events;
  unsigned long long *d_scratch = nullptr;
  void *d_sargs = nullptr; // scalar-call argument block (swim_scalar.cu)
  std::vector<swim_event_t> events; // pending, sorted by round (stable)
  std::string last_error;
  int grids[6] = {0, 0, 0, 0, 0, 0}; // one-wave grid sizes of the per-round kernels (filled on first use)
  uint64_t launches = 0;
  bool profile = false;
  // launch-path switches, read from the environment once per handle (swim_sim_create), not once per call
  bool opt_split = false, opt_round_kernel = true, opt_one_round = false;
  int opt_xmode = -1;                // round_kernel_x (one grid barrier per round): -1 auto (long single-shard launches), 1 always, 0 never
  uint32_t opt_quiet_batch = 4;
  std::vector<cudaEvent_t> prof_events; // pool, reused
  std::vector<std::pair<int, int>> prof_marks; // (phase, index of start event); stop = start + 1
  size_t prof_used = 0;
  double prof_ms[SWIM_PROFILE_SLOTS] = {0, 0, 0, 0, 0, 0};
  uint32_t *d_bar = nullptr;     // [world] cross-GPU barrier words of this rank
  uint32_t *h_bar_err = nullptr;            // pinned + device-mapped watchdog word of the in-kernel waits
  unsigned long long *h_observe = nullptr;  // pinned staging of swim_sim_observe
  // swim_sim_step_observe: results written by the device into mapped pinned memory [counters, mismatches, watchdog, seq]
  unsigned long long *h_obs = nullptr, *d_obs = nullptr, *d_obs_acc = nullptr;
  uint32_t *d_obs_done = nullptr;
  unsigned long long obs_seq = 0;
  uint32_t churn_last_round = 0xFFFFFFF0u; // last round churn_kernel ran for (its list counter has round-parity slots)
  std::vector<void *> ipc_opened; // peer mappings to close
  void *dist = nullptr; // multi-GPU exchange state (swim_dist.cu)
};

namespace swim {
void set_error(swim_sim *sim, const char *fmt, ...);
uint32_t shard_first(uint32_t N, uint32_t world, uint32_t rank);
int rebuild_edges_from_device(swim_sim *sim);
int dist_exchange(swim_sim *sim);
int dist_alloc_edges(swim_sim *sim);
void refresh_peer_tables(swim_sim *sim);
int prof_begin(swim_sim *sim, int phase);
void prof_end(swim_sim *sim, int mark);
int prof_collect(swim_sim *sim);
void dist_teardown(swim_sim *sim);
} // namespace swim
