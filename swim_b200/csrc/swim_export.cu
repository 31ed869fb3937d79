// swim_export.cu — simulated traffic <-> real datagrams (SURVEY §8(f)-2), host side.
//
// Export: the envelopes K1b sent in the last round (sender snapshots `out`, recipients in the candidate
// slots `rl`) are copied to the host and encoded with the reference's wire format by the codec of
// swim_codec.cpp — what `disseminate` would hand to `UDP.sinkToSocket` (Core.hs:127-138,286) if the
// reference had its piggyback queue. Import: a captured datagram becomes SWIM_EV_INJECT events.
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
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

void wire_of_record(const swim_sim *sim, const swim_record_t &r, swim_wire_message_t *w) {
  memset(w, 0, sizeof *w);
  w->kind = r.kind;
  w->incarnation = r.incarnation;
  snprintf(w->node, sizeof w->node, "n%u", r.member);
  if (r.kind == SWIM_MSG_DEAD) snprintf(w->dead_from, sizeof w->dead_from, "n%u", r.from);
  if (r.kind == SWIM_MSG_ALIVE) { w->target = r.member; w->port = (uint16_t)sim->cfg.base_port; }
}

// "n<decimal>" -> id; false if the name is not of that form
bool id_of_name(const char *s, uint32_t n_nodes, uint32_t *id) {
  if (s[0] != 'n' || s[1] == 0) return false;
  char *end = nullptr;
  unsigned long v = strtoul(s + 1, &end, 10);
  if (*end != 0 || v >= n_nodes) return false;
  *id = (uint32_t)v;
  return true;
}

} // namespace

extern "C" int swim_sim_export_round(swim_sim_t *sim, uint8_t *buf, size_t cap, swim_datagram_t *index, size_t index_cap,
                                     size_t *n_datagrams, size_t *n_bytes) {
  if (!sim || !n_datagrams || !n_bytes) return SWIM_EINVAL;
  const SimDev &d = sim->dev;
  if (d.world != 1) { set_error(sim, "swim_sim_export_round: single shard only"); return SWIM_ESTATE; }
  if (sim->rows_edited) { set_error(sim, "swim_sim_export_round: memberships were edited since the last step"); return SWIM_ESTATE; }
  *n_datagrams = 0;
  *n_bytes = 0;
  if (sim->round == 0) return SWIM_OK;
  cudaSetDevice(sim->device);
  CUDA_TRY(sim, cudaStreamSynchronize(sim->stream));
  const uint32_t round = sim->round, par = round & 1, slot3 = round % 3;
  uint32_t n_work = 0;
  CUDA_TRY(sim, cudaMemcpy(&n_work, d.wl_cnt + slot3, 4, cudaMemcpyDeviceToHost));
  if (n_work == 0) return SWIM_OK;
  const uint32_t F = d.fanout, B = d.B;
  std::vector<uint32_t> wl(n_work), rl((size_t)n_work * F);
  CUDA_TRY(sim, cudaMemcpy(wl.data(), d.wl + (size_t)par * d.n, (size_t)n_work * 4, cudaMemcpyDeviceToHost));
  {
    // recipient slots {receiver | bit 31 = dropped at the sender (it still went on the wire), sender}
    std::vector<uint2> slots((size_t)n_work * F);
    CUDA_TRY(sim, cudaMemcpy(slots.data(), d.rl + (size_t)par * d.n * F, slots.size() * sizeof(uint2), cudaMemcpyDeviceToHost));
    for (size_t x = 0; x < slots.size(); ++x) rl[x] = slots[x].x == 0xFFFFFFFFu ? 0xFFFFFFFFu : (slots[x].x & 0x7FFFFFFFu);
  }
  // sender snapshots: gather only the listed senders
  std::vector<uint8_t> cnt(n_work);
  std::vector<swim_record_t> recs((size_t)n_work * B);
  {
    std::vector<uint8_t> all_cnt(d.n);
    CUDA_TRY(sim, cudaMemcpy(all_cnt.data(), d.out_cnt + (size_t)par * d.per, d.n, cudaMemcpyDeviceToHost));
    for (uint32_t k = 0; k < n_work; ++k) cnt[k] = all_cnt[wl[k]];
    for (uint32_t k = 0; k < n_work; ++k) {
      bool sends = false;
      for (uint32_t f = 0; f < F; ++f) sends |= rl[(size_t)k * F + f] != 0xFFFFFFFFu;
      if (!sends) { cnt[k] = 0; continue; }
      CUDA_TRY(sim, cudaMemcpy(&recs[(size_t)k * B], d.out + ((size_t)par * d.per + wl[k]) * B, cnt[k] * sizeof(swim_record_t),
                               cudaMemcpyDeviceToHost));
    }
  }
  // encode one envelope per sender (its recipients all get the same bytes)
  std::vector<std::string> enc(n_work);
  int bad = 0;
#pragma omp parallel for schedule(dynamic, 64)
  for (int64_t k = 0; k < (int64_t)n_work; ++k) {
    if (!cnt[k]) continue;
    std::vector<swim_wire_message_t> msgs(cnt[k]);
    for (uint32_t q = 0; q < cnt[k]; ++q) wire_of_record(sim, recs[(size_t)k * B + q], &msgs[q]);
    std::vector<uint8_t> tmp(8 + (size_t)cnt[k] * 96);
    size_t len = 0;
    if (swim_envelope_encode(msgs.data(), cnt[k], tmp.data(), tmp.size(), &len) != SWIM_OK) {
#pragma omp atomic write
      bad = 1;
      continue;
    }
    enc[k].assign((const char *)tmp.data(), len);
  }
  if (bad) { set_error(sim, "swim_sim_export_round: encoder failed"); return SWIM_EINVAL; }
  size_t nd = 0, nb = 0;
  for (uint32_t k = 0; k < n_work; ++k)
    for (uint32_t f = 0; f < F && cnt[k]; ++f) {
      const uint32_t dst = rl[(size_t)k * F + f];
      if (dst == 0xFFFFFFFFu) continue;
      if (index && nd < index_cap && buf && nb + enc[k].size() <= cap) {
        index[nd].src = d.first + wl[k];
        index[nd].dst = d.first + dst;
        index[nd].length = (uint32_t)enc[k].size();
        index[nd].n_messages = cnt[k];
        index[nd].offset = nb;
        memcpy(buf + nb, enc[k].data(), enc[k].size());
      }
      ++nd;
      nb += enc[k].size();
    }
  *n_datagrams = nd;
  *n_bytes = nb;
  if ((index && nd > index_cap) || (buf && nb > cap)) { set_error(sim, "swim_sim_export_round: %zu datagrams / %zu bytes do not fit", nd, nb); return SWIM_ECAP; }
  return SWIM_OK;
}

extern "C" int swim_sim_inject_datagram(swim_sim_t *sim, uint32_t round, uint32_t node, const uint8_t *data, size_t len) {
  if (!sim || !data) return SWIM_EINVAL;
  std::vector<swim_wire_message_t> msgs(255);
  size_t n = 0;
  int rc = swim_envelope_decode(data, len, msgs.data(), msgs.size(), &n);
  if (rc) { set_error(sim, "swim_sim_inject_datagram: %s", swim_last_error(nullptr)); return rc; }
  std::vector<swim_event_t> ev;
  for (size_t x = 0; x < n; ++x) {
    const swim_wire_message_t &w = msgs[x];
    if (w.kind != SWIM_MSG_SUSPECT && w.kind != SWIM_MSG_ALIVE && w.kind != SWIM_MSG_DEAD) continue; // no state in Ping/Ack
    swim_event_t e;
    memset(&e, 0, sizeof e);
    e.round = round; e.node = node; e.kind = SWIM_EV_INJECT;
    e.msg.kind = w.kind; e.msg.incarnation = w.incarnation; e.msg.target = w.target; e.msg.port = w.port;
    if (!id_of_name(w.node, sim->dev.N, &e.msg.node) ||
        (w.kind == SWIM_MSG_DEAD && !id_of_name(w.dead_from, sim->dev.N, &e.msg.dead_from))) {
      set_error(sim, "swim_sim_inject_datagram: name '%s' is not a simulated node (\"n<id>\")", w.node);
      return SWIM_EINVAL;
    }
    ev.push_back(e);
  }
  return ev.empty() ? SWIM_OK : swim_sim_inject(sim, ev.data(), ev.size());
}
