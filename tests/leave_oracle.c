/*
 * leave_oracle.c — the CPU oracle's graceful leaves (DESIGN.md §2.8). TEST INFRASTRUCTURE ONLY.
 *
 * Compiled together with oracle/swim_oracle.c (included below) into a library of its own, so that every record goes
 * through the oracle's own apply_record and pb_enqueue, exactly as run_events applies a SWIM_EV_INJECT datagram, on a
 * handle made by oracle/liboracle.so (same source, same struct layout). tests/leave_oracle.py builds and loads it.
 */
#include "../oracle/swim_oracle.c"

/* ------------------------------------------------------------------ graceful leaves (DESIGN.md §2.8)
 * memberlist's Leave: Dead about the departing process, from itself. The reference has no leave. Every id is checked
 * first (< N). The leavers are the distinct listed ids that are up. Each goes down as a CRASH at the current round does,
 * and back_at = 0. Then every node m in ascending id that is up, for every leaver L in ascending id whose row holds m
 * Alive or Suspect: Dead(self_inc_L, L, from L) through apply_record (no insert, net = 1) at the current round; a `Just`
 * is enqueued and counted in RECS_APPLIED. */
static int cmp_dir(const void *a, const void *b) {
  const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
  return x < y ? -1 : x > y;
}

EXPORT int oracle_leave(oracle_t *o, const uint32_t *ids, size_t np, uint64_t *n_left, uint64_t *n_delivered) {
  if (o->cfg.world != 1 || !o->view_set) return SWIM_ESTATE;
  for (size_t k = 0; k < np; ++k)
    if (ids[k] >= o->N) return SWIM_EINVAL;
  const uint32_t n = o->n, cap = o->cap;
  uint8_t *leaver = (uint8_t *)calloc(n, 1);
  uint64_t left = 0, delivered = 0;
  for (size_t k = 0; k < np; ++k)
    if (o->alive[ids[k]] && !leaver[ids[k]]) { leaver[ids[k]] = 1; ++left; }
  for (uint32_t L = 0; L < n; ++L)
    if (leaver[L]) { o->alive[L] = 0; o->last_crash[L] = o->round; o->back_at[L] = 0; }
  /* the (recipient m, leaver L) pairs, ordered by m, then L */
  uint64_t *dir = (uint64_t *)malloc(left * cap * 8 + 8);
  size_t nd = 0;
  for (uint32_t L = 0; L < n; ++L) {
    if (!leaver[L]) continue;
    for (uint32_t s = 0; s < cap; ++s) {
      const size_t x = (size_t)L * cap + s;
      if (o->state[x] != SWIM_ALIVE && o->state[x] != SWIM_SUSPECT) continue;
      if (o->alive[o->nbr[x]]) dir[nd++] = (uint64_t)o->nbr[x] << 32 | L;
    }
  }
  qsort(dir, nd, 8, cmp_dir);
  for (size_t x = 0; x < nd; ++x) {
    const uint32_t m = (uint32_t)(dir[x] >> 32), L = (uint32_t)dir[x];
    rec_t r = {L, o->self_inc[L], L, SWIM_MSG_DEAD, 0, 0}, rb;
    if (apply_record(o, m, r, 0, 1, &rb, NULL, o->ctr)) {
      pb_enqueue(o, m, rb, o->ctr);
      o->ctr[SWIM_CTR_RECS_APPLIED]++;
    }
    ++delivered;
  }
  free(leaver);
  free(dir);
  if (n_left) *n_left = left;
  if (n_delivered) *n_delivered = delivered;
  return SWIM_OK;
}
