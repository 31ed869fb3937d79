/*
 * join_oracle.c — the CPU oracle's seed joins (DESIGN.md §2.7). TEST INFRASTRUCTURE ONLY.
 *
 * Built like tests/push_pull_oracle.c, which it includes (and with it oracle/swim_oracle.c): the merge of one sender's
 * state into one receiver is push-pull's pp_merge, so every record goes through the oracle's own apply_record and
 * pb_enqueue on a handle made by oracle/liboracle.so (same source, same struct layout). tests/join_oracle.py builds and
 * loads it.
 */
#include "push_pull_oracle.c"

/* ------------------------------------------------------------------ seed joins (DESIGN.md §2.7)
 * memberlist's Join(joinHosts); the reference parses Config.joinHosts (Types.hs:47, Util.hs:46) and never joins. Every
 * pair is checked first (ids < N, node != seed). With SWIM_JOIN_FRESH every listed joiner that is up loses its row and
 * its piggyback buffer. Then a snapshot, and each pair (j, s) with both up is an exchange: j receives s's state and s
 * receives j's. A receiver merges its distinct senders in ascending id, each once, through pp_merge. */
static int cmp_u64(const void *a, const void *b) {
  const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
  return x < y ? -1 : x > y;
}

EXPORT int oracle_join(oracle_t *o, const uint32_t *node, const uint32_t *seed, size_t np, uint32_t flags,
                       uint64_t *n_exchanges, uint64_t *n_inserted, uint64_t *n_full) {
  if (o->cfg.world != 1 || !o->view_set) return SWIM_ESTATE;
  for (size_t k = 0; k < np; ++k)
    if (node[k] >= o->N || seed[k] >= o->N || node[k] == seed[k]) return SWIM_EINVAL;
  const uint32_t n = o->n, cap = o->cap;
  const size_t slots = (size_t)n * cap;
  if (flags & SWIM_JOIN_FRESH)
    for (size_t k = 0; k < np; ++k) {
      const uint32_t j = node[k];
      if (!o->alive[j]) continue;
      for (uint32_t s = 0; s < cap; ++s) {
        const size_t x = (size_t)j * cap + s;
        o->nbr[x] = SWIM_NO_MEMBER; o->state[x] = SWIM_VACANT; o->timer[x] = 0; o->conf[x] = 0; o->vinc[x] = 0; o->vlast[x] = 0;
      }
      memset(o->pb + (size_t)j * o->B, 0, o->B * sizeof(rec_t));
      o->pb_cnt[j] = 0;
    }
  uint32_t *s_ids = (uint32_t *)malloc(slots * 4), *s_inc = (uint32_t *)malloc(slots * 4);
  uint32_t *s_self = (uint32_t *)malloc((size_t)n * 4);
  uint8_t *s_st = (uint8_t *)malloc(slots);
  uint64_t *dir = (uint64_t *)malloc(2 * np * 8 + 8); /* receiver << 32 | sender */
  memcpy(s_ids, o->nbr, slots * 4);
  memcpy(s_inc, o->vinc, slots * 4);
  memcpy(s_st, o->state, slots);
  memcpy(s_self, o->self_inc, (size_t)n * 4);
  uint64_t ex = 0, ins = 0, full = 0;
  size_t nd = 0;
  for (size_t k = 0; k < np; ++k) {
    if (!o->alive[node[k]] || !o->alive[seed[k]]) continue;
    ++ex;
    dir[nd++] = (uint64_t)node[k] << 32 | seed[k];
    dir[nd++] = (uint64_t)seed[k] << 32 | node[k];
  }
  qsort(dir, nd, 8, cmp_u64);
  for (size_t x = 0; x < nd; ++x)
    if (x == 0 || dir[x] != dir[x - 1])
      pp_merge(o, (uint32_t)(dir[x] >> 32), (uint32_t)dir[x], s_ids, s_st, s_inc, s_self, o->ctr, &ins, &full);
  free(s_ids); free(s_inc); free(s_self); free(s_st); free(dir);
  if (n_exchanges) *n_exchanges = ex;
  if (n_inserted) *n_inserted = ins;
  if (n_full) *n_full = full;
  return SWIM_OK;
}
