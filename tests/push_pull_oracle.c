/*
 * push_pull_oracle.c — the CPU oracle's push-pull state exchange (DESIGN.md §2.6). TEST INFRASTRUCTURE ONLY.
 *
 * Compiled together with oracle/swim_oracle.c (included below) into a library of its own, so that the exchange runs on
 * the oracle's state through its own state machine (apply_record, pb_enqueue): a handle made by oracle/liboracle.so is
 * passed in as is (same source, same struct layout). tests/push_pull_oracle.py builds and loads it.
 */
#include "../oracle/swim_oracle.c"

enum { P_PUSHPULL = 10 }; /* Philox purpose of the partner draw (DESIGN.md §2.3) */

/* ------------------------------------------------------------------ push-pull state exchange (DESIGN.md §2.6)
 * memberlist's anti-entropy between steps; no reference counterpart (Config.joinHosts, Types.hs:47, is parsed and never
 * used). At round r, every up node i with L >= 1 Alive slots picks the floor(x L / 2^32)-th Alive slot, x = word 0 of
 * Philox block (r, i, P_PUSHPULL, 0). If that partner is up the two swap full states, both read from a snapshot taken
 * first: Alive(self_inc, self), then one record per occupied slot (Dead: from = the sender). A receiver merges its senders
 * in ascending id, every record through apply_record with insertion (Core.hs:206-216) and net = 1; a `Just` is enqueued. */
static void pp_merge(oracle_t *o, uint32_t j, uint32_t s, const uint32_t *s_ids, const uint8_t *s_st, const uint32_t *s_inc,
                     const uint32_t *s_self, uint64_t *ctr, uint64_t *ins, uint64_t *full) {
  const uint8_t *st = o->state + (size_t)j * o->cap;
  uint32_t used = 0;
  while (used < o->cap && st[used] != SWIM_VACANT) ++used;
  for (int32_t slot = -1; slot < (int32_t)o->cap; ++slot) {
    rec_t r = {s, s_self[s], 0, SWIM_MSG_ALIVE, 0, 0};
    if (slot >= 0) {
      const size_t x = (size_t)s * o->cap + (uint32_t)slot;
      if (s_st[x] == SWIM_VACANT) continue;
      r.member = s_ids[x];
      r.incarnation = s_inc[x];
      r.kind = s_st[x] == SWIM_ALIVE ? SWIM_MSG_ALIVE : s_st[x] == SWIM_SUSPECT ? SWIM_MSG_SUSPECT : SWIM_MSG_DEAD;
      r.from = s_st[x] == SWIM_DEAD ? s : 0;
    }
    rec_t rb;
    int err = 0;
    if (apply_record(o, j, r, 1, 1, &rb, &err, ctr)) {
      pb_enqueue(o, j, rb, ctr);
      ctr[SWIM_CTR_RECS_APPLIED]++;
    }
    if (err == SWIM_ECAP) ++*full;
    if (used < o->cap && st[used] != SWIM_VACANT) { ++used; ++*ins; } /* vacancies are last: the row grew */
  }
}

EXPORT int oracle_push_pull(oracle_t *o, uint64_t *n_exchanges, uint64_t *n_inserted, uint64_t *n_full) {
  if (o->cfg.world != 1 || !o->view_set) return SWIM_ESTATE;
  const uint32_t n = o->n, cap = o->cap;
  const size_t slots = (size_t)n * cap;
  uint32_t *s_ids = (uint32_t *)malloc(slots * 4), *s_inc = (uint32_t *)malloc(slots * 4);
  uint32_t *s_self = (uint32_t *)malloc((size_t)n * 4 + 4), *part = (uint32_t *)malloc((size_t)n * 4 + 4);
  uint32_t *first = (uint32_t *)calloc((size_t)n + 1, 4), *chooser = (uint32_t *)malloc((size_t)n * 4 + 4);
  uint8_t *s_st = (uint8_t *)malloc(slots);
  memcpy(s_ids, o->nbr, slots * 4);
  memcpy(s_inc, o->vinc, slots * 4);
  memcpy(s_st, o->state, slots);
  memcpy(s_self, o->self_inc, (size_t)n * 4);
  uint64_t ex = 0, ins = 0, full = 0;
  for (uint32_t i = 0; i < n; ++i) {
    part[i] = SWIM_NO_MEMBER;
    if (!o->alive[i]) continue;
    uint32_t L = 0;
    for (uint32_t s = 0; s < cap; ++s) L += s_st[(size_t)i * cap + s] == SWIM_ALIVE;
    if (!L) continue;
    uint32_t c[4] = {o->round, i, P_PUSHPULL, 0}, w[4];
    philox4x32_10(c, o->key, w);
    uint32_t k = bounded(w[0], L), s = 0;
    for (;; ++s)
      if (s_st[(size_t)i * cap + s] == SWIM_ALIVE && k-- == 0) break;
    const uint32_t p = s_ids[(size_t)i * cap + s];
    if (!o->alive[p]) continue; /* a crashed partner: nothing either way */
    part[i] = p;
    ++ex;
  }
  /* choosers of every node, ascending (a counting sort in chooser order) */
  for (uint32_t i = 0; i < n; ++i)
    if (part[i] != SWIM_NO_MEMBER) first[part[i] + 1]++;
  for (uint32_t j = 0; j < n; ++j) first[j + 1] += first[j];
  {
    uint32_t *fill = (uint32_t *)malloc((size_t)n * 4 + 4);
    memcpy(fill, first, (size_t)n * 4);
    for (uint32_t i = 0; i < n; ++i)
      if (part[i] != SWIM_NO_MEMBER) chooser[fill[part[i]]++] = i;
    free(fill);
  }
  uint64_t tot[SWIM_CTR__COUNT] = {0};
#ifdef _OPENMP
#pragma omp parallel
  {
    uint64_t loc[SWIM_CTR__COUNT] = {0}, li = 0, lf = 0;
#pragma omp for schedule(dynamic, 256)
#else
  {
    uint64_t *loc = tot, li = 0, lf = 0;
#endif
    for (int64_t jj = 0; jj < (int64_t)n; ++jj) {
      const uint32_t j = (uint32_t)jj;
      if (!o->alive[j]) continue;
      /* senders: the partner (pull) and the choosers (push), ascending, each once */
      uint32_t pull = part[j], x = first[j];
      for (;;) {
        const uint32_t c = x < first[j + 1] ? chooser[x] : SWIM_NO_MEMBER;
        uint32_t s;
        if (pull != SWIM_NO_MEMBER && pull <= c) { s = pull; pull = SWIM_NO_MEMBER; if (c == s) ++x; }
        else if (c != SWIM_NO_MEMBER) { s = c; ++x; }
        else break;
        pp_merge(o, j, s, s_ids, s_st, s_inc, s_self, loc, &li, &lf);
      }
    }
#ifdef _OPENMP
#pragma omp critical
    {
      for (int c = 0; c < SWIM_CTR__COUNT; ++c) tot[c] += loc[c];
      ins += li; full += lf;
    }
  }
#else
    ins += li; full += lf;
  }
#endif
  for (int c = 0; c < SWIM_CTR__COUNT; ++c) o->ctr[c] += tot[c];
  free(s_ids); free(s_inc); free(s_self); free(part); free(first); free(chooser); free(s_st);
  if (n_exchanges) *n_exchanges = ex;
  if (n_inserted) *n_inserted = ins;
  if (n_full) *n_full = full;
  return SWIM_OK;
}
