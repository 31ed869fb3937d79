/*
 * between_steps_oracle.c — the CPU oracle's calls between steps: the push-pull state exchange (DESIGN.md §2.6), seed
 * joins (§2.7) and graceful leaves (§2.8). TEST INFRASTRUCTURE ONLY.
 *
 * Compiled together with oracle/swim_oracle.c (included below) into a library of its own, so that every record goes
 * through the oracle's own state machine (apply_record, pb_enqueue): a handle made by oracle/liboracle.so is passed in
 * as is (same source, same struct layout). tests/between_steps_oracle.py builds and loads it.
 */
#include "../oracle/swim_oracle.c"

enum { P_PUSHPULL = 10 }; /* Philox purpose of the partner draw (DESIGN.md §2.3) */

/* The senders' state of an exchange, copied before any row changes. */
typedef struct {
  uint32_t *ids, *inc, *self;
  uint8_t *st;
} snap_t;

static snap_t snap_take(const oracle_t *o) {
  const size_t slots = (size_t)o->n * o->cap;
  snap_t s = {(uint32_t *)malloc(slots * 4), (uint32_t *)malloc(slots * 4), (uint32_t *)malloc((size_t)o->n * 4 + 4),
              (uint8_t *)malloc(slots)};
  memcpy(s.ids, o->nbr, slots * 4);
  memcpy(s.inc, o->vinc, slots * 4);
  memcpy(s.self, o->self_inc, (size_t)o->n * 4);
  memcpy(s.st, o->state, slots);
  return s;
}

static void snap_free(snap_t *s) { free(s->ids); free(s->inc); free(s->self); free(s->st); }

static int cmp_u64(const void *a, const void *b) {
  const uint64_t x = *(const uint64_t *)a, y = *(const uint64_t *)b;
  return x < y ? -1 : x > y;
}

/* ------------------------------------------------------------------ push-pull state exchange (DESIGN.md §2.6)
 * memberlist's anti-entropy between steps; no reference counterpart (Config.joinHosts, Types.hs:47, is parsed and never
 * used). At round r, every up node i with L >= 1 Alive slots picks the floor(x L / 2^32)-th Alive slot, x = word 0 of
 * Philox block (r, i, P_PUSHPULL, 0). If that partner is up the two swap full states, both read from a snapshot taken
 * first: Alive(self_inc, self), then one record per occupied slot (Dead: from = the sender). A receiver merges its senders
 * in ascending id, every record through apply_record with insertion (Core.hs:206-216) and net = 1; a `Just` is enqueued. */
static void pp_merge(oracle_t *o, uint32_t j, uint32_t s, const snap_t *sn, uint64_t *ctr, uint64_t *ins, uint64_t *full) {
  const uint8_t *st = o->state + (size_t)j * o->cap;
  uint32_t used = 0;
  while (used < o->cap && st[used] != SWIM_VACANT) ++used;
  for (int32_t slot = -1; slot < (int32_t)o->cap; ++slot) {
    rec_t r = {s, sn->self[s], 0, SWIM_MSG_ALIVE, 0, 0};
    if (slot >= 0) {
      const size_t x = (size_t)s * o->cap + (uint32_t)slot;
      if (sn->st[x] == SWIM_VACANT) continue;
      r.member = sn->ids[x];
      r.incarnation = sn->inc[x];
      r.kind = sn->st[x] == SWIM_ALIVE ? SWIM_MSG_ALIVE : sn->st[x] == SWIM_SUSPECT ? SWIM_MSG_SUSPECT : SWIM_MSG_DEAD;
      r.from = sn->st[x] == SWIM_DEAD ? s : 0;
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
  snap_t sn = snap_take(o);
  uint32_t *part = (uint32_t *)malloc((size_t)n * 4 + 4), *first = (uint32_t *)calloc((size_t)n + 1, 4);
  uint32_t *chooser = (uint32_t *)malloc((size_t)n * 4 + 4);
  uint64_t ex = 0, ins = 0, full = 0;
  for (uint32_t i = 0; i < n; ++i) {
    part[i] = SWIM_NO_MEMBER;
    if (!o->alive[i]) continue;
    uint32_t L = 0;
    for (uint32_t s = 0; s < cap; ++s) L += sn.st[(size_t)i * cap + s] == SWIM_ALIVE;
    if (!L) continue;
    uint32_t c[4] = {o->round, i, P_PUSHPULL, 0}, w[4];
    philox4x32_10(c, o->key, w);
    uint32_t k = bounded(w[0], L), s = 0;
    for (;; ++s)
      if (sn.st[(size_t)i * cap + s] == SWIM_ALIVE && k-- == 0) break;
    const uint32_t p = sn.ids[(size_t)i * cap + s];
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
        pp_merge(o, j, s, &sn, loc, &li, &lf);
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
  snap_free(&sn);
  free(part); free(first); free(chooser);
  if (n_exchanges) *n_exchanges = ex;
  if (n_inserted) *n_inserted = ins;
  if (n_full) *n_full = full;
  return SWIM_OK;
}

/* ------------------------------------------------------------------ seed joins (DESIGN.md §2.7)
 * memberlist's Join(joinHosts); the reference parses Config.joinHosts (Types.hs:47, Util.hs:46) and never joins. Every
 * pair is checked first (ids < N, node != seed). With SWIM_JOIN_FRESH every listed joiner that is up loses its row and
 * its piggyback buffer. Then a snapshot, and each pair (j, s) with both up is an exchange: j receives s's state and s
 * receives j's. A receiver merges its distinct senders in ascending id, each once, through pp_merge. */
EXPORT int oracle_join(oracle_t *o, const uint32_t *node, const uint32_t *seed, size_t np, uint32_t flags,
                       uint64_t *n_exchanges, uint64_t *n_inserted, uint64_t *n_full) {
  if (o->cfg.world != 1 || !o->view_set) return SWIM_ESTATE;
  for (size_t k = 0; k < np; ++k)
    if (node[k] >= o->N || seed[k] >= o->N || node[k] == seed[k]) return SWIM_EINVAL;
  const uint32_t cap = o->cap;
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
  snap_t sn = snap_take(o);
  uint64_t *dir = (uint64_t *)malloc(2 * np * 8 + 8); /* receiver << 32 | sender */
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
    if (x == 0 || dir[x] != dir[x - 1]) pp_merge(o, (uint32_t)(dir[x] >> 32), (uint32_t)dir[x], &sn, o->ctr, &ins, &full);
  snap_free(&sn);
  free(dir);
  if (n_exchanges) *n_exchanges = ex;
  if (n_inserted) *n_inserted = ins;
  if (n_full) *n_full = full;
  return SWIM_OK;
}

/* ------------------------------------------------------------------ graceful leaves (DESIGN.md §2.8)
 * memberlist's Leave: Dead about the departing process, from itself. The reference has no leave. Every id is checked
 * first (< N). The leavers are the distinct listed ids that are up. Each goes down as a CRASH at the current round does,
 * and back_at = 0. Then every node m in ascending id that is up, for every leaver L in ascending id whose row holds m
 * Alive or Suspect: Dead(self_inc_L, L, from L) through apply_record (no insert, net = 1) at the current round, exactly
 * as run_events applies a SWIM_EV_INJECT datagram; a `Just` is enqueued and counted in RECS_APPLIED. */
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
  qsort(dir, nd, 8, cmp_u64);
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
