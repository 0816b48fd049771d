/* tools/spec_model.c — DESIGN MODEL / TEST INFRASTRUCTURE, not product code.
 *
 * A CPU model of the decision rules of the product's speculative assign pass
 * (blance_b200/csrc/assign_pass_spec.cuh), run INSIDE the array-form oracle (oracle/fast.c): every step is
 * still executed by the oracle's one_step() (the truth), and before each step the model states what the
 * kernel would have decided from possibly stale "scout" results:
 *
 *   - a scout evaluated step j at some earlier moment (epoch tag e): exact keys of the partition's K
 *     current nodes with  n2n = qstat[j][q] + A[top][c]  (qstat: the number of earlier eligible steps of the
 *     pass with the same (top, node) pair; A: the deviation matrix that only non-sticky outcomes touch),
 *     T = the worst of them, perm = their (score, position) order;
 *   - the leader accepts it iff every current node c has lastchg[c] <= e and T < B0, the smallest base key
 *     (score with n2n = 0 and no stickiness) over all live nodes.
 *
 * The model asserts that every accepted step is sticky in the oracle (same nodes, same order) and that
 * qstat + A equals the oracle's nodeToNodeCounts; it also models the sorted list of the smallest base keys
 * with which the leader resolves movers alone, asserts its answer whenever its bound test passes, and
 * prints how often each path would be taken.  Scout timing is randomised (seeded) - exactness must not
 * depend on it.
 */
#include <stdint.h>
#include <stdio.h>

static void spec_pass(void* f, const void* order, int32_t lim, int32_t s);
#define FO_PASS(f, order, lim, s) spec_pass((void*)(f), (const void*)(order), (lim), (s))
#include "../oracle/fast.c"

/* extended resolve of a failed bound proof (K winners found, the K-th not below ub): the exact scores of the unlisted,
 * live, unblocked nodes whose base key is lex-below the K-th winner decide the step together with the listed and the
 * current nodes.  xhist: how many such nodes there were, in buckets 0 | 1 | 2 | 3-4 | 5-8 | 9-16 | 17-32 | 33-64 |
 * 65-128 | more. */
#define XHIST 10
typedef struct {
  long long steps, elig, fast, slow_sticky, movers, inelig, stale, t_ge_b0;
  long long list_ok, list_fail, list_rebuild, list_ok_sticky;
  long long asserts_failed;
  long long list_fail_k;               /* of list_fail: K winners found (the extended resolve applies) */
  long long xres_ok;                   /* extended resolves checked against the oracle's outcome */
  long long xmax;                      /* the largest extended set */
  long long xhist[XHIST];
} spec_stats_t;
static spec_stats_t g_st;
static int g_H = 256, g_resweeps = 2, g_L = 32, g_Lmin = 6;
static uint64_t g_rng = 88172645463325252ull;
static uint64_t rnd(void) { g_rng ^= g_rng << 13; g_rng ^= g_rng >> 7; g_rng ^= g_rng << 17; return g_rng; }

typedef struct { double T; int32_t Tpos; int32_t tag; uint8_t perm[4]; uint8_t have; } scout_t;
typedef struct { int32_t p, top, n_cur, elig; int32_t cur[4]; int32_t qstat[4]; double stick; int64_t wp; } rec_t;

static double base_score(const fo_t* f, int32_t s, int32_t n) {
  const blance_plan_in* in = f->in;
  double filled = 0.0;
  if (f->P > 0) filled = (0.001 * (double)f->tot[n]) / (double)f->P;
  double r = (double)f->counts[(size_t)s * f->N + n];
  r = r + 0.0;
  r = r + filled;
  if (in->has_node_weights && in->node_has_weight[n]) {
    int32_t w = in->node_weight[n];
    if (w > 0) r = r / (double)w;
    else if (w < 0 && in->booster_kind == BLANCE_BOOSTER_CBGT_MAX) { double b = (double)(-(int64_t)w); if (b < 0.0) b = 0.0; r = r + b; }
  }
  r = r - 0.0;
  return r;
}
/* exact score with an explicit n2n count q */
static double score_q(const fo_t* f, int32_t s, int32_t n, int64_t q, double cur) {
  const blance_plan_in* in = f->in;
  double lower = 0.0, filled = 0.0;
  if (f->P > 0) { lower = (double)q / (double)f->P; filled = (0.001 * (double)f->tot[n]) / (double)f->P; }
  double r = (double)f->counts[(size_t)s * f->N + n];
  r = r + lower;
  r = r + filled;
  if (in->has_node_weights && in->node_has_weight[n]) {
    int32_t w = in->node_weight[n];
    if (w > 0) r = r / (double)w;
    else if (w < 0 && in->booster_kind == BLANCE_BOOSTER_CBGT_MAX) { double b = (double)(-(int64_t)w); if (b < cur) b = cur; r = r + b; }
  }
  r = r - cur;
  return r;
}
static int lex_lt(double a, int32_t pa, double b, int32_t pb) { return a < b || (a == b && pa < pb); }

static void scout_eval(const fo_t* f, int32_t s, int K, const rec_t* r, const int32_t* A, int32_t epoch, scout_t* o) {
  o->have = 1; o->tag = epoch;
  double key[4];
  int ok = 1;
  for (int q = 0; q < K; q++) {
    const int32_t c = r->cur[q];
    if (!f->valid[c]) ok = 0;
    key[q] = score_q(f, s, c, (int64_t)r->qstat[q] + A[(size_t)r->top * f->N + c], r->stick);
  }
  int worst = 0;
  for (int q = 1; q < K; q++) if (lex_lt(key[worst], r->cur[worst], key[q], r->cur[q])) worst = q;
  o->T = ok ? key[worst] : 1e300; o->Tpos = r->cur[worst];
  for (int q = 0; q < K; q++) {
    int rank = 0;
    for (int t = 0; t < K; t++) if (t != q && lex_lt(key[t], r->cur[t], key[q], r->cur[q])) rank++;
    o->perm[rank] = (uint8_t)q;
  }
}

typedef struct { double k; int32_t n; } lent_t;

static void spec_pass(void* fv, const void* ov, int32_t lim, int32_t s) {
  fo_t* f = (fo_t*)fv;
  const okey_t* order = (const okey_t*)ov;
  const blance_plan_in* in = f->in;
  const int32_t N = f->N, K = in->state_constraints[s];
  const int rules = in->has_hier_rules && in->rule_off[s + 1] > in->rule_off[s];
  if (rules || K > 4 || lim < 1) { for (int32_t i = 0; i < lim; i++) one_step(f, order[i].p, s); return; }
  const int32_t lo = in->state_slot_off[s], hi = in->state_slot_off[s + 1];
  uint32_t higher = 0;
  for (int s2 = 0; s2 < f->S; s2++) if (in->state_priority[s2] < in->state_priority[s]) higher |= 1u << s2;

  rec_t* rec = (rec_t*)calloc((size_t)lim, sizeof(rec_t));
  scout_t* sc = (scout_t*)calloc((size_t)lim, sizeof(scout_t));
  int32_t* A = (int32_t*)calloc((size_t)(f->NU + 1) * N, sizeof(int32_t));
  int32_t* paircnt = (int32_t*)calloc((size_t)(f->NU + 1) * N, sizeof(int32_t));
  int32_t* lastchg = (int32_t*)calloc((size_t)N, sizeof(int32_t));
  double* base = (double*)calloc((size_t)N, sizeof(double));
  int32_t epoch = 0;

  /* records + qstat (rows only change at their own step, so the records are static for the pass) */
  for (int32_t j = 0; j < lim; j++) {
    rec_t* r = &rec[j];
    const int32_t p = order[j].p;
    const int32_t* row = row_of(f->rows, f->SL, p);
    r->p = p; r->wp = 1; r->stick = 1.5;
    if (in->has_part_weights) {
      if (in->part_has_weight[p]) { r->wp = in->part_weight[p]; r->stick = (double)in->part_weight[p]; }
      else if (in->state_has_stickiness[s]) r->stick = (double)in->state_stickiness[s];
    }
    r->top = f->NU;
    { int32_t tlo = in->state_slot_off[in->top_state]; if (tlo < in->state_slot_off[in->top_state + 1] && row[tlo] != NONE) r->top = row[tlo]; }
    int n_cur = 0, clean = 1;
    for (int a = lo; a < hi && row[a] != NONE; a++) {
      n_cur++;
      if (row[a] >= N) clean = 0;
      for (int b = 0; b < f->SL; b++) if (b != a && row[b] == row[a]) clean = 0;
    }
    r->n_cur = n_cur;
    r->elig = clean && n_cur == K && f->shape[(size_t)p * f->S + s] != BLANCE_SHAPE_ABSENT;
    if (r->elig)
      for (int q = 0; q < K; q++) {
        r->cur[q] = row[lo + q];
        r->qstat[q] = paircnt[(size_t)r->top * N + r->cur[q]]++;
      }
  }

  /* sorted list of the smallest base keys + lower bound of everything unlisted */
  lent_t* L = (lent_t*)calloc((size_t)g_L + 1, sizeof(lent_t));
  int Llen = 0; double ubk = 1e308; int32_t ubp = 0x7fffffff;
  uint8_t* listed = (uint8_t*)calloc((size_t)N, 1);
#define REBUILD() do { \
    for (int32_t n_ = 0; n_ < N; n_++) { base[n_] = base_score(f, s, n_); listed[n_] = 0; } \
    Llen = 0; ubk = 1e308; ubp = 0x7fffffff; \
    for (int r_ = 0; r_ <= g_L; r_++) { \
      int32_t b_ = -1; \
      for (int32_t n_ = 0; n_ < N; n_++) if (f->valid[n_] && !listed[n_] && (b_ < 0 || base[n_] < base[b_])) b_ = n_; \
      if (b_ < 0) break; \
      if (r_ == g_L) { ubk = base[b_]; ubp = b_; break; } \
      L[Llen].k = base[b_]; L[Llen].n = b_; Llen++; listed[b_] = 1; } \
    g_st.list_rebuild++; } while (0)
  REBUILD();

  int32_t scouted_to = -1;
  for (int32_t j = 0; j < lim; j++) {
    /* scouts: new entries entering the region, with the state of this moment */
    int32_t far = j + g_H < lim ? j + g_H : lim - 1;
    /* entries enter the region at a random time after they become reachable (models scout latency) */
    while (scouted_to < far && (scouted_to < j + g_H / 2 || (rnd() & 3) == 0)) {
      scouted_to++;
      if (rec[scouted_to].elig) scout_eval(f, s, K, &rec[scouted_to], A, epoch, &sc[scouted_to]);
    }
    for (int r = 0; r < g_resweeps; r++) {
      int32_t x = j + (int32_t)(rnd() % (uint64_t)g_H);
      if (x <= scouted_to && x < lim && rec[x].elig) scout_eval(f, s, K, &rec[x], A, epoch, &sc[x]);
    }
    const rec_t* r = &rec[j];
    g_st.steps++;
    /* B0 */
    double b0k = Llen ? L[0].k : ubk; int32_t b0p = Llen ? L[0].n : ubp;
    int predicted = 0;
    if (r->elig) {
      g_st.elig++;
      /* model check: qstat + A == actual n2n for the current nodes */
      for (int q = 0; q < K; q++)
        if ((int64_t)r->qstat[q] + A[(size_t)r->top * N + r->cur[q]] != f->n2n[(size_t)r->top * N + r->cur[q]]) {
          g_st.asserts_failed++;
          if (g_st.asserts_failed < 10) fprintf(stderr, "MODEL: qstat+A != n2n at step %d q %d\n", j, q);
        }
      if (sc[j].have) {
        int valid = 1;
        for (int q = 0; q < K; q++) if (lastchg[r->cur[q]] > sc[j].tag) valid = 0;
        if (!valid) g_st.stale++;
        else if (!lex_lt(sc[j].T, sc[j].Tpos, b0k, b0p)) g_st.t_ge_b0++;
        else predicted = 1;
      } else g_st.stale++;
    } else g_st.inelig++;

    /* list-based resolution of the steps the scouts did not decide */
    int list_pred = 0; int32_t list_ch[4]; int list_n = 0;
    int x_pred = 0; int32_t x_ch[4];
    if (!predicted && r->elig && Llen > 0) {
      const int32_t* row = row_of(f->rows, f->SL, r->p);
#define BLOCKED(n_, out_) do { \
        out_ = 0; \
        for (int q_ = 0; q_ < K; q_++) out_ |= (r->cur[q_] == (n_)); \
        for (int s2_ = 0; s2_ < f->S; s2_++) \
          if (((higher >> s2_) & 1u) && f->shape[(size_t)r->p * f->S + s2_] != BLANCE_SHAPE_ABSENT) \
            out_ |= list_has(row, in->state_slot_off[s2_], in->state_slot_off[s2_ + 1], (n_)); } while (0)
      /* candidates: current nodes + listed nodes, minus nodes of higher-priority states, minus dead nodes */
      int32_t* cn = (int32_t*)malloc(sizeof(int32_t) * ((size_t)N + 8)); double* ck = (double*)malloc(sizeof(double) * ((size_t)N + 8));
      uint8_t* used = (uint8_t*)calloc((size_t)N + 8, 1);
      int nc = 0;
      for (int q = 0; q < K; q++) if (f->valid[r->cur[q]]) { cn[nc] = r->cur[q]; ck[nc] = score_q(f, s, r->cur[q], f->n2n[(size_t)r->top * N + r->cur[q]], r->stick); nc++; }
      for (int x = 0; x < Llen; x++) {
        const int32_t n = L[x].n;
        int blocked;
        BLOCKED(n, blocked);
        if (blocked) continue;
        cn[nc] = n; ck[nc] = score_q(f, s, n, f->n2n[(size_t)r->top * N + n], 0.0); nc++;
      }
      /* current nodes held by a higher-priority state are not candidates either (row clean => cannot happen) */
      double wk = 0.0; int32_t wn = -1;
      for (int t = 0; t < K && t < nc; t++) {
        int b = -1;
        for (int x = 0; x < nc; x++) if (!used[x] && (b < 0 || lex_lt(ck[x], cn[x], ck[b], cn[b]))) b = x;
        used[b] = 1; list_ch[list_n++] = cn[b];
        wk = ck[b]; wn = cn[b];
        if (t == K - 1 && lex_lt(ck[b], cn[b], ubk, ubp)) list_pred = 1;
      }
      if (list_n < K) list_pred = 0;
      if (!list_pred && list_n == K) {
        /* the extended resolve: every node outside listed + current whose base key is lex-below the K-th winner W.
         * A node's exact score is never below its base key, so a node whose base key is not below W cannot beat
         * the K candidates already at or below W; the new K-th winner is <= W, so the set never has to grow. */
        g_st.list_fail_k++;
        int nx = 0;
        for (int32_t n = 0; n < N; n++) {
          if (!f->valid[n] || listed[n] || !lex_lt(base[n], n, wk, wn)) continue;
          int blocked;
          BLOCKED(n, blocked);
          if (blocked) continue;
          cn[nc] = n; ck[nc] = score_q(f, s, n, f->n2n[(size_t)r->top * N + n], 0.0); nc++; nx++;
        }
        int hb = 0;
        while (hb < XHIST - 1 && nx > (hb == 0 ? 0 : (1 << (hb - 1)))) hb++;
        g_st.xhist[hb]++;
        if (nx > g_st.xmax) g_st.xmax = nx;
        memset(used, 0, (size_t)nc);
        for (int t = 0; t < K; t++) {
          int b = -1;
          for (int x = 0; x < nc; x++) if (!used[x] && (b < 0 || lex_lt(ck[x], cn[x], ck[b], cn[b]))) b = x;
          used[b] = 1; x_ch[t] = cn[b];
        }
        x_pred = 1;
      }
#undef BLOCKED
      free(cn); free(ck); free(used);
    }

    /* ---- the truth ---- */
    int32_t* row = row_of(f->rows, f->SL, r->p);
    int32_t before[32];
    for (int i = 0; i < f->SL; i++) before[i] = row[i];
    one_step(f, r->p, s);
    int same = r->elig;
    int32_t chosen[16]; int n_ch = 0;
    for (int a = lo; a < hi && row[a] != NONE; a++) chosen[n_ch++] = row[a];
    if (r->elig) {
      if (n_ch != K) same = 0;
      else for (int q = 0; q < K; q++) { int hit = 0; for (int t = 0; t < K; t++) hit |= (chosen[t] == r->cur[q]); if (!hit) same = 0; }
    }
    if (predicted) {
      g_st.fast++;
      int ok = same;
      if (ok) for (int q = 0; q < K; q++) if (chosen[q] != r->cur[sc[j].perm[q]]) ok = 0;
      if (!ok) { g_st.asserts_failed++; if (g_st.asserts_failed < 10) fprintf(stderr, "MODEL: accepted step %d is not sticky / wrong order\n", j); }
    } else if (same) g_st.slow_sticky++;
    if (!same) g_st.movers++;
    if (!predicted && r->elig && Llen > 0) {
      if (list_pred) {
        g_st.list_ok++;
        if (same) g_st.list_ok_sticky++;
        int ok = (n_ch == list_n);
        for (int q = 0; ok && q < n_ch; q++) if (chosen[q] != list_ch[q]) ok = 0;
        if (!ok) { g_st.asserts_failed++; if (g_st.asserts_failed < 10) fprintf(stderr, "MODEL: list resolution wrong at step %d\n", j); }
      } else g_st.list_fail++;
    }
    if (x_pred) {
      int ok = (n_ch == K);
      for (int q = 0; ok && q < K; q++) if (chosen[q] != x_ch[q]) ok = 0;
      if (ok) g_st.xres_ok++;
      else { g_st.asserts_failed++; if (g_st.asserts_failed < 10) fprintf(stderr, "MODEL: extended resolve wrong at step %d\n", j); }
    }
    /* ---- bookkeeping of a count change ---- */
    if (!same) {
      epoch++;
      /* nodes whose count (any state) or A entry changed */
      int32_t touched[80]; int nt = 0;
      for (int i = lo; i < hi; i++) if (before[i] != NONE && before[i] < N) touched[nt++] = before[i];   /* old nodes of the state */
      for (int q = 0; q < n_ch; q++) touched[nt++] = chosen[q];                                            /* new nodes (also leave other states) */
      for (int q = 0; q < n_ch; q++) A[(size_t)r->top * N + chosen[q]]++;
      if (r->elig) for (int q = 0; q < K; q++) A[(size_t)r->top * N + r->cur[q]]--;
      for (int x = 0; x < nt; x++) {
        const int32_t n = touched[x];
        if (lastchg[n] == epoch) continue;
        lastchg[n] = epoch;
        /* list maintenance */
        if (listed[n]) { int at = 0; while (L[at].n != n) at++; for (int y = at; y + 1 < Llen; y++) L[y] = L[y + 1]; Llen--; listed[n] = 0; }
        base[n] = base_score(f, s, n);
        if (f->valid[n] && lex_lt(base[n], n, ubk, ubp)) {
          int at = 0;
          while (at < Llen && lex_lt(L[at].k, L[at].n, base[n], n)) at++;
          for (int y = Llen; y > at; y--) L[y] = L[y - 1];
          L[at].k = base[n]; L[at].n = n; Llen++; listed[n] = 1;
          if (Llen > g_L) { Llen--; ubk = L[Llen].k; ubp = L[Llen].n; listed[L[Llen].n] = 0; }
        }
      }
      if (Llen < g_Lmin) REBUILD();
    }
  }
  free(rec); free(sc); free(A); free(paircnt); free(lastchg); free(base); free(L); free(listed);
}

FO_EXPORT int spec_model_plan(const blance_plan_in* in, blance_plan_out* out, int H, int resweeps, int Llen, int Lmin, long long* stats_out) {
  memset(&g_st, 0, sizeof g_st);
  g_H = H; g_resweeps = resweeps; g_L = Llen; g_Lmin = Lmin;
  int rc = oracle_fast_plan_next_map_capped(in, out, -1);
  memcpy(stats_out, &g_st, sizeof g_st);
  return rc;
}
