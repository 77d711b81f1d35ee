/* TEST INFRASTRUCTURE — not part of the library.
 * The CPU oracle of the AIR constraint check: check_constraints_fn! (stark.rs:2899-3015) as an OpenMP loop over rows that calls
 * the oracle's generated evaluators orc_air_eval_* (oracle/c/air_eval_gen.c, pinned to the reference's golden fingerprint by
 * tests/test_air.py), compiled into this library unchanged.  init on row 0, cons on every row, tran on the pairs (i, i+1) for
 * i < n - 1, term on row n - 1.
 * Build: gcc -O2 -fopenmp -shared -fPIC tests/host/air_check_oracle.c -o tests/host/_build/libair_check_oracle.so */
#include <stdlib.h>
#include "../../oracle/c/air_eval_gen.c"

#define NC 604
#define NMAIN 379
#define NAUX3 270

static void eval_category(int cat, const u64 *mc, const u64 *ac, const u64 *mn, const u64 *an, const u64 *ch, u64 *out) {
  if (cat == 0) orc_air_eval_init(mc, ac, mn, an, ch, out);
  else if (cat == 1) orc_air_eval_cons(mc, ac, mn, an, ch, out);
  else if (cat == 2) orc_air_eval_tran(mc, ac, mn, an, ch, out);
  else orc_air_eval_term(mc, ac, mn, an, ch, out);
}

/* main: [379][n]; aux: [270][n] planar (plane 3q + d), challenges [63][3], all Montgomery.  Per constraint of the evaluator
 * order: the number of rows where it is non-zero and the first and last such row (UINT64_MAX when there is none). */
void air_check_oracle(const u64 *main, const u64 *aux, size_t n, const u64 *ch, u64 *counts, u64 *first, u64 *last) {
  for (size_t j = 0; j < NC; j++) { counts[j] = 0; first[j] = UINT64_MAX; last[j] = UINT64_MAX; }
#pragma omp parallel
  {
    u64 *mc = (u64 *)malloc((2 * NMAIN + 2 * NAUX3) * sizeof(u64));
    u64 *mn = mc + NMAIN, *ac = mn + NMAIN, *an = ac + NAUX3;
    u64 *vals = (u64 *)malloc(3 * 512 * sizeof(u64));
    u64 *cnt = (u64 *)calloc(3 * NC, sizeof(u64)), *fst = cnt + NC, *lst = fst + NC;
    for (size_t j = 0; j < NC; j++) { fst[j] = UINT64_MAX; lst[j] = UINT64_MAX; }
#pragma omp for schedule(static)
    for (size_t i = 0; i < n; i++) {
      size_t nx = i + 1 < n ? i + 1 : i;
      for (size_t c = 0; c < NMAIN; c++) { mc[c] = main[c * n + i]; mn[c] = main[c * n + nx]; }
      for (size_t c = 0; c < NAUX3; c++) { ac[c] = aux[c * n + i]; an[c] = aux[c * n + nx]; }
      size_t off = 0;
      for (int cat = 0; cat < 4; cat++) {
        int applies = cat == 1 || (cat == 0 && i == 0) || (cat == 2 && i + 1 < n) || (cat == 3 && i + 1 == n);
        if (applies) {
          eval_category(cat, mc, ac, mn, an, ch, vals);
          for (int k = 0; k < ORC_AIR_NUM_CONSTRAINTS[cat]; k++) {
            if (!(vals[3 * k] | vals[3 * k + 1] | vals[3 * k + 2])) continue;
            size_t j = off + k;
            cnt[j]++;
            if (fst[j] == UINT64_MAX || i < fst[j]) fst[j] = i;
            if (lst[j] == UINT64_MAX || i > lst[j]) lst[j] = i;
          }
        }
        off += ORC_AIR_NUM_CONSTRAINTS[cat];
      }
    }
#pragma omp critical
    for (size_t j = 0; j < NC; j++) {
      if (!cnt[j]) continue;
      counts[j] += cnt[j];
      if (first[j] == UINT64_MAX || fst[j] < first[j]) first[j] = fst[j];
      if (last[j] == UINT64_MAX || lst[j] > last[j]) last[j] = lst[j];
    }
    free(mc); free(vals); free(cnt);
  }
}
