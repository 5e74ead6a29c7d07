/* lev_oracle.c — plain O(|a| |b|) dynamic programme of the unit-cost Levenshtein distance over int32 code points
 * (TEST INFRASTRUCTURE ONLY).  The independent restatement the device kernel (levenshtein.cu) is checked against:
 * one DP row per pair, no bit tricks, OpenMP over the rows of the output. */
#include <stdint.h>
#include <stdlib.h>
#include <omp.h>

static int32_t lev_dp(const int32_t* a, int64_t n, const int32_t* b, int64_t m, int32_t* row) {
  /* row[k] = D[x][k] for the current prefix a[0..x) of a, over the prefixes b[0..k) */
  for (int64_t k = 0; k <= m; k++) row[k] = (int32_t)k;
  for (int64_t x = 1; x <= n; x++) {
    int32_t diag = row[0];
    row[0] = (int32_t)x;
    for (int64_t k = 1; k <= m; k++) {
      const int32_t up = row[k];
      int32_t best = diag + (a[x - 1] != b[k - 1]);
      if (up + 1 < best) best = up + 1;
      if (row[k - 1] + 1 < best) best = row[k - 1] + 1;
      diag = up;
      row[k] = best;
    }
  }
  return row[m];
}

int oracle_lev_max_threads(void) { return omp_get_max_threads(); }

/* out[na x nb] (int32) = distance(a_i, b_j); a_i = a_ids[a_off[i] .. a_off[i+1]), likewise b. */
void oracle_levenshtein(const int32_t* a_ids, const int64_t* a_off, int64_t na, const int32_t* b_ids,
                        const int64_t* b_off, int64_t nb, int32_t* out, int threads) {
  int64_t max_b = 0;
  for (int64_t j = 0; j < nb; j++)
    if (b_off[j + 1] - b_off[j] > max_b) max_b = b_off[j + 1] - b_off[j];
#pragma omp parallel num_threads(threads)
  {
    int32_t* row = (int32_t*)malloc(sizeof(int32_t) * (size_t)(max_b + 1));
#pragma omp for schedule(dynamic, 16)
    for (int64_t i = 0; i < na; i++)
      for (int64_t j = 0; j < nb; j++)
        out[i * nb + j] = lev_dp(a_ids + a_off[i], a_off[i + 1] - a_off[i], b_ids + b_off[j], b_off[j + 1] - b_off[j],
                                 row);
    free(row);
  }
}
