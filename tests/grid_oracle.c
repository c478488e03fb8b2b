/* grid_oracle.c -- CPU oracle of snp_grid_clumping's inner call (test infrastructure only, compiled by tests/grid_ref.py).
 *
 * src/clumping-cached.cpp:11-110  clumping_chr_cached, restated for one thread: the reference's OpenMP loop spin-waits on
 * keep[] so its result is that of the sequential pass in rank order.  The statistic (:84-92) reads the FBM.code256 values
 * code256[byte] as SubBMCode256Acc does (NA_real for a missing code, so r2 is NA and never > thr).  The r2 cache is a dense
 * sq_dim x sq_dim column-major matrix holding what the reference's sparse matrix holds (an absent entry reads 0): entry
 * (spInd[j], spInd[j0]) is read from sqcor and, when it is 0, recomputed and written to new_sqcor (:76-94).  keep must come in
 * filled with -1. */
#include <math.h>
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

/* src/clumping-utils.h:12-43 */
static int which_to_check(int j0, const int *keep, const int *rankInd, const double *pos, int m, double size, int *out) {
  int cnt = 0;
  double pos_min = pos[j0] - size, pos_max = pos[j0] + size;
  int not_min = 1, not_max = 1;
  for (int k = 1; not_max || not_min; k++) {
    if (not_max) {
      int j = j0 + k;
      not_max = (j < m) && (pos[j] <= pos_max);
      if (not_max && (rankInd[j0] > rankInd[j]) && (keep[j] != 0)) out[cnt++] = j;
    }
    if (not_min) {
      int j = j0 - k;
      not_min = (j >= 0) && (pos[j] >= pos_min);
      if (not_min && (rankInd[j0] > rankInd[j]) && (keep[j] != 0)) out[cnt++] = j;
    }
  }
  return cnt;
}

int grc_clumping_chr_cached(const uint8_t *mat, int n_tot, const double *code256, const double *sqcor, double *new_sqcor,
                            int sq_dim, const int *spInd, const int *rowInd, int nr, const int *colInd, int nc,
                            const int *ordInd, const int *rankInd, const double *pos, const double *sumX,
                            const double *denoX, double size, double thr, int *keep) {
  int *chk = (int *)malloc((size_t)(nc ? nc : 1) * sizeof(int));
  if (!chk) return 7;
  size_t n = (size_t)nr, m = (size_t)nc;
  for (size_t k = 0; k < m; k++) {
    size_t j0 = (size_t)ordInd[k] - 1;
    int j0_sp = spInd[j0];
    int nb_check = which_to_check((int)j0, keep, rankInd, pos, (int)m, size, chk);
    int keep_j0 = 1;
    for (int k2 = 0; k2 < nb_check; k2++) {
      int jk = chk[k2];
      if (keep[jk] == 0) continue; /* pruned: no need to check (one thread: never -1 here) */
      size_t j = (size_t)jk;
      int j_sp = spInd[j];
      size_t at = (size_t)j_sp + (size_t)j0_sp * (size_t)sq_dim;
      double r2 = sqcor[at];
      if (r2 == 0) {
        const uint8_t *cj = mat + (size_t)(colInd[j] - 1) * (size_t)n_tot;
        const uint8_t *cj0 = mat + (size_t)(colInd[j0] - 1) * (size_t)n_tot;
        double xySum = 0;
        for (size_t i = 0; i < n; i++) {
          size_t r = (size_t)rowInd[i] - 1;
          xySum += code256[cj[r]] * code256[cj0[r]];
        }
        double num = xySum - sumX[j] * sumX[j0] / n;
        r2 = num * num / (denoX[j] * denoX[j0]);
        new_sqcor[at] = r2; /* cache for later use */
      }
      if (r2 > thr) {
        keep_j0 = 0;
        break;
      }
    }
    keep[j0] = keep_j0;
  }
  free(chk);
  return 0;
}
