/* CPU oracle of snp_ldsplit's three native steps -- test infrastructure only.
 *
 * Literal scalar restatements of get_L, get_C and get_perc (src/split-LD.cpp:15-61, :65-145, :149-182), written from
 * their semantics.  Built with -O2 -ffp-contract=off (no FMA contraction, as the reference's build).  One thread.
 *
 * corr: the lower triangle in CSC (Matrix::tril), p[m + 1], rows i sorted within each column, diagonal stored first.
 * L: m x (m + 1) CSC (lp[m + 2], li, lx), rows sorted within each column; L(row, col) is found by binary search, as an
 * arma::sp_mat element read finds it.
 */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

/* get_L: count the triplets when li == NULL, else write them (by column of corr, row descending) */
long long ldo_get_L(const long long *p, const int *i, const double *x, int m, double thr_r2, double max_r2, int *li, int *lj,
                    double *lx) {
  long long n = 0;
  int col, row;
  for (col = 0; col < m; col++) {
    double l = 0;
    long long k = p[col + 1] - 1; /* the diagonal makes the column non-empty */
    for (row = i[k]; row > col; row--) {
      if (row == i[k]) {
        double r2 = x[k] * x[k];
        if (r2 >= thr_r2) {
          if (r2 > max_r2)
            l = INFINITY;
          else
            l += r2;
        }
        k--;
      }
      if (l > 0) {
        if (li) {
          li[n] = col;
          lj[n] = row;
          lx[n] = l;
        }
        n++;
      }
    }
  }
  return n;
}

static double L_at(const long long *lp, const int *li, const double *lx, int row, int col) {
  long long lo = lp[col], hi = lp[col + 1];
  while (lo < hi) {
    long long mid = lo + (hi - lo) / 2;
    if (li[mid] < row)
      lo = mid + 1;
    else
      hi = mid;
  }
  return (lo < lp[col + 1] && li[lo] == row) ? lx[lo] : 0.0;
}

/* get_C: C and best_ind are m x max_K column-major; best_ind 1-based, NA_integer_ where unset.  Returns the number of
 * stored E values, or -1 on allocation failure.  layers (may be NULL): the layers run, counting layer 0. */
long long ldo_get_C(const long long *lp, const int *li, const double *lx, int m, int min_size, int max_size, int max_K,
                    double max_cost, const double *pos_scaled, double *C1, int *best_ind, int *layers) {
  const int NA = (int)0x80000000;
  float **E = calloc(m ? m : 1, sizeof(float *));
  int *nE = calloc(m ? m : 1, sizeof(int));
  double *C2 = malloc((size_t)m * max_K * sizeof(double) + 1);
  long long total = 0;
  int col, row, k, size, nk = max_K;
  if (!E || !nE || !C2) return -1;
  for (col = 0; col < m; col++) {
    double e = 0, pos_min = pos_scaled[col] - 1;
    int count = 0;
    E[col] = malloc((size_t)(max_size > 0 ? max_size : 1) * sizeof(float));
    if (!E[col]) return -1;
    for (row = col; row >= 0; row--) {
      if (pos_scaled[row] < pos_min) break;
      e += L_at(lp, li, lx, row, col + 1);
      if (e > max_cost) break;
      count++;
      if (count >= min_size) {
        E[col][nE[col]++] = (float)e;
        if (count == max_size) break;
      }
    }
    total += nE[col];
  }
  for (k = 0; k < m * max_K; k++) {
    best_ind[k] = NA;
    C1[k] = INFINITY;
    C2[k] = INFINITY;
  }
  {
    double pos_min = pos_scaled[m - 1] - 1;
    for (size = min_size; size <= max_size; size++) {
      row = m - size;
      if (pos_scaled[row] < pos_min) break;
      best_ind[row] = m;
      C1[row] = 0;
      C2[row] = (double)size * size;
    }
  }
  for (k = 1; k < max_K; k++) {
    double *c1 = C1 + (size_t)k * m, *c2 = C2 + (size_t)k * m;
    const double *p1 = C1 + (size_t)(k - 1) * m, *p2 = C2 + (size_t)(k - 1) * m;
    int *bi = best_ind + (size_t)k * m;
    for (col = m - 1; col >= 0; col--) {
      /* C(m, k - 1) reads past the column: in column-major order it is C(0, k), still +Inf here */
      const double prev1 = col + 1 < m ? p1[col + 1] : c1[0], prev2 = col + 1 < m ? p2[col + 1] : c2[0];
      int t;
      row = col - min_size + 1;
      for (t = 0; t < nE[col]; t++, row--) {
        double cost1 = (double)E[col][t] + prev1;
        double sz = col - row + 1;
        if (cost1 < c1[row]) {
          bi[row] = col + 1;
          c1[row] = cost1;
          c2[row] = sz * sz + prev2;
        } else if (cost1 == c1[row]) {
          double cost2 = sz * sz + prev2;
          if (cost2 < c2[row]) {
            bi[row] = col + 1;
            c2[row] = cost2;
          }
        }
      }
    }
    if (c1[0] > max_cost && c1[0] > p1[0]) {
      nk = k + 1;
      break;
    }
  }
  if (layers) *layers = nk;
  for (col = 0; col < m; col++) free(E[col]);
  free(E);
  free(nE);
  free(C2);
  return total;
}

/* get_perc: all_last 0-based, one per block */
double ldo_get_perc(const double *p, const int *i, int m, long long nnz, const int *all_last) {
  double count_all = (double)(2 * nnz - m);
  double count_within = count_all;
  int grp_num = 0, limit = all_last[0], j;
  for (j = 0; j < m; j++) {
    size_t lo, up, k;
    if (j > limit) {
      grp_num++;
      limit = all_last[grp_num];
    }
    lo = (size_t)p[j];
    up = (size_t)p[j + 1];
    for (k = up - 1; k > lo; k--) {
      if (i[k] > limit)
        count_within -= 2;
      else
        break;
    }
  }
  return count_within / count_all;
}
