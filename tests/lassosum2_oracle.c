/* CPU oracle of lassosum2 and ld_scores_sfbm over bigsparser's SFBM storage -- test infrastructure only.
 *
 * Literal scalar restatements of src/lassosum2.cpp:20-70 and src/ld-scores-sfbm.cpp:9-69, written from their semantics.
 * Built with -O2 -ffp-contract=off (no FMA contraction, as the reference's build): every update is d += x * shift with two
 * roundings.  OpenMP runs the grid points in parallel, never one descent.
 *
 * Storage: p[ncol + 1]; first_i == NULL: data interleaves (row, value), column j at data[2 p[j] .. 2 p[j + 1]);
 * first_i != NULL: values only, column j at data[p[j] .. p[j + 1]) for the rows first_i[j], first_i[j] + 1, ...
 */
#define _POSIX_C_SOURCE 199309L
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

static double soft_thres(double z, double l1, double one_plus_l2) {
  double num;
  if (z > 0) {
    num = z - l1;
    return num > 0 ? num / one_plus_l2 : 0;
  }
  num = z + l1;
  return num < 0 ? num / one_plus_l2 : 0;
}

static double na_real(void) {
  const uint64_t bits = 0x7FF00000000007A2ULL; /* R's NA_real_ */
  double d;
  memcpy(&d, &bits, sizeof d);
  return d;
}

/* dotprods += shift * column j2 (bigsparser's incr_mult_col) */
static void incr_mult_col(const double *p, const double *data, const int *first_i, int j2, double shift, double *dot) {
  size_t lo = (size_t)p[j2], up = (size_t)p[j2 + 1], k;
  if (first_i) {
    int i = first_i[j2];
    for (k = lo; k < up; k++, i++) dot[i] += data[k] * shift;
  } else {
    for (k = lo; k < up; k++) dot[(size_t)data[2 * k]] += data[2 * k + 1] * shift;
  }
}

/* One grid point: beta (m), returns num_iter; moves (column updates) and entries (stored values they read) when non-NULL */
static int lassosum2_one(const double *p, const double *data, const int *first_i, int ncol, const double *beta_hat, int m,
                         const int *ind_sub, const double *lambda, const double *dp1, double dfmax, int maxiter, double tol,
                         double *beta, long long *moves, long long *entries) {
  double *dot = calloc(ncol ? ncol : 1, sizeof(double));
  double gap0 = 0;
  long long nmv = 0, nent = 0;
  int j, k = 0;
  if (!dot) return -1;
  for (j = 0; j < m; j++) gap0 = gap0 + beta_hat[j] * beta_hat[j];
  gap0 = 2 * gap0;
  for (j = 0; j < m; j++) beta[j] = 0;
  for (; k < maxiter; k++) {
    int conv = 1;
    double df = 0, gap = 0;
    for (j = 0; j < m; j++) {
      int j2 = ind_sub[j];
      double u = beta_hat[j] - (dot[j2] - beta[j]);
      double nb = soft_thres(u, lambda[j], dp1[j]);
      double shift;
      if (nb != 0) {
        gap += nb * nb;
        df++;
      }
      shift = nb - beta[j];
      if (shift != 0) {
        if (conv && fabs(shift) > tol) conv = 0;
        beta[j] = nb;
        incr_mult_col(p, data, first_i, j2, shift, dot);
        nmv++;
        nent += (long long)(p[j2 + 1] - p[j2]);
      }
    }
    if (gap > gap0) {
      for (j = 0; j < m; j++) beta[j] = na_real();
      break;
    }
    if (conv || df > dfmax) break;
  }
  free(dot);
  if (moves) *moves = nmv;
  if (entries) *entries = nent;
  return k + 1;
}

/* ngrid points: lambda / dp1 / beta m x ngrid column-major; seconds[g] wall time of point g (NULL allowed) */
int lso_lassosum2(const double *p, const double *data, const int *first_i, int ncol, const double *beta_hat, int m,
                  const int *ind_sub, int ngrid, const double *lambda, const double *dp1, double dfmax, int maxiter, double tol,
                  double *beta, int *num_iter, long long *moves, long long *entries, double *seconds, int nthreads) {
  int g, bad = 0;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads) reduction(| : bad)
  for (g = 0; g < ngrid; g++) {
    struct timespec t0, t1;
    const size_t o = (size_t)g * m;
    clock_gettime(CLOCK_MONOTONIC, &t0);
    num_iter[g] = lassosum2_one(p, data, first_i, ncol, beta_hat, m, ind_sub, lambda + o, dp1 + o, dfmax, maxiter, tol,
                                beta + o, moves ? moves + g : NULL, entries ? entries + g : NULL);
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (num_iter[g] < 0) bad = 1;
    if (seconds) seconds[g] = (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
  }
  return bad;
}

/* ld_scores_sfbm: out[j] = sum of x^2 over the stored entries of column ind_sub[j] whose row is in ind_sub (0-based) */
int lso_ld_scores(const double *p, const double *data, const int *first_i, int nrow, int ncol, const int *ind_sub, int m,
                  double *out) {
  char *use = calloc((nrow > ncol ? nrow : ncol) + 1, 1);
  int j;
  if (!use) return -1;
  for (j = 0; j < m; j++) use[ind_sub[j]] = 1;
  for (j = 0; j < m; j++) {
    int j2 = ind_sub[j];
    size_t lo = (size_t)p[j2], up = (size_t)p[j2 + 1], k;
    double s = 0;
    if (first_i) {
      int i = first_i[j2];
      for (k = lo; k < up; k++, i++)
        if (use[i]) s += data[k] * data[k];
    } else {
      for (k = lo; k < up; k++)
        if (use[(size_t)data[2 * k]]) s += data[2 * k + 1] * data[2 * k + 1];
    }
    out[j] = s;
  }
  free(use);
  return 0;
}
