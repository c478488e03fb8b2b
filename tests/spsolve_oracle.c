/* CPU oracle of sp_solve_sym over bigsparser's SFBM storage -- test infrastructure only.
 *
 * Eigen's ConjugateGradient (identity preconditioner, x0 = 0), as bigsparser::sp_solve_sym calls it at R/LDpred2.R:38-39,
 * restated with this project's declared reduction order (DESIGN.md §4.13), not with Eigen's SIMD dot order: its results
 * are what the device solver must return bit for bit, not bigsparser's bits.
 *   - (A p + d o p)_j: lane l (0..31) folds the entries lo + l, lo + l + 32, ... of column j in ascending order from 0;
 *     the 32 lane sums are combined by the xor tree 16, 8, 4, 2, 1; then sum + d_j * p_j.
 *   - u.v: chunks of 1024 entries (+0 past n), each a pairwise tree (k + 512, then k + 256, ..., k + 1), chunk sums folded
 *     serially from 0 in chunk order.
 * Built with -O2 -ffp-contract=off: every product and sum rounds once.  OpenMP runs columns and chunks in parallel; the
 * order inside each is fixed, so the thread count does not change a bit.
 *
 * Storage: p[ncol + 1]; first_i == NULL: data interleaves (row, value), column j at data[2 p[j] .. 2 p[j + 1]);
 * first_i != NULL: values only, column j at data[p[j] .. p[j + 1]) for the rows first_i[j], first_i[j] + 1, ...
 */
#include <float.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#define CH 1024

static double chunk_tree(const double *u, const double *v, long long n, long long c) {
  double s[CH / 2];
  int k, w;
  for (k = 0; k < CH / 2; k++) {
    long long i0 = c * CH + k, i1 = i0 + CH / 2;
    double a = i0 < n ? (v ? u[i0] * v[i0] : u[i0] * u[i0]) : 0;
    double b = i1 < n ? (v ? u[i1] * v[i1] : u[i1] * u[i1]) : 0;
    s[k] = a + b;
  }
  for (w = CH / 4; w; w >>= 1)
    for (k = 0; k < w; k++) s[k] = s[k] + s[k + w];
  return s[0];
}

/* u.v (v == NULL: u.u) */
static double dot(const double *u, const double *v, long long n, double *part, int nthreads) {
  long long nch = (n + CH - 1) / CH, c;
  double s = 0;
#pragma omp parallel for schedule(static) num_threads(nthreads)
  for (c = 0; c < nch; c++) part[c] = chunk_tree(u, v, n, c);
  for (c = 0; c < nch; c++) s = s + part[c];
  return s;
}

static void matvec(const double *p, const double *data, const int *first_i, int n, const double *d, int dlen,
                   const double *v, double *t, int nthreads) {
  int j;
#pragma omp parallel for schedule(dynamic, 64) num_threads(nthreads)
  for (j = 0; j < n; j++) {
    long long lo = (long long)p[j], up = (long long)p[j + 1], q;
    double lane[32], nxt[32];
    int l, o;
    for (l = 0; l < 32; l++) lane[l] = 0;
    for (q = lo; q < up; q++) {
      double xv, pv;
      if (first_i) {
        xv = data[q];
        pv = v[first_i[j] + (q - lo)];
      } else {
        xv = data[2 * q + 1];
        pv = v[(long long)data[2 * q]];
      }
      l = (int)((q - lo) % 32);
      lane[l] = lane[l] + xv * pv;
    }
    for (o = 16; o; o >>= 1) {
      for (l = 0; l < 32; l++) nxt[l] = lane[l] + lane[l ^ o];
      memcpy(lane, nxt, sizeof lane);
    }
    t[j] = lane[0] + d[dlen == 1 ? 0 : j] * v[j];
  }
}

/* Returns 0, or -1 on an allocation failure.  x[n] out; iters, error as Eigen's iterations() / error(). */
int spo_solve(const double *p, const double *data, const int *first_i, int n, const double *b, const double *d, int dlen,
              double tol, int maxiter, double *x, int *iters, double *error, int nthreads) {
  long long nch = ((long long)n + CH - 1) / CH;
  double *r = malloc((n ? n : 1) * sizeof(double)), *pv = malloc((n ? n : 1) * sizeof(double));
  double *t = malloc((n ? n : 1) * sizeof(double)), *part = malloc((nch ? nch : 1) * sizeof(double));
  double rhs2, threshold, rn2, abs_new;
  int i = 0, j;
  if (!r || !pv || !t || !part) {
    free(r), free(pv), free(t), free(part);
    return -1;
  }
  for (j = 0; j < n; j++) x[j] = 0, r[j] = b[j], pv[j] = b[j];
  rhs2 = dot(b, NULL, n, part, nthreads);
  if (rhs2 == 0) {
    *iters = 0, *error = 0;
    goto out;
  }
  threshold = tol * tol * rhs2;
  if (threshold < DBL_MIN) threshold = DBL_MIN;
  rn2 = rhs2;
  if (rn2 < threshold) {
    *iters = 0, *error = sqrt(rn2 / rhs2);
    goto out;
  }
  abs_new = rn2;
  while (i < maxiter) {
    double alpha, beta;
    matvec(p, data, first_i, n, d, dlen, pv, t, nthreads);
    alpha = abs_new / dot(pv, t, n, part, nthreads);
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (j = 0; j < n; j++) {
      x[j] = x[j] + alpha * pv[j];
      r[j] = r[j] - alpha * t[j];
    }
    rn2 = dot(r, NULL, n, part, nthreads);
    if (rn2 < threshold) break;
    beta = rn2 / abs_new;
    abs_new = rn2;
#pragma omp parallel for schedule(static) num_threads(nthreads)
    for (j = 0; j < n; j++) pv[j] = r[j] + beta * pv[j];
    i++;
  }
  *iters = i, *error = sqrt(rn2 / rhs2);
out:
  free(r), free(pv), free(t), free(part);
  return 0;
}
