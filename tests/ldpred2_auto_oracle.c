/* CPU oracle of LDpred2-auto over bigsparser's SFBM storage -- test infrastructure only.
 *
 * A literal sequential restatement of src/ldpred2-auto.cpp:56-202 (ldpred2_gibbs_auto), written from its semantics, with
 * the draws and the math of bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh (the header the device kernel compiles).  Built with
 * -O2 -ffp-contract=off: no FMA contraction.  The MLE step is the header's profile minimiser, its sums taken in the
 * device's fixed order (lda_red below).  OpenMP runs the chains in parallel, never one chain.
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

#include "../bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh"

#define LT 256 /* threads of the device CTA: the order of the MLE's sums */

static double na_real(void) {
  const uint64_t bits = 0x7FF00000000007A2ULL; /* R's NA_real_ */
  double d;
  memcpy(&d, &bits, sizeof d);
  return d;
}

static void incr_mult_col(const double *p, const double *data, const int *first_i, int j2, double shift, double *dot) {
  size_t lo = (size_t)p[j2], up = (size_t)p[j2 + 1], k;
  if (first_i) {
    int i = first_i[j2];
    for (k = lo; k < up; k++, i++) dot[i] += data[k] * shift;
  } else {
    for (k = lo; k < up; k++) dot[(size_t)data[2 * k]] += data[2 * k + 1] * shift;
  }
}

/* sum over k < nb of b_k exp(-t a_k) (b != NULL) or of a_k: v[i] folds k = i, i + LT, ... from 0, then the pairwise tree
 * v[i] += v[i + w] for w = LT / 2 .. 1 */
static double lda_red(const double *a, const double *b, double t, int nb) {
  double v[LT];
  int i, k, w;
  for (i = 0; i < LT; i++) v[i] = 0;
  for (k = 0; k < nb; k++) v[k % LT] += b ? b[k] * lda_exp(-t * a[k]) : a[k];
  for (w = LT / 2; w >= 1; w >>= 1)
    for (i = 0; i < w; i++) v[i] = v[i] + v[i + w];
  return v[0];
}

/* MLE_alpha's step: par = (alpha + 1, sigma2) minimising the objective over [t_lo, t_hi] x [par[1] / 2, 2 par[1]]; nb == 0
 * leaves par as it is */
void lda_mle_fit(const double *a, const double *b, int nb, double t_lo, double t_hi, double *par) {
  lda_golden g;
  double t, s2, C, sum_a, s2_lo, s2_hi;
  if (nb == 0) return;
  sum_a = lda_red(a, NULL, 0, nb);
  s2_lo = par[1] / 2.0, s2_hi = par[1] * 2.0;
  t = lda_golden_start(&g, t_lo, t_hi);
  for (;;) {
    C = lda_red(a, b, t, nb);
    if (!lda_golden_next(&g, lda_mle_profile(t, sum_a, C, nb, s2_lo, s2_hi, &s2), &t)) break;
  }
  C = lda_red(a, b, g.best_t, nb);
  lda_mle_profile(g.best_t, sum_a, C, nb, s2_lo, s2_hi, &s2);
  par[0] = g.best_t, par[1] = s2;
}

/* the profiled objective (for the tests) */
double lda_mle_objective(const double *a, const double *b, int nb, double t, double s2_lo, double s2_hi, double *s2) {
  return lda_mle_profile(t, lda_red(a, NULL, 0, nb), lda_red(a, b, t, nb), nb, s2_lo, s2_hi, s2);
}

typedef struct {
  const double *p, *data;
  const int *first_i;
  int ncol;
  const double *beta_hat, *n_vec, *log_var;
  int m;
  const int *ind_sub;
  double h2_init;
  int burn_in, num_iter, report_step, no_jump_sign, use_mle;
  double shrink, p_lo, p_hi, t_lo, t_hi, mean_ld;
} lda_in;

/* one chain; sample (m x num_iter / report_step) may be NULL; moves / entries: column updates and the values they read */
static int chain(const lda_in *in, double p_init, uint32_t *s, double *beta_est, double *postp_est, double *corr_est,
                 double *path_p, double *path_h2, double *path_alpha, double *sample, long long *moves, long long *entries) {
  const int m = in->m, T = in->burn_in + in->num_iter;
  double *dot = calloc(in->ncol ? in->ncol : 1, sizeof(double));
  double *cb = calloc(m, sizeof(double)), *avg_b = calloc(m, sizeof(double)), *avg_p = calloc(m, sizeof(double));
  double *avg_bh = calloc(m, sizeof(double)), *a = malloc(m * sizeof(double)), *b = malloc(m * sizeof(double));
  int *causal = malloc(m * sizeof(int));
  double gap0 = 0, cur_h2 = 0, h2, p, par[2];
  long long nmv = 0, nent = 0;
  int j, k, ind_report = 0, next_k = in->burn_in + in->report_step - 1, rc = 0;
  if (!dot || !cb || !avg_b || !avg_p || !avg_bh || !a || !b || !causal) {
    rc = -1;
    goto out;
  }
  for (k = 0; k < T; k++) path_p[k] = path_h2[k] = path_alpha[k] = na_real();
  h2 = in->h2_init < 1e-3 ? 1e-3 : in->h2_init;
  p = in->p_lo < p_init ? p_init : in->p_lo;
  p = in->p_hi < p ? in->p_hi : p;
  par[0] = 0, par[1] = h2 / (m * p);
  for (j = 0; j < m; j++) gap0 = gap0 + in->beta_hat[j] * in->beta_hat[j];
  gap0 = 2 * gap0;
  for (k = 0; k < T; k++) {
    const double inv_odd_p = (1 - p) / p, alpha_plus_one = par[0], sigma2 = par[1];
    double gap = 0;
    int nb = 0;
    for (j = 0; j < m; j++) {
      const int j2 = in->ind_sub[j];
      const double prev_beta = cb[j];
      const lda_coord_t co = lda_coord(in->beta_hat[j], dot[j2], prev_beta, in->n_vec[j], in->log_var[j], in->shrink,
                                       in->use_mle, alpha_plus_one, sigma2, inv_odd_p);
      double diff = -prev_beta;
      if (k >= in->burn_in) {
        avg_p[j] += co.postp;
        avg_b[j] += co.C3 * co.postp;
        avg_bh[j] += co.dps;
      }
      if (co.postp > lda_unif(s)) {
        const double samp_beta = lda_rnorm(co.C3, sqrt(co.C4), s);
        if (in->no_jump_sign && (samp_beta * prev_beta) < 0) {
          cb[j] = 0;
        } else {
          cb[j] = samp_beta;
          diff += samp_beta;
          causal[nb++] = j;
          gap += samp_beta * samp_beta;
        }
      } else {
        cb[j] = 0;
      }
      if (diff != 0) {
        cur_h2 += diff * (2 * co.dps + diff);
        incr_mult_col(in->p, in->data, in->first_i, j2, diff, dot);
        nmv++;
        nent += (long long)(in->p[j2 + 1] - in->p[j2]);
      }
    }
    if (gap > gap0) {
      for (j = 0; j < m; j++) avg_b[j] = avg_p[j] = avg_bh[j] = na_real();
      break;
    }
    p = lda_draw_p(nb, m, in->mean_ld, in->p_lo, in->p_hi, s);
    h2 = cur_h2 < 1e-3 ? 1e-3 : cur_h2;
    if (in->use_mle) {
      int kk;
      for (kk = 0; kk < nb; kk++) {
        const int jc = causal[(int)(nb * lda_unif(s))];
        a[kk] = in->log_var[jc];
        b[kk] = cb[jc] * cb[jc];
      }
      lda_mle_fit(a, b, nb, in->t_lo, in->t_hi, par);
    } else {
      par[1] = h2 / (m * p);
    }
    path_p[k] = p;
    path_h2[k] = h2;
    if (in->use_mle) path_alpha[k] = par[0] - 1;
    if (k == next_k) {
      if (sample)
        for (j = 0; j < nb; j++) sample[causal[j] + (size_t)ind_report * m] = cb[causal[j]];
      ind_report++;
      next_k += in->report_step;
    }
  }
  for (j = 0; j < m; j++) {
    beta_est[j] = isnan(avg_b[j]) ? avg_b[j] : avg_b[j] / in->num_iter;
    postp_est[j] = isnan(avg_p[j]) ? avg_p[j] : avg_p[j] / in->num_iter;
    corr_est[j] = isnan(avg_bh[j]) ? avg_bh[j] : avg_bh[j] / in->num_iter;
  }
out:
  free(dot), free(cb), free(avg_b), free(avg_p), free(avg_bh), free(a), free(b), free(causal);
  if (moves) *moves = nmv;
  if (entries) *entries = nent;
  return rc;
}

/* nchain chains, outputs column-major one column per chain (as bsg_ldpred2_auto); rng 6 x nchain; sample may be NULL;
 * moves / entries / seconds per chain, NULL allowed */
int lda_ldpred2_auto(const double *p, const double *data, const int *first_i, int ncol, const double *beta_hat,
                     const double *n_vec, const double *log_var, int m, const int *ind_sub, int nchain, const double *p_init,
                     double h2_init, int burn_in, int num_iter, int report_step, int no_jump_sign, double shrink_corr,
                     int use_mle, const double *p_bounds, const double *alpha_bounds, double mean_ld, const uint32_t *rng,
                     double *beta_est, double *postp_est, double *corr_est, double *path_p, double *path_h2,
                     double *path_alpha, double *sample, long long *moves, long long *entries, double *seconds,
                     int nthreads) {
  const lda_in in = {p, data, first_i, ncol, beta_hat, n_vec, log_var, m, ind_sub, h2_init, burn_in, num_iter,
                     report_step, no_jump_sign, use_mle, shrink_corr, p_bounds[0], p_bounds[1], alpha_bounds[0],
                     alpha_bounds[1], mean_ld};
  const int T = burn_in + num_iter, nrep = num_iter / report_step;
  int c, bad = 0;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads) reduction(| : bad)
  for (c = 0; c < nchain; c++) {
    struct timespec t0, t1;
    const size_t o = (size_t)c * m, ot = (size_t)c * T;
    uint32_t s[6];
    memcpy(s, rng + 6 * c, sizeof s);
    clock_gettime(CLOCK_MONOTONIC, &t0);
    if (sample) memset(sample + o * nrep, 0, sizeof(double) * m * nrep);
    if (chain(&in, p_init[c], s, beta_est + o, postp_est + o, corr_est + o, path_p + ot, path_h2 + ot, path_alpha + ot,
              sample ? sample + o * nrep : NULL, moves ? moves + c : NULL, entries ? entries + c : NULL))
      bad = 1;
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (seconds) seconds[c] = (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
  }
  return bad;
}

/* ---- the header's functions, for the tests ---- */

void lda_unif_n(uint32_t *s, int n, double *out) {
  int i;
  for (i = 0; i < n; i++) out[i] = lda_unif(s);
}

void lda_skip_k(uint32_t *s, uint64_t k) {
  lda_mat pw[64];
  lda_pow2_table(pw, 64);
  lda_skip(s, k, pw);
}

void lda_jump(uint32_t *s) { lda_jump127(s); }

void lda_exp_n(const double *x, int n, double *out) {
  int i;
  for (i = 0; i < n; i++) out[i] = lda_exp(x[i]);
}

void lda_log_n(const double *x, int n, double *out) {
  int i;
  for (i = 0; i < n; i++) out[i] = lda_log(x[i]);
}

void lda_qnorm_n(const double *x, int n, double *out) {
  int i;
  for (i = 0; i < n; i++) out[i] = lda_qnorm(x[i]);
}

void lda_rnorm_n(double mu, double sigma, uint32_t *s, int n, double *out) {
  int i;
  for (i = 0; i < n; i++) out[i] = lda_rnorm(mu, sigma, s);
}

void lda_rbeta_n(double a, double b, uint32_t *s, int n, double *out) {
  int i;
  for (i = 0; i < n; i++) out[i] = lda_rbeta(a, b, s);
}

double lda_draw_p_1(int nb, int m, double mean_ld, double p_lo, double p_hi, uint32_t *s) {
  return lda_draw_p(nb, m, mean_ld, p_lo, p_hi, s);
}

/* lda_coord's four values into out[4] */
void lda_coord_1(double beta_hat, double dotprod, double cur, double n, double log_var, double shrink, int use_mle,
                 double alpha_plus_one, double sigma2, double inv_odd_p, double *out) {
  const lda_coord_t co = lda_coord(beta_hat, dotprod, cur, n, log_var, shrink, use_mle, alpha_plus_one, sigma2, inv_odd_p);
  out[0] = co.postp, out[1] = co.C3, out[2] = co.C4, out[3] = co.dps;
}
