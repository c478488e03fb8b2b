/* CPU oracle of LDpred2-grid over bigsparser's SFBM storage -- test infrastructure only.
 *
 * Literal sequential restatements of src/ldpred2.cpp:9-69 (ldpred2_gibbs_one) and src/ldpred2-sampling.cpp:9-59
 * (ldpred2_gibbs_one_sampling), written from their semantics, one coordinate at a time with incr_mult_col on the CPU, the
 * coordinate arithmetic and the draws those of bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh (the header the device kernel
 * compiles).  Built with -O2 -ffp-contract=off: no FMA contraction.  OpenMP runs the points in parallel, never one point.
 *
 * It includes tests/ldpred2_auto_oracle.c for LDpred2-auto's chain, so that the sparse step of snp_ldpred2_auto
 * (R/LDpred2.R:266-279) can be restated from each chain's final state (lda_ldpred2_auto_state).
 *
 * Storage: as tests/ldpred2_auto_oracle.c.
 */
#include "ldpred2_auto_oracle.c"

typedef struct {
  const double *p, *data;
  const int *first_i;
  int ncol;
  const double *beta_hat, *n_vec;
  int m;
  const int *ind_sub;
  int burn_in, num_iter;
} ldg_in;

/* src/ldpred2.cpp:9-69 for one point: beta_est[m] (NA_real on divergence); moves / entries / sweeps: column updates,
 * the stored values they read and the sweeps run (the diverging one included) */
static int gibbs_one(const ldg_in *in, double h2, double p, int sparse, uint32_t *s, double *beta_est, long long *moves,
                     long long *entries, int *sweeps) {
  const int m = in->m;
  double *curr_beta = calloc(m, sizeof(double)), *avg_beta = calloc(m, sizeof(double));
  double *dotprods = calloc(in->ncol ? in->ncol : 1, sizeof(double));
  const double h2_per_var = h2 / (m * p), inv_odd_p = (1 - p) / p;
  double gap0 = 0;
  long long nmv = 0, nent = 0;
  int j, k, diverged = 0, nsw = 0;
  if (!curr_beta || !avg_beta || !dotprods) {
    free(curr_beta), free(avg_beta), free(dotprods);
    return -1;
  }
  for (j = 0; j < m; j++) gap0 = gap0 + in->beta_hat[j] * in->beta_hat[j];
  gap0 = 2 * gap0;
  for (k = -in->burn_in; k < in->num_iter && !diverged; k++) {
    double gap = 0;
    for (j = 0; j < m; j++) {
      const int j2 = in->ind_sub[j];
      const double res_beta_hat_j = lda_grid_res(in->beta_hat[j], dotprods[j2], curr_beta[j], 0);
      const lda_gcoord_t co = lda_grid_coord(res_beta_hat_j, h2_per_var, in->n_vec[j], inv_odd_p);
      double diff = -curr_beta[j];
      if (!lda_grid_draws(sparse, co.postp, p)) {
        curr_beta[j] = 0;
      } else {
        if (co.postp > lda_unif(s)) {
          curr_beta[j] = lda_rnorm(co.C3, sqrt(co.C4), s);
          diff += curr_beta[j];
          gap += curr_beta[j] * curr_beta[j];
        } else {
          curr_beta[j] = 0;
        }
        if (k >= 0) avg_beta[j] += co.C3 * co.postp;
      }
      if (diff != 0) {
        incr_mult_col(in->p, in->data, in->first_i, j2, diff, dotprods);
        nmv++;
        nent += (long long)(in->p[j2 + 1] - in->p[j2]);
      }
    }
    nsw++;
    if (gap > gap0) diverged = 1;
  }
  for (j = 0; j < m; j++) beta_est[j] = diverged ? na_real() : avg_beta[j] / in->num_iter;
  free(curr_beta), free(avg_beta), free(dotprods);
  if (moves) *moves = nmv;
  if (entries) *entries = nent;
  if (sweeps) *sweeps = nsw;
  return 0;
}

/* src/ldpred2-sampling.cpp:9-59: sample_beta (m x num_iter, column-major) */
static int gibbs_one_sampling(const ldg_in *in, double h2, double p, int sparse, uint32_t *s, double *sample_beta) {
  const int m = in->m;
  double *curr_beta = calloc(m, sizeof(double)), *dotprods = calloc(in->ncol ? in->ncol : 1, sizeof(double));
  const double h2_per_var = h2 / (m * p), inv_odd_p = (1 - p) / p;
  int j, k;
  if (!curr_beta || !dotprods) {
    free(curr_beta), free(dotprods);
    return -1;
  }
  memset(sample_beta, 0, sizeof(double) * m * in->num_iter);
  for (k = -in->burn_in; k < in->num_iter; k++) {
    for (j = 0; j < m; j++) {
      const int j2 = in->ind_sub[j];
      const double res_beta_hat_j = lda_grid_res(in->beta_hat[j], dotprods[j2], curr_beta[j], 1);
      const lda_gcoord_t co = lda_grid_coord(res_beta_hat_j, h2_per_var, in->n_vec[j], inv_odd_p);
      double diff = -curr_beta[j];
      if (!lda_grid_draws(sparse, co.postp, p)) {
        curr_beta[j] = 0;
      } else {
        curr_beta[j] = (co.postp > lda_unif(s)) ? lda_rnorm(co.C3, sqrt(co.C4), s) : 0;
        diff += curr_beta[j];
        if (k >= 0) sample_beta[j + (size_t)k * m] = curr_beta[j];
      }
      if (diff != 0) incr_mult_col(in->p, in->data, in->first_i, j2, diff, dotprods);
    }
  }
  free(curr_beta), free(dotprods);
  return 0;
}

/* npoint points, point g with pv[g], h2[g], sparse[g] from rng[6 g ..]; beta_est m x npoint column-major; with
 * sampling (npoint 1), sample m x num_iter instead.  rng_out (6 x npoint), moves / entries / sweeps / seconds per point:
 * NULL allowed. */
int ldg_ldpred2_grid(const double *p, const double *data, const int *first_i, int ncol, const double *beta_hat,
                     const double *n_vec, int m, const int *ind_sub, int npoint, const double *pv, const double *h2,
                     const int *sparse, int burn_in, int num_iter, int sampling, const uint32_t *rng, double *beta_est,
                     double *sample, uint32_t *rng_out, long long *moves, long long *entries, int *sweeps,
                     double *seconds, int nthreads) {
  const ldg_in in = {p, data, first_i, ncol, beta_hat, n_vec, m, ind_sub, burn_in, num_iter};
  int g, bad = 0;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads) reduction(| : bad)
  for (g = 0; g < npoint; g++) {
    struct timespec t0, t1;
    uint32_t s[6];
    memcpy(s, rng + 6 * g, sizeof s);
    clock_gettime(CLOCK_MONOTONIC, &t0);
    if (sampling ? gibbs_one_sampling(&in, h2[g], pv[g], sparse[g], s, sample)
                 : gibbs_one(&in, h2[g], pv[g], sparse[g], s, beta_est + (size_t)g * m, moves ? moves + g : NULL,
                             entries ? entries + g : NULL, sweeps ? sweeps + g : NULL))
      bad = 1;
    clock_gettime(CLOCK_MONOTONIC, &t1);
    if (rng_out) memcpy(rng_out + 6 * g, s, sizeof s);
    if (seconds) seconds[g] = (t1.tv_sec - t0.tv_sec) + 1e-9 * (t1.tv_nsec - t0.tv_nsec);
  }
  return bad;
}

/* lda_ldpred2_auto, and rng_out (6 x nchain) receives each chain's state after its last sweep */
int lda_ldpred2_auto_state(const double *p, const double *data, const int *first_i, int ncol, const double *beta_hat,
                           const double *n_vec, const double *log_var, int m, const int *ind_sub, int nchain,
                           const double *p_init, double h2_init, int burn_in, int num_iter, int report_step,
                           int no_jump_sign, double shrink_corr, int use_mle, const double *p_bounds,
                           const double *alpha_bounds, double mean_ld, const uint32_t *rng, double *beta_est,
                           double *postp_est, double *corr_est, double *path_p, double *path_h2, double *path_alpha,
                           uint32_t *rng_out, int nthreads) {
  const lda_in in = {p, data, first_i, ncol, beta_hat, n_vec, log_var, m, ind_sub, h2_init, burn_in, num_iter,
                     report_step, no_jump_sign, use_mle, shrink_corr, p_bounds[0], p_bounds[1], alpha_bounds[0],
                     alpha_bounds[1], mean_ld};
  const int T = burn_in + num_iter;
  int c, bad = 0;
#pragma omp parallel for schedule(dynamic, 1) num_threads(nthreads) reduction(| : bad)
  for (c = 0; c < nchain; c++) {
    const size_t o = (size_t)c * m, ot = (size_t)c * T;
    uint32_t s[6];
    memcpy(s, rng + 6 * c, sizeof s);
    if (chain(&in, p_init[c], s, beta_est + o, postp_est + o, corr_est + o, path_p + ot, path_h2 + ot, path_alpha + ot,
              NULL, NULL, NULL))
      bad = 1;
    memcpy(rng_out + 6 * c, s, sizeof s);
  }
  return bad;
}

/* ---- the header's grid functions, for the tests ---- */

/* lda_grid_coord's three values into out[3], from the residual the variant forms */
void ldg_coord_1(double beta_hat, double dotprod, double cur, int sampling, double h2_per_var, double n, double inv_odd_p,
                 double *out) {
  const lda_gcoord_t co = lda_grid_coord(lda_grid_res(beta_hat, dotprod, cur, sampling), h2_per_var, n, inv_odd_p);
  out[0] = co.postp, out[1] = co.C3, out[2] = co.C4;
}

int ldg_offset(uint32_t draws, int lane) { return lda_grid_offset(draws, lane); }
