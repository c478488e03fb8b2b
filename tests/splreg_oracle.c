/* CPU oracle of big_spLinReg / big_spLogReg -- test infrastructure only.  The same algorithm and arithmetic as
 * tests/splreg_ref.py (the definition) and the device (bigsnpr_b200/csrc/bsg_splreg.cu): one rounding per operation
 * (built with -ffp-contract=off), exp / log from bsg_ldpred2_auto.cuh, every sum over observations the segmented
 * 256-slot sum.  Fits run in parallel over OpenMP threads; each fit is sequential. */
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include "../bigsnpr_b200/csrc/bsg_ldpred2_auto.cuh"

#define ST 256
#define SEG 8192
#define W_MIN 1e-5

/* the segmented 256-slot sum of v[0 .. n-1] */
static double ssum(const double *v, int n) {
  double tot = 0.0;
  for (int b = 0; b < n || b == 0; b += SEG) {
    double acc[ST];
    for (int t = 0; t < ST; t++) acc[t] = 0.0;
    const int e = n < b + SEG ? n : b + SEG;
    for (int i = b; i < e; i++) acc[(i - b) % ST] += v[i];
    for (int h = ST / 2; h >= 1; h >>= 1)
      for (int t = 0; t < h; t++) acc[t] = acc[t] + acc[t + h];
    tot = b == 0 ? acc[0] : tot + acc[0];
    if (n == 0) break;
  }
  return tot;
}

static double soft(double u, double t) { return u > t ? u - t : (u < -t ? u + t : 0.0); }
static double prob(double eta) { return 1.0 / (1.0 + lda_exp(-eta)); }

typedef struct {
  const double *X; /* [J][nr] standardised, by observation */
  int nr, J, family, max_iter;
  const double *y, *base, *pf;
  double alpha, oma, eps;
  const int *pos;  /* [nr] observations: training, then validation */
  int n;
  double *R, *W, *S, *t1, *t2, *beta, *v, b0;
} Fit;

static double xt(const Fit *F, int j, int q) { return F->X[(size_t)j * F->nr + F->pos[q]]; }

static int cd_pass(Fit *F, double lam, const int *ws, int nws) {
  const int n = F->n, nr = F->nr;
  const double dn = (double)n, la1 = lam * F->alpha, la2 = lam * F->oma;
  double maxd, d0;
  if (F->family == 0) {
    d0 = ssum(F->R, n) / dn;
    for (int q = 0; q < nr; q++) F->R[q] = F->R[q] - d0;
  } else {
    for (int q = 0; q < n; q++) {
      const double p = prob(F->R[q]);
      const double w = p * (1.0 - p);
      F->W[q] = w > W_MIN ? w : W_MIN;
      F->S[q] = F->y[F->pos[q]] - p;
    }
    d0 = ssum(F->S, n) / ssum(F->W, n);
    for (int q = 0; q < nr; q++) F->R[q] = F->R[q] + d0;
    for (int q = 0; q < n; q++) F->S[q] = F->S[q] - F->W[q] * d0;
  }
  F->b0 = F->b0 + d0;
  maxd = fabs(d0);
  double maxb = fabs(F->b0);
  for (int i = 0; i < nws; i++) {
    const int j = ws[i];
    const double bj = F->beta[j];
    double g, h;
    if (F->family == 0) {
      if (F->v[j] < 0) {
        for (int q = 0; q < n; q++) {
          const double x = xt(F, j, q);
          F->t1[q] = x * x;
        }
        F->v[j] = ssum(F->t1, n) / dn;
      }
      h = F->v[j];
      for (int q = 0; q < n; q++) F->t1[q] = xt(F, j, q) * F->R[q];
      g = ssum(F->t1, n) / dn;
    } else {
      for (int q = 0; q < n; q++) {
        const double x = xt(F, j, q);
        F->t1[q] = x * F->S[q];
        F->t2[q] = (F->W[q] * x) * x;
      }
      g = ssum(F->t1, n) / dn;
      h = ssum(F->t2, n) / dn;
    }
    const double pf = F->pf[j];
    const double u = g + h * bj;
    const double bn = soft(u, la1 * pf) / (h + la2 * pf);
    const double d = bn - bj;
    if (d != 0.0) {
      for (int q = 0; q < nr; q++) {
        const double x = xt(F, j, q);
        if (F->family == 0) {
          F->R[q] = F->R[q] - x * d;
        } else {
          F->R[q] = F->R[q] + x * d;
          if (q < n) F->S[q] = F->S[q] - (F->W[q] * x) * d;
        }
      }
      F->beta[j] = bn;
    }
    if (fabs(d) > maxd) maxd = fabs(d);
    if (fabs(bn) > maxb) maxb = fabs(bn);
  }
  return maxd <= F->eps * maxb;
}

static void full_pass(Fit *F, double *z) {
  const int n = F->n;
  const double *res = F->R;
  if (F->family == 1) {
    for (int q = 0; q < n; q++) F->S[q] = F->y[F->pos[q]] - prob(F->R[q]);
    res = F->S;
  }
  for (int j = 0; j < F->J; j++) {
    for (int q = 0; q < n; q++) F->t1[q] = xt(F, j, q) * res[q];
    z[j] = ssum(F->t1, n) / (double)n;
  }
}

static double val_loss(Fit *F) {
  const int n = F->n, nv = F->nr - F->n;
  for (int q = n; q < F->nr; q++) {
    const double e = F->R[q];
    if (F->family == 0) {
      F->t1[q - n] = e * e;
    } else {
      const double l = e > 0 ? e + lda_log(1.0 + lda_exp(-e)) : lda_log(1.0 + lda_exp(e));
      F->t1[q - n] = l - F->y[F->pos[q]] * e;
    }
  }
  const double m = ssum(F->t1, nv) / (double)nv;
  return F->family == 0 ? m : 2.0 * m;
}

/* One fit per (alpha, fold), f = ia * K + k; outputs as bsg_splreg (pbeta / pb0 may be NULL).  Returns 0, or -1 when
 * scratch could not be allocated. */
int splreg_fits(const double *X, int nr, int J, const double *y, const double *base, const double *pf, int family,
                const double *alphas, int nalpha, const int *sets, int K, int nlambda, double step, int nlam_min,
                int n_abort, int dfmax, double eps, int max_iter, double *beta_out, double *b0_out, int *best_out,
                int *len_out, int *msg_out, double *lam_out, double *loss_out, int *nnz_out, int *npass_out,
                double *pbeta, double *pb0) {
  const int F_ = nalpha * K;
  int err = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(| : err)
  for (int f = 0; f < F_; f++) {
    const int k = f % K + 1;
    Fit F;
    memset(&F, 0, sizeof F);
    F.X = X, F.nr = nr, F.J = J, F.family = family, F.max_iter = max_iter, F.y = y, F.base = base, F.pf = pf;
    F.alpha = alphas[f / K], F.oma = 1.0 - F.alpha, F.eps = eps;
    int *pos = malloc(sizeof(int) * nr), *ws = malloc(sizeof(int) * (J + 1));
    unsigned char *wsm = calloc(J + 1, 1), *ever = calloc(J + 1, 1);
    double *mem = malloc(sizeof(double) * ((size_t)nr * 5 + (size_t)J * 4 + 4));
    if (!pos || !ws || !wsm || !ever || !mem) {
      err = 1;
      free(pos), free(ws), free(wsm), free(ever), free(mem);
      continue;
    }
    int q = 0;
    for (int o = 0; o < nr; o++)
      if (sets[o] != k) pos[q++] = o;
    F.n = q;
    for (int o = 0; o < nr; o++)
      if (sets[o] == k) pos[q++] = o;
    F.pos = pos;
    F.R = mem, F.W = mem + nr, F.S = mem + 2 * (size_t)nr, F.t1 = mem + 3 * (size_t)nr, F.t2 = mem + 4 * (size_t)nr;
    F.beta = mem + 5 * (size_t)nr;
    F.v = F.beta + J;
    double *z = F.v + J, *bbest = z + J;
    for (int j = 0; j < J; j++) F.beta[j] = 0.0, F.v[j] = -1.0, bbest[j] = 0.0;
    for (int i = 0; i < nr; i++) {
      const int o = pos[i];
      F.R[i] = family == 1 ? base[o] : y[o] - base[o];
    }
    F.b0 = 0.0;
    int nws = 0;
    for (int j = 0; j < J; j++)
      if (pf[j] == 0.0) ws[nws++] = j, wsm[j] = 1;
    for (int it = 0; it < max_iter; it++)
      if (cd_pass(&F, 0.0, ws, nws)) break;
    full_pass(&F, z);
    double lmax = 0.0;
    for (int j = 0; j < J; j++)
      if (pf[j] > 0) {
        const double r = fabs(z[j]) / (F.alpha * pf[j]);
        if (r > lmax) lmax = r;
      }
    double lam = lmax, lprev = lmax, best_loss = INFINITY, b0best = 0.0;
    int best = 0, stop = -1, kk;
    for (kk = 0; kk < nlambda; kk++) {
      if (kk > 0) lam = lam * step;
      const double thr = F.alpha * (2.0 * lam - lprev), la1 = lam * F.alpha;
      for (int j = 0; j < J; j++) wsm[j] = ever[j] || fabs(z[j]) >= thr * pf[j];
      int passes = 0;
      for (;;) {
        nws = 0;
        for (int j = 0; j < J; j++)
          if (wsm[j]) ws[nws++] = j;
        int conv;
        do {
          conv = cd_pass(&F, lam, ws, nws);
          passes++;
        } while (!conv && passes < max_iter);
        full_pass(&F, z);
        int viol = 0;
        for (int j = 0; j < J; j++)
          if (!wsm[j] && fabs(z[j]) > la1 * pf[j]) wsm[j] = 1, viol = 1;
        if (!viol) break;
      }
      int nz = 0;
      for (int j = 0; j < J; j++)
        if (F.beta[j] != 0.0) ever[j] = 1, nz++;
      const double loss = val_loss(&F);
      const size_t rec = (size_t)f * nlambda + kk;
      lam_out[rec] = lam, loss_out[rec] = loss, nnz_out[rec] = nz, npass_out[rec] = passes;
      if (pbeta) memcpy(pbeta + rec * J, F.beta, sizeof(double) * J);
      if (pb0) pb0[rec] = F.b0;
      if (loss < best_loss) {
        best_loss = loss, best = kk, b0best = F.b0;
        memcpy(bbest, F.beta, sizeof(double) * J);
      }
      lprev = lam;
      if (nz > dfmax) stop = 2;
      else if (kk - best >= n_abort && kk + 1 >= nlam_min) stop = 1;
      else if (kk == nlambda - 1) stop = 0;
      if (stop >= 0) break;
    }
    memcpy(beta_out + (size_t)f * J, bbest, sizeof(double) * J);
    b0_out[f] = b0best, best_out[f] = best, len_out[f] = kk + 1, msg_out[f] = stop;
    free(pos), free(ws), free(wsm), free(ever), free(mem);
  }
  return err ? -1 : 0;
}
