// bsg_splreg.cu -- penalised regression over the resident genotypes (bigstatsr's big_spLinReg / big_spLogReg, elastic
// net with cross-model selection and averaging; not vendored in the reference, restated in DESIGN.md section 4.19).
//
// Every fit f = (alpha index, fold k) of a call runs on one thread-block cluster of CS = 8 CTAs, the whole lambda path
// in one launch: state (residual or eta, IRLS weights, beta, working set, path records) stays in device memory and the
// host reads the results back once.
//   - k_sp_stats: the centre and scale of every selected column over the ind.train observations, one warp per column,
//     and the NA flag of each (a refusal).
//   - k_splreg: per fit, the null fit of the unpenalised columns, lambda_max, then per lambda the sequential strong rule,
//     coordinate descent over the working set, a full gradient pass (the KKT check, reused as the next lambda's
//     screening), the validation loss and the stopping rules.
// Every sum over observations is the segmented sum of tests/splreg_ref.py: 8,192-position segments, each a 256-slot sum
// (slot t accumulates positions t, t + 256, ... from +0, then the slots are halved pairwise), added in segment order.
// Each segment belongs to one CTA of the cluster; the segment sums are combined in order through distributed shared
// memory, so a fit's bytes depend on its problem alone -- not on the other fits, the grid, the cluster size or the
// column order.  Every floating operation is an __d*_rn intrinsic (no contraction) and exp / log are the shared fdlibm
// restatement, so the NumPy and C restatements in tests/ reproduce the device byte for byte.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <math.h>
#include <vector>

#include "bsg_internal.cuh"
#include "bsg_ldpred2_auto.cuh"

#include <cooperative_groups.h>
namespace cg = cooperative_groups;

namespace bsg {
namespace splreg {

constexpr int ST = 256;  // threads per CTA = slots of every sum over observations
constexpr double W_MIN = 1e-5;   // logistic: IRLS weights p (1 - p) are floored here
constexpr double SD_MIN = 1e-8;  // columns whose sd over ind.train is not above this are dropped

constexpr int SEG = 8192;  // positions per segment of every sum over observations
constexpr int CS = 8;      // CTAs per fit (one thread-block cluster)
constexpr int SL = 16;     // segments one CTA may own: n_train <= SEG * CS * SL
constexpr int64_t NMAX = (int64_t)SEG * CS * SL;

// The column sources, a compile-time parameter of both kernels: columns j < G come from the source, columns j >= G are
// the covariates.  Cols reads the resident genotypes; Dense<T> reads a staged column-major block of float or double.
struct Cols {
  const uint8_t *P;    // hard calls: copy A; dosages: the value copy
  int64_t stride;
  double D;            // dosages: x = byte / D; hard calls: 0 (x = the 2-bit code)
  const int *rows;     // [nr] 0-based sample of each observation
  const int *lines;    // [G] genotype lines
  const double *cov;   // [J - G][nr] covariates, column-major by observation
  int nr, G;
};

template <class T>
struct Dense {
  const T *X;          // [ncol][nr] the staged block: X[ind_row, ind_col], column-major by observation
  const int *lines;    // [G] columns of the block
  const double *cov;   // [J - G][nr] covariates, column-major by observation
  int nr, G;
};

// column j at observation o, sample row `row`
__device__ __forceinline__ double xraw(const Cols &c, int j, int o, int row) {
  if (j >= c.G) return c.cov[(int64_t)(j - c.G) * c.nr + o];
  const uint8_t *p = c.P + (int64_t)c.lines[j] * c.stride;
  if (c.D > 0) return __ddiv_rn((double)p[row], c.D);
  return (double)((p[row >> 2] >> (2 * (row & 3))) & 3);
}

// the block is staged by observation, so the sample row is not needed; float widens to double exactly
template <class T>
__device__ __forceinline__ double xraw(const Dense<T> &c, int j, int o, int) {
  if (j >= c.G) return c.cov[(int64_t)(j - c.G) * c.nr + o];
  return (double)c.X[(int64_t)c.lines[j] * c.nr + o];
}

__device__ __forceinline__ int row_of(const Cols &c, int o) { return c.rows[o]; }
template <class T>
__device__ __forceinline__ int row_of(const Dense<T> &, int o) { return o; }

// a refused cell of column j < G at observation o: an NA code, or a non-finite value
__device__ __forceinline__ bool cell_bad(const Cols &c, int j, int o, const uint8_t *raw, int n, const int *lut) {
  const int row = c.rows[o];
  if (c.D > 0) return lut[raw[(int64_t)c.lines[j] * n + row]] < 0;
  return ((c.P[(int64_t)c.lines[j] * c.stride + (row >> 2)] >> (2 * (row & 3))) & 3) == 3;
}

template <class T>
__device__ __forceinline__ bool cell_bad(const Dense<T> &c, int j, int o, const uint8_t *, int, const int *) {
  return !isfinite(c.X[(int64_t)c.lines[j] * c.nr + o]);
}

// the 256-slot sum of f(b .. e-1) by one warp (slot t: positions b + t, b + t + 256, ...; then the halving tree)
template <class F>
__device__ __forceinline__ double warp_sum256(int b, int e, F f) {
  const int lane = threadIdx.x & 31;
  double acc[8] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
  for (int c = b; c < e; c += ST) {
#pragma unroll
    for (int q = 0; q < 8; q++) {
      const int i = c + lane + 32 * q;
      if (i < e) acc[q] = __dadd_rn(acc[q], f(i));
    }
  }
#pragma unroll
  for (int q = 0; q < 4; q++) acc[q] = __dadd_rn(acc[q], acc[q + 4]);
  acc[0] = __dadd_rn(acc[0], acc[2]);
  acc[1] = __dadd_rn(acc[1], acc[3]);
  double v = __dadd_rn(acc[0], acc[1]);
#pragma unroll
  for (int h = 16; h >= 1; h >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, h));
  return __shfl_sync(0xffffffffu, v, 0);
}

// the segmented sum of f(0 .. n-1) by one warp: each SEG-position segment's 256-slot sum, added in segment order
template <class F>
__device__ __forceinline__ double warp_sum(int n, F f) {
  double tot = 0.0;
  for (int b = 0; b < n; b += SEG) {
    const double v = warp_sum256(b, min(n, b + SEG), f);
    tot = b == 0 ? v : __dadd_rn(tot, v);
  }
  return tot;
}

template <class Src>
__global__ void __launch_bounds__(ST) k_sp_stats(const Src c, int J, const uint8_t *raw, int n, const int *lut,
                                                 double *center, double *scale, uint8_t *na) {
  const int j = blockIdx.x * (ST / 32) + (threadIdx.x >> 5);
  if (j >= J) return;
  int bad = 0;
  if (j < c.G)
    for (int o = threadIdx.x & 31; o < c.nr; o += 32) bad |= cell_bad(c, j, o, raw, n, lut);
  bad = __any_sync(0xffffffffu, bad);
  const double ctr = __ddiv_rn(warp_sum(c.nr, [&](int o) { return xraw(c, j, o, row_of(c, o)); }), (double)c.nr);
  const double var = __ddiv_rn(warp_sum(c.nr, [&](int o) {
    const double d = __dsub_rn(xraw(c, j, o, row_of(c, o)), ctr);
    return __dmul_rn(d, d);
  }), (double)c.nr);
  if ((threadIdx.x & 31) == 0) {
    center[j] = ctr;
    scale[j] = __dsqrt_rn(var);
    na[j] = (uint8_t)bad;
  }
}

template <class Src>
struct FArgs {
  Src c;
  int J;
  const double *center, *iscale, *pf;  // [J]
  const double *y, *base;              // [nr] by observation
  const int *pos;                      // [K][nr] observation at each position: the fold's training rows, then its own
  const int *prow;                     // [K][nr] sample row at each position
  const int *ntr;                      // [K] training positions of each fold
  const double *alphas;
  int K, family, nlambda, nlam_min, n_abort, dfmax, max_iter;
  double eps, step;                    // step = lambda_min_ratio^(1 / (nlambda - 1))
  double *r, *w, *s;                   // [F][nr]: linear r = y - eta; logistic r = eta, w weights, s working residual
  double *beta, *z, *v;                // [F][J]
  uint8_t *flag;                       // [F][CS][J] bit 0 working set, bit 1 ever active (one copy per CTA)
  int *wl;                             // [F][CS][J] working set list (one copy per CTA)
  double *bbest, *b0best;              // [F][J], [F]
  int *best, *len, *msg;               // [F]
  double *lam, *loss;                  // [F][nlambda]
  int *nnz, *npass;                    // [F][nlambda]
  double *pbeta, *pb0;                 // NULL, or [F][nlambda][J] and [F][nlambda]
};

__device__ __forceinline__ double soft(double u, double t) {
  return u > t ? __dsub_rn(u, t) : (u < -t ? __dadd_rn(u, t) : 0.0);
}

// log(1 + e^eta) - y eta, the binomial loss of one observation
__device__ __forceinline__ double binom_loss(double eta, double y) {
  const double l = eta > 0 ? __dadd_rn(eta, lda_log(__dadd_rn(1.0, lda_exp(-eta))))
                           : lda_log(__dadd_rn(1.0, lda_exp(eta)));
  return __dsub_rn(l, __dmul_rn(y, eta));
}

__device__ __forceinline__ double prob(double eta) { return __ddiv_rn(1.0, __dadd_rn(1.0, lda_exp(-eta))); }

struct Smem {
  double red[2][SL][ST];   // slot values of the CTA's segments
  double seg[2][2][SL];    // [buffer][value][local segment] segment sums, read by the whole cluster
  double bc[2];
  double mx[ST / 32];
  int cnt;
};

// One fit per cluster of CS CTAs.  Segment s of the training positions [0, n) (and of the validation positions [n, nr),
// counted from n) belongs to CTA s % CS: that CTA alone updates the residuals there and forms the segment's 256-slot
// sum; every CTA then adds all segment sums in segment order through distributed shared memory, so all CTAs hold the
// same bits and take the same decisions.  Column loops over all positions (the full pass) give whole columns to warps,
// columns split over the cluster.
template <class Src>
__global__ void __launch_bounds__(ST) k_splreg(const FArgs<Src> a) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  Smem &sm = *reinterpret_cast<Smem *>(smem_raw);
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int f = blockIdx.x / CS, t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int k = f % a.K, J = a.J, nr = a.c.nr;
  const bool logit = a.family == 1;
  const double alpha = a.alphas[f / a.K], oma = __dsub_rn(1.0, alpha);
  const int n = a.ntr[k], nv = nr - n;
  const double dn = (double)n;
  const int *pos = a.pos + (int64_t)k * nr, *prow = a.prow + (int64_t)k * nr;
  double *R = a.r + (int64_t)f * nr, *W = a.w ? a.w + (int64_t)f * nr : nullptr, *S = a.s ? a.s + (int64_t)f * nr : nullptr;
  double *beta = a.beta + (int64_t)f * J, *z = a.z + (int64_t)f * J, *vc = a.v + (int64_t)f * J;
  uint8_t *flag = a.flag + ((int64_t)f * CS + rank) * J;
  int *wl = a.wl + ((int64_t)f * CS + rank) * J;
  const bool lead = rank == 0;
  auto xt = [&](int j, double cj, double ij, int q) {
    return __dmul_rn(__dsub_rn(xraw(a.c, j, pos[q], prow[q]), cj), ij);
  };
  // this CTA's positions of the range [b, e): segments b + (rank + CS u) SEG
  auto for_own = [&](int b, int e, auto &&body) {
    for (int s0 = b + rank * SEG; s0 < e; s0 += CS * SEG)
      for (int q = s0 + t; q < min(e, s0 + SEG); q += ST) body(q);
  };
  int buf = 0;
  // the segmented sum over [b, b + m) of NV values per position, on every thread of every CTA of the cluster
  auto cl_sum = [&](int b, int m, int NV, auto &&val, double *out) {
    const int nseg = (m + SEG - 1) / SEG;
    int u = 0;
    for (int s = rank; s < nseg; s += CS, u++) {
      double acc0 = 0.0, acc1 = 0.0;
      const int e = min(m, (s + 1) * SEG);
      for (int i = s * SEG + t; i < e; i += ST) {
        double v0, v1;
        val(b + i, v0, v1);
        acc0 = __dadd_rn(acc0, v0);
        if (NV > 1) acc1 = __dadd_rn(acc1, v1);
      }
      sm.red[0][u][t] = acc0;
      sm.red[1][u][t] = acc1;
    }
    const int nloc = u;
    __syncthreads();
    for (int h = ST / 2; h >= 32; h >>= 1) {
      if (t < h)
        for (int uu = 0; uu < nloc; uu++)
          for (int c = 0; c < NV; c++) sm.red[c][uu][t] = __dadd_rn(sm.red[c][uu][t], sm.red[c][uu][t + h]);
      __syncthreads();
    }
    for (int uu = warp; uu < nloc; uu += ST / 32)
      for (int c = 0; c < NV; c++) {
        double v = sm.red[c][uu][lane];
        for (int h = 16; h >= 1; h >>= 1) v = __dadd_rn(v, __shfl_xor_sync(0xffffffffu, v, h));
        if (lane == 0) sm.seg[buf][c][uu] = v;
      }
    cl.sync();
    if (t == 0) {
      for (int c = 0; c < NV; c++) {
        double tot = 0.0;
        for (int s = 0; s < nseg; s++) {
          const double *rs = cl.map_shared_rank(&sm.seg[buf][c][0], s % CS);
          tot = s == 0 ? rs[s / CS] : __dadd_rn(tot, rs[s / CS]);
        }
        sm.bc[c] = tot;
      }
    }
    __syncthreads();
    for (int c = 0; c < NV; c++) out[c] = sm.bc[c];
    __syncthreads();
    buf ^= 1;
  };
  for_own(0, n, [&](int q) { R[q] = logit ? a.base[pos[q]] : __dsub_rn(a.y[pos[q]], a.base[pos[q]]); });
  for_own(n, nr, [&](int q) { R[q] = logit ? a.base[pos[q]] : __dsub_rn(a.y[pos[q]], a.base[pos[q]]); });
  for (int j = t; j < J; j += ST) {
    if (lead) beta[j] = 0.0, vc[j] = -1.0;
    flag[j] = a.pf[j] == 0.0 ? 1 : 0;
  }
  cl.sync();
  double b0 = 0.0;
  double sums[2];

  // working-set list from bit 0 of flag, in column order (warp 0, one ballot per 32 columns)
  auto build_list = [&]() {
    __syncthreads();
    if (warp == 0) {
      int cnt = 0;
      for (int j0 = 0; j0 < J; j0 += 32) {
        const int j = j0 + lane;
        const bool in = j < J && (flag[j] & 1);
        const unsigned m = __ballot_sync(0xffffffffu, in);
        if (in) wl[cnt + __popc(m & ((1u << lane) - 1))] = j;
        cnt += __popc(m);
      }
      if (lane == 0) sm.cnt = cnt;
    }
    __syncthreads();
  };

  // one coordinate-descent pass over the working set at lambda; true when converged
  auto cd_pass = [&](double lam) -> bool {
    const double la1 = __dmul_rn(lam, alpha), la2 = __dmul_rn(lam, oma);
    double maxd, maxb;
    if (!logit) {
      cl_sum(0, n, 1, [&](int q, double &v0, double &) { v0 = R[q]; }, sums);
      const double d0 = __ddiv_rn(sums[0], dn);
      for_own(0, n, [&](int q) { R[q] = __dsub_rn(R[q], d0); });
      for_own(n, nr, [&](int q) { R[q] = __dsub_rn(R[q], d0); });
      b0 = __dadd_rn(b0, d0);
      maxd = fabs(d0);
    } else {
      // p, the weights and the working residual from eta, afresh at the start of every pass
      for_own(0, n, [&](int q) {
        const double p = prob(R[q]);
        W[q] = fmax(__dmul_rn(p, __dsub_rn(1.0, p)), W_MIN);
        S[q] = __dsub_rn(a.y[pos[q]], p);
      });
      cl_sum(0, n, 2, [&](int q, double &v0, double &v1) { v0 = S[q], v1 = W[q]; }, sums);
      const double d0 = __ddiv_rn(sums[0], sums[1]);
      for_own(0, n, [&](int q) {
        R[q] = __dadd_rn(R[q], d0);
        S[q] = __dsub_rn(S[q], __dmul_rn(W[q], d0));
      });
      for_own(n, nr, [&](int q) { R[q] = __dadd_rn(R[q], d0); });
      b0 = __dadd_rn(b0, d0);
      maxd = fabs(d0);
    }
    maxb = fabs(b0);
    const int nws = sm.cnt;
    for (int i = 0; i < nws; i++) {
      const int j = wl[i];
      const double bj = beta[j], cj = a.center[j], ij = a.iscale[j];
      double g, h;
      if (!logit) {
        h = vc[j];
        if (h < 0) {
          cl_sum(0, n, 1, [&](int q, double &v0, double &) {
            const double x = xt(j, cj, ij, q);
            v0 = __dmul_rn(x, x);
          }, sums);
          h = __ddiv_rn(sums[0], dn);
        }
        cl_sum(0, n, 1, [&](int q, double &v0, double &) { v0 = __dmul_rn(xt(j, cj, ij, q), R[q]); }, sums);
        g = __ddiv_rn(sums[0], dn);
      } else {
        cl_sum(0, n, 2, [&](int q, double &v0, double &v1) {
          const double x = xt(j, cj, ij, q);
          v0 = __dmul_rn(x, S[q]);
          v1 = __dmul_rn(__dmul_rn(W[q], x), x);
        }, sums);
        g = __ddiv_rn(sums[0], dn);
        h = __ddiv_rn(sums[1], dn);
      }
      const double pf = a.pf[j];
      const double u = __dadd_rn(g, __dmul_rn(h, bj));
      const double bn = __ddiv_rn(soft(u, __dmul_rn(la1, pf)), __dadd_rn(h, __dmul_rn(la2, pf)));
      const double d = __dsub_rn(bn, bj);
      if (d != 0.0) {
        for_own(0, n, [&](int q) {
          const double x = xt(j, cj, ij, q);
          if (!logit) {
            R[q] = __dsub_rn(R[q], __dmul_rn(x, d));
          } else {
            R[q] = __dadd_rn(R[q], __dmul_rn(x, d));
            S[q] = __dsub_rn(S[q], __dmul_rn(__dmul_rn(W[q], x), d));
          }
        });
        for_own(n, nr, [&](int q) {
          const double x = xt(j, cj, ij, q);
          R[q] = logit ? __dadd_rn(R[q], __dmul_rn(x, d)) : __dsub_rn(R[q], __dmul_rn(x, d));
        });
      }
      // beta[j] and vc[j] are read again only after later cluster barriers
      if (lead && t == 0) {
        beta[j] = bn;
        if (!logit) vc[j] = h;
      }
      maxd = fmax(maxd, fabs(d));
      maxb = fmax(maxb, fabs(bn));
    }
    cl.sync();
    return maxd <= __dmul_rn(a.eps, maxb);
  };

  // z_j = x_j' r / n at the training positions for every column (logistic: r = y - p, from eta afresh); columns split
  // over the cluster, whole columns per warp
  auto full_pass = [&]() {
    if (logit) {
      for_own(0, n, [&](int q) { S[q] = __dsub_rn(a.y[pos[q]], prob(R[q])); });
      cl.sync();
    }
    const double *res = logit ? S : R;
    for (int j = rank * (ST / 32) + warp; j < J; j += CS * (ST / 32)) {
      const double cj = a.center[j], ij = a.iscale[j];
      const double sj = warp_sum(n, [&](int q) { return __dmul_rn(xt(j, cj, ij, q), res[q]); });
      if (lane == 0) z[j] = __ddiv_rn(sj, dn);
    }
    cl.sync();
  };

  // null fit: the intercept and the unpenalised columns
  build_list();
  for (int it = 0; it < a.max_iter; it++)
    if (cd_pass(0.0)) break;
  full_pass();
  double lmax = 0.0;
  for (int j = t; j < J; j += ST)
    if (a.pf[j] > 0) lmax = fmax(lmax, __ddiv_rn(fabs(z[j]), __dmul_rn(alpha, a.pf[j])));
  for (int h = 16; h >= 1; h >>= 1) lmax = fmax(lmax, __shfl_xor_sync(0xffffffffu, lmax, h));
  if (lane == 0) sm.mx[warp] = lmax;
  __syncthreads();
  lmax = 0.0;
  for (int u = 0; u < ST / 32; u++) lmax = fmax(lmax, sm.mx[u]);
  __syncthreads();

  double lam = lmax, lprev = lmax, best_loss = __longlong_as_double(0x7ff0000000000000LL);
  int best = 0, stop = -1, kk = 0;
  for (kk = 0; kk < a.nlambda; kk++) {
    if (kk > 0) lam = __dmul_rn(lam, a.step);
    const double thr = __dmul_rn(alpha, __dsub_rn(__dmul_rn(2.0, lam), lprev));
    for (int j = t; j < J; j += ST)
      if ((flag[j] & 2) || fabs(z[j]) >= __dmul_rn(thr, a.pf[j])) flag[j] |= 1;
      else flag[j] &= 2;
    build_list();
    const double la1 = __dmul_rn(lam, alpha);
    int passes = 0;
    while (true) {
      bool conv;
      do {
        conv = cd_pass(lam);
        passes++;
      } while (!conv && passes < a.max_iter);
      full_pass();
      int viol = 0;
      for (int j = t; j < J; j += ST)
        if (!(flag[j] & 1) && fabs(z[j]) > __dmul_rn(la1, a.pf[j])) flag[j] |= 1, viol = 1;
      if (!__syncthreads_or(viol)) break;  // every CTA of the cluster reads the same z: the same decision
      build_list();
    }
    int cnt = 0;
    for (int j = t; j < J; j += ST)
      if (beta[j] != 0.0) flag[j] |= 2, cnt++;
    for (int h = 16; h >= 1; h >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, h);
    if (lane == 0) sm.mx[warp] = (double)cnt;
    __syncthreads();
    int nz = 0;
    for (int u = 0; u < ST / 32; u++) nz += (int)sm.mx[u];
    __syncthreads();
    cl_sum(n, nv, 1, [&](int q, double &v0, double &) {
      v0 = logit ? binom_loss(R[q], a.y[pos[q]]) : __dmul_rn(R[q], R[q]);
    }, sums);
    double loss = __ddiv_rn(sums[0], (double)nv);
    if (logit) loss = __dmul_rn(2.0, loss);
    const int64_t rec = (int64_t)f * a.nlambda + kk;
    if (lead && t == 0) {
      a.lam[rec] = lam;
      a.loss[rec] = loss;
      a.nnz[rec] = nz;
      a.npass[rec] = passes;
      if (a.pb0) a.pb0[rec] = b0;
    }
    if (lead && a.pbeta)
      for (int j = t; j < J; j += ST) a.pbeta[rec * J + j] = beta[j];
    if (loss < best_loss) {
      best_loss = loss, best = kk;
      if (lead) {
        for (int j = t; j < J; j += ST) a.bbest[(int64_t)f * J + j] = beta[j];
        if (t == 0) a.b0best[f] = b0;
      }
    }
    lprev = lam;
    if (nz > a.dfmax) stop = 2;
    else if (kk - best >= a.n_abort && kk + 1 >= a.nlam_min) stop = 1;
    else if (kk == a.nlambda - 1) stop = 0;
    cl.sync();
    if (stop >= 0) break;
  }
  if (lead && t == 0) {
    a.best[f] = best;
    a.len[f] = kk + 1;
    a.msg[f] = stop;
  }
}

static thread_local double g_last_ms = 0, g_stage_ms = 0;

static bool finite_all(const double *p, int64_t n) {
  for (int64_t i = 0; i < n; i++)
    if (!std::isfinite(p[i])) return false;
  return true;
}

// What an entry point hands the driver: the kernels' column source Src, the bounds n / m of ind_row / ind_col, the
// stream, the device bytes stage() allocates (counted in the memory check), stage() itself (makes the nc selected columns
// readable as source columns 0..nc-1 for the statistics), line() (the source column of selected column c in the fit),
// what k_sp_stats' NA-code check reads, and the refusal of a flagged column.

// the resident genotypes of a handle: hard calls, or the value copy of a dosage FBM
struct BedOp {
  using Src = Cols;
  bsg_bed *h;
  int n, m;
  cudaStream_t s;
  const uint8_t *raw;
  const int *lut = nullptr;
  const char *bad_msg = "Column %d holds a missing value on a training row; impute it first (snp_fastImputeSimple).";
  size_t stage_bytes(int, int) const { return 0; }
  int stage(const std::vector<int> &row0, const std::vector<int> &col0, int nc, Bufs &b, Cols &cs) {
    Genotypes g;
    BSG_TRY(genotypes(h, b, &g));
    int *d_rows, *d_cols;
    b.up(&d_rows, row0, s);
    b.up(&d_cols, col0.data(), (size_t)nc, s);
    BSG_TRY(b.status("big_spLinReg scratch"));
    lut = g.lut;
    cs.P = g.P;
    cs.stride = g.stride;
    cs.D = g.D;
    cs.rows = d_rows, cs.lines = d_cols;
    return BSG_OK;
  }
  int line(int c, const std::vector<int> &col0) const { return col0[c]; }
};

// pinned host buffers of the dense staging, freed with their events
struct Pinned {
  void *p[2] = {nullptr, nullptr};
  cudaEvent_t ev[2] = {nullptr, nullptr};
  ~Pinned() {
    for (int i = 0; i < 2; i++) {
      if (ev[i]) cudaEventSynchronize(ev[i]), cudaEventDestroy(ev[i]);
      if (p[i]) cudaFreeHost(p[i]);
    }
  }
};

// a host column-major matrix of T (leading dimension ld): X[ind_row, ind_col] is gathered into pinned chunks of whole
// columns and uploaded once, so the block lives on the device as nc columns of nr observations
template <class T>
struct DenseOp {
  using Src = Dense<T>;
  static constexpr size_t CHUNK = (size_t)64 << 20;  // bytes per pinned buffer (two of them)
  const T *X;
  int64_t ld;
  int n, m;
  cudaStream_t s;
  const uint8_t *raw = nullptr;
  const int *lut = nullptr;
  const char *bad_msg = "Column %d holds a non-finite value on a training row.";
  size_t stage_bytes(int nr, int nc) const { return (size_t)nr * nc * sizeof(T) + (size_t)nc * sizeof(int); }
  int stage(const std::vector<int> &row0, const std::vector<int> &col0, int nc, Bufs &b, Dense<T> &cs) {
    const int nr = (int)row0.size();
    std::vector<int> iota(nc);
    for (int c = 0; c < nc; c++) iota[c] = c;
    T *d_X;
    int *d_cols;
    b.alloc(&d_X, (size_t)nr * nc);
    b.up(&d_cols, iota, s);
    BSG_TRY(b.status("big_spLinReg scratch"));
    bool contiguous = true;  // ind_row a run of consecutive rows: one copy per column
    for (int r = 1; r < nr && contiguous; r++) contiguous = row0[r] == row0[0] + r;
    const size_t colb = (size_t)nr * sizeof(T);
    const int per = (int)std::max<size_t>(1, std::min<size_t>(CHUNK / std::max<size_t>(colb, 1), (size_t)nc));
    Pinned pin;
    for (int i = 0; i < 2 && nc > 0; i++) {
      BSG_CUDA(cudaMallocHost(&pin.p[i], (size_t)per * colb));
      BSG_CUDA(cudaEventCreateWithFlags(&pin.ev[i], cudaEventDisableTiming));
    }
    for (int c0 = 0, u = 0; c0 < nc; c0 += per, u ^= 1) {
      const int cnt = std::min(per, nc - c0);
      BSG_CUDA(cudaEventSynchronize(pin.ev[u]));
      T *dst = static_cast<T *>(pin.p[u]);
      for (int c = 0; c < cnt; c++, dst += nr) {
        const T *src = X + (int64_t)col0[c0 + c] * ld;
        if (contiguous) std::copy(src + row0[0], src + row0[0] + nr, dst);
        else
          for (int r = 0; r < nr; r++) dst[r] = src[row0[r]];
      }
      BSG_CUDA(cudaMemcpyAsync(d_X + (size_t)c0 * nr, pin.p[u], (size_t)cnt * colb, cudaMemcpyHostToDevice, s));
      BSG_CUDA(cudaEventRecord(pin.ev[u], s));
    }
    BSG_CUDA(cudaStreamSynchronize(s));
    cs.X = d_X, cs.lines = d_cols;
    return BSG_OK;
  }
  int line(int c, const std::vector<int> &) const { return c; }
};

// validation, folds, memory check, staging, column statistics, the fits' launch, read-back and unpermute, for any
// operand (bsg_splreg and bsg_splreg_dense)
template <class Op>
static int splreg_drive(Op &op, const int *ind_row, int nr, const int *ind_col, int nc, int family, const double *y,
                        const double *covar, int Kc, const double *base, const double *pf_X, const double *pf_covar,
                        const double *alphas, int nalpha, const int *ind_sets, int K, int nlambda,
                        double lambda_min_ratio, int nlam_min, int n_abort, int dfmax, double eps, int max_iter,
                        double power_scale, double power_adaptive, double *center, double *scale, uint8_t *kept,
                        double *beta, double *intercept, int *best, int *length, int *message, double *lambda,
                        double *loss, int *nnz, int *npass, double *path_beta, double *path_b0) {
  if (!ind_row) nr = op.n;
  if (!ind_col) nc = op.m;
  if (nr < 2 || nc < 0 || Kc < 0 || (Kc > 0 && !covar)) return fail(BSG_ERR_ARG, "Incompatibility between dimensions.");
  if (family != 0 && family != 1) return fail(BSG_ERR_ARG, "family must be 0 (linear) or 1 (logistic).");
  if (power_scale != 1.0) return fail(BSG_ERR_ARG, "Only 'power_scale = 1' is supported on the device.");
  if (power_adaptive != 0.0) return fail(BSG_ERR_ARG, "Only 'power_adaptive = 0' is supported on the device.");
  if (nalpha < 1 || !alphas) return fail(BSG_ERR_ARG, "'alphas' must not be empty.");
  for (int i = 0; i < nalpha; i++)
    if (!(alphas[i] > 0 && alphas[i] <= 1)) return fail(BSG_ERR_ARG, "'alphas' must be in (0, 1].");
  if (K < 2) return fail(BSG_ERR_ARG, "'K' must be at least 2.");
  if (nlambda < 1 || !(lambda_min_ratio > 0 && lambda_min_ratio < 1) || nlam_min < 1 || n_abort < 1 || dfmax < 0 ||
      !(eps > 0) || max_iter < 1)
    return fail(BSG_ERR_ARG, "Invalid path or stopping parameter.");
  if (!y || !ind_sets || !center || !scale || !kept || !beta || !intercept || !best || !length || !message || !lambda ||
      !loss || !nnz || !npass)
    return fail(BSG_ERR_ARG, "null argument");
  const int n = op.n;
  std::vector<int> row0, col0;
  BSG_TRY(host_index(ind_row, nr, n, "", row0));
  BSG_TRY(host_index(ind_col, nc, op.m, "", col0));
  if (!finite_all(y, nr)) return fail(BSG_ERR_ARG, "'y.train' must be finite.");
  if (family == 1)
    for (int r = 0; r < nr; r++)
      if (!(y[r] == 0.0 || y[r] == 1.0)) return fail(BSG_ERR_ARG, "'y01.train' must be 0 or 1 (entry %d is not).", r + 1);
  if (Kc > 0 && !finite_all(covar, (int64_t)nr * Kc)) return fail(BSG_ERR_ARG, "'covar.train' must be finite.");
  if (base && !finite_all(base, nr)) return fail(BSG_ERR_ARG, "'base.train' must be finite.");
  for (int c = 0; c < nc; c++)
    if (pf_X && !(std::isfinite(pf_X[c]) && pf_X[c] >= 0)) return fail(BSG_ERR_ARG, "'pf.X' must be finite and >= 0.");
  for (int c = 0; c < Kc; c++)
    if (pf_covar && !(std::isfinite(pf_covar[c]) && pf_covar[c] >= 0))
      return fail(BSG_ERR_ARG, "'pf.covar' must be finite and >= 0.");
  // folds: position maps (training observations of fold k in order, then its own)
  std::vector<int> pos((size_t)K * nr), ntr(K, 0);
  for (int r = 0; r < nr; r++) {
    if (ind_sets[r] < 1 || ind_sets[r] > K) return fail(BSG_ERR_ARG, "'ind.sets' must take values in 1..K.");
  }
  for (int k = 0; k < K; k++) {
    int q = 0;
    for (int r = 0; r < nr; r++)
      if (ind_sets[r] != k + 1) pos[(size_t)k * nr + q++] = r;
    ntr[k] = q;
    for (int r = 0; r < nr; r++)
      if (ind_sets[r] == k + 1) pos[(size_t)k * nr + q++] = r;
    if (ntr[k] == nr || ntr[k] < 2) return fail(BSG_ERR_ARG, "Every fold of 'ind.sets' must hold at least one "
                                                               "observation and leave two for training.");
  }
  if ((int64_t)nr > NMAX)
    return fail(BSG_ERR_ARG, "big_spLinReg / big_spLogReg on the device take at most %lld observations (%d given).",
                (long long)NMAX, nr);
  const int F = nalpha * K, Jall = nc + Kc;
  const size_t need = (size_t)nr * (4 + 8 + 8 + 4 * K) + (size_t)Jall * (4 + 8 * 2 + 1) +
                      (size_t)F * ((size_t)nr * 8 * (family == 1 ? 3 : 1) + (size_t)Jall * (8 * 4 + (1 + 4) * CS) +
                                   (size_t)nlambda * 24 + 32) +
                      (path_beta ? (size_t)F * nlambda * Jall * 8 : 0) + op.stage_bytes(nr, nc) + (1 << 20);
  size_t fr = 0, tot = 0;
  BSG_CUDA(cudaMemGetInfo(&fr, &tot));
  if (need > fr)
    return fail(BSG_ERR_ALLOC, "big_spLinReg / big_spLogReg need %.0f bytes of device memory (%d fits, %d observations, "
                               "%d columns, %.0f bytes staged), %.0f are free.", (double)need, F, nr, Jall,
                (double)op.stage_bytes(nr, nc), (double)fr);
  cudaStream_t s = op.s;
  std::vector<double> zero(nr, 0.0);
  Bufs b;
  typename Op::Src cs{};
  const auto t0 = std::chrono::steady_clock::now();
  BSG_TRY(op.stage(row0, col0, nc, b, cs));
  g_stage_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
  double *d_cov = nullptr, *d_ctr, *d_sc;
  uint8_t *d_na;
  if (Kc > 0) b.up(&d_cov, covar, (size_t)nr * Kc, s);
  b.alloc(&d_ctr, (size_t)Jall);
  b.alloc(&d_sc, (size_t)Jall);
  b.alloc(&d_na, (size_t)Jall);
  BSG_TRY(b.status("big_spLinReg scratch"));
  cs.cov = d_cov, cs.nr = nr, cs.G = nc;
  CallTimer tm;
  BSG_CUDA(tm.start(s));
  if (Jall > 0) {
    k_sp_stats<<<(Jall + ST / 32 - 1) / (ST / 32), ST, 0, s>>>(cs, Jall, op.raw, n, op.lut, d_ctr, d_sc, d_na);
    count_launch();
    BSG_CUDA(cudaGetLastError());
  }
  std::vector<uint8_t> na(Jall);
  BSG_CUDA(cudaMemcpyAsync(center, d_ctr, (size_t)Jall * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(scale, d_sc, (size_t)Jall * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(na.data(), d_na, (size_t)Jall, cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  for (int c = 0; c < nc; c++)
    if (na[c]) return fail(BSG_ERR_ARG, op.bad_msg, ind_col ? ind_col[c] : c + 1);
  for (int c = 0; c < Kc; c++)
    if (!(scale[nc + c] > SD_MIN)) return fail(BSG_ERR_ARG, "Covariate %d is constant over 'ind.train'.", c + 1);
  // the fit's columns: kept columns by index in the matrix (genotype line or dense column; ties in ind_col order), so
  // that coordinate descent visits them in an order that does not depend on how ind_col is permuted, then the
  // covariates; results go back in ind_col order
  std::vector<int> lines, ord;
  std::vector<double> fc, fis, fpf;
  for (int c = 0; c < nc; c++) {
    kept[c] = scale[c] > SD_MIN;
    if (kept[c]) ord.push_back(c);
  }
  std::stable_sort(ord.begin(), ord.end(), [&](int u, int v) { return col0[u] < col0[v]; });
  for (int c : ord) {
    lines.push_back(op.line(c, col0));
    fc.push_back(center[c]);
    fis.push_back(1.0 / scale[c]);
    fpf.push_back(pf_X ? pf_X[c] : 1.0);
  }
  const int G = (int)lines.size(), J = G + Kc;
  for (int c = 0; c < Kc; c++) {
    fc.push_back(center[nc + c]);
    fis.push_back(1.0 / scale[nc + c]);
    fpf.push_back(pf_covar ? pf_covar[c] : 1.0);
  }
  if (J == 0) return fail(BSG_ERR_ARG, "No column varies over 'ind.train'.");
  FArgs<typename Op::Src> a;
  a.c = cs;
  a.c.G = G;
  a.J = J;
  a.K = K, a.family = family, a.nlambda = nlambda, a.nlam_min = nlam_min, a.n_abort = n_abort, a.dfmax = dfmax;
  a.max_iter = max_iter, a.eps = eps;
  a.step = nlambda > 1 ? std::pow(lambda_min_ratio, 1.0 / (nlambda - 1)) : 1.0;
  int *d_lines, *d_pos, *d_prow, *d_ntr;
  std::vector<int> prow(pos.size());
  for (size_t i = 0; i < pos.size(); i++) prow[i] = row0[pos[i]];
  double *d_fc, *d_fis, *d_fpf, *d_y, *d_base, *d_al;
  b.up(&d_lines, lines.data(), lines.size(), s);
  b.up(&d_fc, fc, s);
  b.up(&d_fis, fis, s);
  b.up(&d_fpf, fpf, s);
  b.up(&d_y, y, (size_t)nr, s);
  b.up(&d_base, base ? base : zero.data(), (size_t)nr, s);
  b.up(&d_al, alphas, (size_t)nalpha, s);
  b.up(&d_pos, pos, s);
  b.up(&d_prow, prow, s);
  b.up(&d_ntr, ntr, s);
  double *d_r, *d_w = nullptr, *d_s = nullptr, *d_beta, *d_z, *d_v, *d_bb, *d_b0, *d_lam, *d_loss, *d_pb = nullptr,
         *d_pb0 = nullptr;
  uint8_t *d_flag;
  int *d_wl, *d_best, *d_len, *d_msg, *d_nnz, *d_np;
  const size_t FJ = (size_t)F * J, FL = (size_t)F * nlambda;
  b.alloc(&d_r, (size_t)F * nr);
  if (family == 1) b.alloc(&d_w, (size_t)F * nr);
  if (family == 1) b.alloc(&d_s, (size_t)F * nr);
  b.alloc(&d_beta, FJ);
  b.alloc(&d_z, FJ);
  b.alloc(&d_v, FJ);
  b.alloc(&d_bb, FJ);
  b.alloc(&d_flag, FJ * CS);
  b.alloc(&d_wl, FJ * CS);
  b.alloc(&d_b0, (size_t)F);
  b.alloc(&d_best, (size_t)F);
  b.alloc(&d_len, (size_t)F);
  b.alloc(&d_msg, (size_t)F);
  b.alloc(&d_lam, FL);
  b.alloc(&d_loss, FL);
  b.alloc(&d_nnz, FL);
  b.alloc(&d_np, FL);
  if (path_beta) b.alloc(&d_pb, FL * J);
  if (path_b0) b.alloc(&d_pb0, FL);
  BSG_TRY(b.status("big_spLinReg scratch"));
  BSG_CUDA(cudaMemsetAsync(d_bb, 0, FJ * sizeof(double), s));
  BSG_CUDA(cudaMemsetAsync(d_b0, 0, (size_t)F * sizeof(double), s));
  BSG_CUDA(cudaMemsetAsync(d_lam, 0, FL * sizeof(double), s));
  BSG_CUDA(cudaMemsetAsync(d_loss, 0, FL * sizeof(double), s));
  BSG_CUDA(cudaMemsetAsync(d_nnz, 0, FL * sizeof(int), s));
  BSG_CUDA(cudaMemsetAsync(d_np, 0, FL * sizeof(int), s));
  if (d_pb) BSG_CUDA(cudaMemsetAsync(d_pb, 0, FL * J * sizeof(double), s));
  if (d_pb0) BSG_CUDA(cudaMemsetAsync(d_pb0, 0, FL * sizeof(double), s));
  a.c.lines = d_lines;
  if (Kc > 0) a.c.cov = d_cov;
  a.center = d_fc, a.iscale = d_fis, a.pf = d_fpf, a.y = d_y, a.base = d_base, a.pos = d_pos, a.prow = d_prow, a.ntr = d_ntr;
  a.alphas = d_al;
  a.r = d_r, a.w = d_w, a.s = d_s, a.beta = d_beta, a.z = d_z, a.v = d_v, a.flag = d_flag, a.wl = d_wl;
  a.bbest = d_bb, a.b0best = d_b0, a.best = d_best, a.len = d_len, a.msg = d_msg;
  a.lam = d_lam, a.loss = d_loss, a.nnz = d_nnz, a.npass = d_np, a.pbeta = d_pb, a.pb0 = d_pb0;
  BSG_CUDA(cudaFuncSetAttribute(k_splreg<typename Op::Src>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                (int)sizeof(Smem)));
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(F * CS);
  cfg.blockDim = dim3(ST);
  cfg.dynamicSmemBytes = sizeof(Smem);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CS, at[0].val.clusterDim.y = 1, at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  BSG_CUDA(cudaLaunchKernelEx(&cfg, k_splreg<typename Op::Src>, a));
  count_launch();
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(tm.stop(s));
  BSG_CUDA(cudaMemcpyAsync(beta, d_bb, FJ * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(intercept, d_b0, (size_t)F * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(best, d_best, (size_t)F * sizeof(int), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(length, d_len, (size_t)F * sizeof(int), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(message, d_msg, (size_t)F * sizeof(int), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(lambda, d_lam, FL * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(loss, d_loss, FL * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(nnz, d_nnz, FL * sizeof(int), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(npass, d_np, FL * sizeof(int), cudaMemcpyDeviceToHost, s));
  if (d_pb) BSG_CUDA(cudaMemcpyAsync(path_beta, d_pb, FL * J * sizeof(double), cudaMemcpyDeviceToHost, s));
  if (d_pb0) BSG_CUDA(cudaMemcpyAsync(path_b0, d_pb0, FL * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  // internal column i (line order) is output column rank[i] (kept columns in ind_col order)
  std::vector<int> slot(nc, 0), inv(G);
  for (int c = 0, i = 0; c < nc; c++) slot[c] = kept[c] ? i++ : -1;
  for (int i = 0; i < G; i++) inv[i] = slot[ord[i]];
  std::vector<double> tmp(J);
  auto unpermute = [&](double *v, size_t rows) {
    for (size_t r = 0; r < rows; r++) {
      double *x = v + r * J;
      for (int i = 0; i < G; i++) tmp[inv[i]] = x[i];
      std::copy(tmp.begin(), tmp.begin() + G, x);
    }
  };
  unpermute(beta, (size_t)F);
  if (path_beta) unpermute(path_beta, FL);
  g_last_ms = tm.ms();
  return BSG_OK;
}

}  // namespace splreg
}  // namespace bsg

using namespace bsg;

extern "C" {

int bsg_splreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, int family, const double *y,
               const double *covar, int Kc, const double *base, const double *pf_X, const double *pf_covar,
               const double *alphas, int nalpha, const int *ind_sets, int K, int nlambda, double lambda_min_ratio,
               int nlam_min, int n_abort, int dfmax, double eps, int max_iter, double power_scale, double power_adaptive,
               double *center, double *scale, uint8_t *kept, double *beta, double *intercept, int *best, int *length,
               int *message, double *lambda, double *loss, int *nnz, int *npass, double *path_beta, double *path_b0) {
  using namespace splreg;
  if (!h) return fail(BSG_ERR_ARG, "null handle");
  BSG_TRY(genotypes_check(h, "big_spLinReg / big_spLogReg on the device need"));
  BSG_TRY(bind_device(h));
  BedOp op{h, h->n, h->m, h->stream, h->raw};
  return splreg_drive(op, ind_row, nr, ind_col, nc, family, y, covar, Kc, base, pf_X, pf_covar, alphas, nalpha,
                      ind_sets, K, nlambda, lambda_min_ratio, nlam_min, n_abort, dfmax, eps, max_iter, power_scale,
                      power_adaptive, center, scale, kept, beta, intercept, best, length, message, lambda, loss, nnz,
                      npass, path_beta, path_b0);
}

int bsg_splreg_dense(const void *X, int dtype, int64_t ld, int nrow, int ncol, const int *ind_row, int nr,
                     const int *ind_col, int nc, int device, int family, const double *y, const double *covar, int Kc,
                     const double *base, const double *pf_X, const double *pf_covar, const double *alphas, int nalpha,
                     const int *ind_sets, int K, int nlambda, double lambda_min_ratio, int nlam_min, int n_abort,
                     int dfmax, double eps, int max_iter, double power_scale, double power_adaptive, double *center,
                     double *scale, uint8_t *kept, double *beta, double *intercept, int *best, int *length,
                     int *message, double *lambda, double *loss, int *nnz, int *npass, double *path_beta,
                     double *path_b0) {
  using namespace splreg;
  if (dtype != 0 && dtype != 1) return fail(BSG_ERR_TYPE, "dtype must be 0 (float) or 1 (double).");
  if (nrow < 0 || ncol < 0 || ld < std::max(nrow, 1) || (!X && (int64_t)nrow * ncol > 0))
    return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  if (cudaSetDevice(device) != cudaSuccess) {
    cudaGetLastError();
    return fail(BSG_ERR_CUDA, "CUDA device %d is not available (no CPU fallback).", device);
  }
  struct Stream {
    cudaStream_t s = nullptr;
    ~Stream() {
      if (s) cudaStreamSynchronize(s), cudaStreamDestroy(s);
    }
  } st;
  BSG_CUDA(cudaStreamCreateWithFlags(&st.s, cudaStreamNonBlocking));
#define BSG_SPLREG_TAIL                                                                                                  \
  ind_row, nr, ind_col, nc, family, y, covar, Kc, base, pf_X, pf_covar, alphas, nalpha, ind_sets, K, nlambda,           \
      lambda_min_ratio, nlam_min, n_abort, dfmax, eps, max_iter, power_scale, power_adaptive, center, scale, kept, beta, \
      intercept, best, length, message, lambda, loss, nnz, npass, path_beta, path_b0
  if (dtype == 0) {
    DenseOp<float> op{static_cast<const float *>(X), ld, nrow, ncol, st.s};
    return splreg_drive(op, BSG_SPLREG_TAIL);
  }
  DenseOp<double> op{static_cast<const double *>(X), ld, nrow, ncol, st.s};
  return splreg_drive(op, BSG_SPLREG_TAIL);
#undef BSG_SPLREG_TAIL
}

double bsg_splreg_last_ms(void) { return splreg::g_last_ms; }

double bsg_splreg_last_stage_ms(void) { return splreg::g_stage_ms; }

}  // extern "C"
