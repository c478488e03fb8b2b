// bsg_sparse.cu -- a sparse LD matrix resident on the device (bigsparser's SFBM, as bigsnpr reads it) and its two readers:
// ld_scores_sfbm (src/ld-scores-sfbm.cpp:9-69) and lassosum2 (src/lassosum2.cpp:20-70) over a whole (lambda, delta) grid.
//
// Storage (src/ld-scores-sfbm.cpp:14-66): p[ncol + 1] doubles; non-compact data interleaves (row, value) doubles, column j at
// data[2 p[j] .. 2 p[j + 1]); compact data holds values only, column j at data[p[j] .. p[j + 1]) for the rows first_i[j],
// first_i[j] + 1, ...  Both forms stay on the device as given: int32 rows (non-compact) or first_i (compact), fp64 values.
//
// lassosum2: one CTA per grid point runs every sweep of its coordinate descent in the kernel.  The state (dotprods over all
// ncol columns, curr_beta over the m coordinates) lives in global memory and changes only when a coordinate moves
// (shift != 0).  So warp 0 evaluates the next 32 coordinates from the current state, takes the first lane that moves
// (ballot), folds gap / df of the lanes before it and of itself, commits its beta, and the whole CTA applies
// dotprods[i] += x_ij * shift over column j2 before the warp resumes at the next coordinate.  Lanes that do not move leave
// the state as it was, so every coordinate sees exactly the state the sequential loop gives it.  The arithmetic is the
// reference's, uncontracted: u_j in its order, soft_thres with its IEEE division, the update as dadd(d, dmul(x, shift)),
// gap folded serially in coordinate order, df a count.  Hence bit-identical beta_est and num_iter.
//
// sp_solve_sym (bigsparser, called at R/LDpred2.R:38-39): Eigen's ConjugateGradient with the identity preconditioner and
// x0 = 0, over A + diag(d) with A the SFBM as stored.  Every sum is taken in one fixed order, independent of the launch:
//   - (A p + d o p)_j: a warp per column, lane l folding the entries q = lo + l, lo + l + 32, ... in ascending q, then the
//     xor-shuffle tree 16, 8, 4, 2, 1, then dadd(sum, dmul(d_j, p_j));
//   - a vector dot u.v: chunks of CG_CH = 1024 entries (entries past n are +0), each summed as a pairwise tree (level 1
//     pairs k and k + 512, then k and k + 256, ... down to k and k + 1), chunk sums folded serially from 0 in chunk order.
// No FMA contraction (__dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn).  One iteration is four launches (t = A p + d o p;
// chunk sums of p.t; alpha, x, r and chunk sums of r.r; the stopping test and p); a done flag in device memory turns the
// rest of a block of CG_BLOCK enqueued iterations into no-ops, and the host reads it once per block.
//
// LDpred2-auto (src/ldpred2-auto.cpp:56-202): one CTA per chain, lassosum2's scan over a seeded MRG32k3a stream per chain,
// the arithmetic in bsg_ldpred2_auto.cuh (DESIGN.md §4.15).
//
// LDpred2-grid (src/ldpred2.cpp:9-69, src/ldpred2-sampling.cpp:9-59): one CTA per grid point, the same scan, streams and
// header; a sparse point's coordinates with postp < p take no uniform (DESIGN.md §4.18).
#include <float.h>
#include <limits.h>
#include <math.h>
#include <string.h>

#include <cmath>
#include <vector>

#include "bsg_internal.cuh"
#include "bsg_ldpred2_auto.cuh"

struct bsg_sfbm {
  int device = 0;
  int nrow = 0, ncol = 0;
  int compact = 0;
  long long nnz = 0;
  long long *p = nullptr;  // ncol + 1 offsets
  int *rows = nullptr;     // nnz rows (non-compact)
  int *first_i = nullptr;  // ncol first rows (compact)
  double *x = nullptr;     // nnz values
  cudaStream_t stream = nullptr;
  double last_solve_ms = 0;  // ms, device time of the last bsg_sfbm_solve's iterations (CUDA events)
};

namespace bsg {
namespace sparse {

constexpr int LT = 256;  // threads of a lassosum2 CTA
// R's NA_real_: the NaN with payload 1954, what curr_beta.fill(NA_REAL) writes on divergence
__device__ __forceinline__ double na_real() { return __longlong_as_double(0x7FF00000000007A2LL); }

__device__ __forceinline__ unsigned long long globaltimer() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// src/lassosum2.cpp:8-16
__device__ __forceinline__ double soft_thres(double z, double l1, double one_plus_l2) {
  if (z > 0) {
    const double num = __dsub_rn(z, l1);
    return (num > 0) ? __ddiv_rn(num, one_plus_l2) : 0;
  } else {
    const double num = __dadd_rn(z, l1);
    return (num < 0) ? __ddiv_rn(num, one_plus_l2) : 0;
  }
}

// sfbm->incr_mult_col(j2, dotprods, shift) by the LT threads of a CTA, thread t from entry t: dp[i] += x_ij * shift over the
// stored entries of column j2.  Each row of a column is stored once, so the updates do not collide.  t keeps the type the
// kernel holds its thread index in (unsigned threadIdx.x or an int): ptxas allocates each kernel's registers as it did
// when the loop was written inline, without spills.
template <typename Tid>
__device__ __forceinline__ void incr_mult_col(const long long *__restrict__ p, const int *__restrict__ rows,
                                              const int *__restrict__ first_i, const double *__restrict__ x, int j2,
                                              double shift, double *dp, Tid t) {
  const long long lo = p[j2], up = p[j2 + 1];
  if (rows) {
    for (long long q = lo + t; q < up; q += LT) {
      const int i = rows[q];
      dp[i] = __dadd_rn(dp[i], __dmul_rn(x[q], shift));
    }
  } else {
    const int i0 = first_i[j2];
    for (long long q = lo + t; q < up; q += LT) {
      const int i = i0 + (int)(q - lo);
      dp[i] = __dadd_rn(dp[i], __dmul_rn(x[q], shift));
    }
  }
}

// Shared command of a lassosum2 CTA after each scan of warp 0: >= 0 the column j2 to apply shift to, else the end of a
// sweep and what follows it.
enum { CMD_NEXT_SWEEP = -1, CMD_DIVERGED = -2, CMD_STOP = -3 };

// Grid point g = blockIdx.x: lambda / dp1 / beta / dotprods are its columns (m, m, m, ncol doubles).
__global__ void __launch_bounds__(LT) k_lassosum2(const long long *__restrict__ p, const int *__restrict__ rows,
                                                  const int *__restrict__ first_i, const double *__restrict__ x, int ncol,
                                                  const double *__restrict__ beta_hat, int m, const int *__restrict__ ind_sub,
                                                  const double *__restrict__ lambda, const double *__restrict__ dp1,
                                                  double dfmax, int maxiter, double tol, double gap0, double *dotprods,
                                                  double *beta, int *num_iter, unsigned long long *ns) {
  __shared__ int s_cmd;
  __shared__ double s_shift;
  const int g = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const unsigned long long t0 = globaltimer();
  double *dp = dotprods + (size_t)g * ncol, *cb = beta + (size_t)g * m;
  const double *lam = lambda + (size_t)g * m, *del = dp1 + (size_t)g * m;
  for (int i = threadIdx.x; i < ncol; i += LT) dp[i] = 0;
  for (int i = threadIdx.x; i < m; i += LT) cb[i] = 0;
  __syncthreads();
  int k = 0;
  // warp 0's sweep state (every lane holds the same values)
  bool conv = true;
  long long df = 0;
  double gap = 0;
  int j = 0;
  for (; k < maxiter; k++) {
    if (warp == 0) {
      conv = true;
      df = 0;
      gap = 0;
      j = 0;
    }
    for (;;) {
      if (warp == 0) {
        int cmd = CMD_NEXT_SWEEP;
        double shift = 0;
        while (j < m) {
          const int jj = j + lane;
          const bool valid = jj < m;
          int j2 = 0;
          double nb = 0, sh = 0, cur = 0;
          if (valid) {
            j2 = ind_sub[jj];
            cur = cb[jj];
            const double u = __dsub_rn(beta_hat[jj], __dsub_rn(dp[j2], cur));
            nb = soft_thres(u, lam[jj], del[jj]);
            sh = __dsub_rn(nb, cur);
          }
          const unsigned mv = __ballot_sync(0xffffffffu, valid && sh != 0);
          const int last = mv ? __ffs(mv) - 1 : 31;  // lanes 0..last are consumed by this step
          const unsigned upto = last == 31 ? 0xffffffffu : (2u << last) - 1;
          unsigned nz = __ballot_sync(0xffffffffu, valid && nb != 0) & upto;
          df += __popc(nz);
          const double sq = __dmul_rn(nb, nb);
          while (nz) {  // gap += nb * nb in lane order
            const int l = __ffs(nz) - 1;
            gap = __dadd_rn(gap, __shfl_sync(0xffffffffu, sq, l));
            nz &= nz - 1;
          }
          if (mv) {
            shift = __shfl_sync(0xffffffffu, sh, last);
            cmd = __shfl_sync(0xffffffffu, j2, last);
            if (fabs(shift) > tol) conv = false;
            if (lane == last) cb[jj] = nb;
            j += last + 1;
            break;
          }
          j += 32;
        }
        if (cmd == CMD_NEXT_SWEEP) {  // src/lassosum2.cpp:62-63
          if (gap > gap0)
            cmd = CMD_DIVERGED;
          else if (conv || (double)df > dfmax)
            cmd = CMD_STOP;
        }
        if (lane == 0) {
          s_cmd = cmd;
          s_shift = shift;
        }
      }
      __syncthreads();
      const int cmd = s_cmd;
      if (cmd < 0) {
        if (cmd == CMD_NEXT_SWEEP) break;
        if (cmd == CMD_DIVERGED)
          for (int i = threadIdx.x; i < m; i += LT) cb[i] = na_real();
        goto done;
      }
      incr_mult_col(p, rows, first_i, x, cmd, s_shift, dp, threadIdx.x);
      __syncthreads();
    }
    __syncthreads();  // s_cmd is rewritten by the next sweep
  }
done:
  if (threadIdx.x == 0) {
    num_iter[g] = k + 1;
    if (ns) ns[g] = globaltimer() - t0;
  }
}

// ld_scores_sfbm: one warp per selected column, sum of x^2 over the stored rows flagged in use
__global__ void k_ld_scores_sfbm(const long long *__restrict__ p, const int *__restrict__ rows, const int *__restrict__ first_i,
                                 const double *__restrict__ x, const int *__restrict__ ind_sub, int m,
                                 const uint8_t *__restrict__ use, double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < m; j += nw) {
    const int j2 = ind_sub[j];
    const long long lo = p[j2], up = p[j2 + 1];
    double s = 0;
    for (long long q = lo + lane; q < up; q += 32) {
      const int i = rows ? rows[q] : first_i[j2] + (int)(q - lo);
      if (use[i]) s += x[q] * x[q];
    }
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[j] = s;
  }
}

// ---- sp_solve_sym: conjugate gradient ------------------------------------------------------------------------------------

constexpr int CG_CH = 1024;       // entries per chunk of a vector dot
constexpr int CG_DT = CG_CH / 2;  // threads of a chunk CTA: two entries each
constexpr int CG_MT = 256;        // threads of a matvec CTA (a warp per column)
constexpr int CG_BLOCK = 64;      // iterations enqueued between two reads of the done flag

struct CgState {
  double ab[2];   // absNew of iteration i in ab[i & 1] (read by every CTA of iteration i, written for i + 1)
  double rhs2;    // b.b
  double rn2;     // r.r of the last iteration run
  int done;       // r.r < threshold was reached
  int iters;      // the iteration that reached it (Eigen does not count it)
};

// Sum of the chunk's 1024 values in the fixed pairwise tree; a and b are entries k and k + 512 of thread k.  Valid in
// thread 0.
__device__ __forceinline__ double cg_chunk_tree(double a, double b, double *sh) {
  const int k = threadIdx.x;
  double s = __dadd_rn(a, b);
  sh[k] = s;
  __syncthreads();
  for (int w = CG_DT / 2; w >= 32; w >>= 1) {
    if (k < w) sh[k] = s = __dadd_rn(s, sh[k + w]);
    __syncthreads();
  }
  if (k < 32)
    for (int w = 16; w; w >>= 1) s = __dadd_rn(s, __shfl_down_sync(0xffffffffu, s, w));
  return s;
}

// The chunk sums folded serially from 0 in chunk order, by warp 0 (every lane holds the result); broadcast through sh.
__device__ __forceinline__ double cg_fold(const double *__restrict__ part, int nch, double *sh) {
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    double s = 0;
    for (int base = 0; base < nch; base += 32) {
      const double v = base + lane < nch ? part[base + lane] : 0;
      const int cnt = min(32, nch - base);
      for (int l = 0; l < cnt; l++) s = __dadd_rn(s, __shfl_sync(0xffffffffu, v, l));
    }
    if (lane == 0) sh[0] = s;
  }
  __syncthreads();
  const double s = sh[0];
  __syncthreads();  // sh is reused by the chunk tree
  return s;
}

// x = 0, r = p = b, chunk sums of b.b
__global__ void __launch_bounds__(CG_DT) k_cg_init(const double *__restrict__ b, int n, double *x, double *r, double *p,
                                                   double *part) {
  __shared__ double sh[CG_DT];
  const int i0 = blockIdx.x * CG_CH + threadIdx.x, i1 = i0 + CG_DT;
  double a = 0, c = 0;
  if (i0 < n) {
    const double v = b[i0];
    x[i0] = 0, r[i0] = v, p[i0] = v;
    a = __dmul_rn(v, v);
  }
  if (i1 < n) {
    const double v = b[i1];
    x[i1] = 0, r[i1] = v, p[i1] = v;
    c = __dmul_rn(v, v);
  }
  const double s = cg_chunk_tree(a, c, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

__global__ void k_cg_init_fold(const double *__restrict__ part, int nch, CgState *st) {
  __shared__ double sh[1];
  const double s = cg_fold(part, nch, sh);
  if (threadIdx.x == 0) {
    st->rhs2 = s, st->rn2 = s, st->ab[0] = s, st->ab[1] = 0;
    st->done = 0, st->iters = 0;
  }
}

// t_j = dadd(sum_q x_q p[row_q], dmul(d_j, p_j)); d has length 1 (dlen == 1) or n
__global__ void __launch_bounds__(CG_MT) k_cg_matvec(const long long *__restrict__ cp, const int *__restrict__ rows,
                                                     const int *__restrict__ first_i, const double *__restrict__ x, int n,
                                                     const double *__restrict__ d, int dlen, const double *__restrict__ p,
                                                     double *__restrict__ t, const CgState *st) {
  if (st->done) return;
  const int lane = threadIdx.x & 31;
  const int nw = (gridDim.x * blockDim.x) >> 5;
  for (int j = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; j < n; j += nw) {
    const long long lo = cp[j], up = cp[j + 1];
    double s = 0;
    if (rows) {
#pragma unroll 4
      for (long long q = lo + lane; q < up; q += 32) s = __dadd_rn(s, __dmul_rn(x[q], p[rows[q]]));
    } else {  // compact: entry lo + k is row first_i[j] + k
      const double *xc = x + lo, *pc = p + first_i[j];
      const int len = (int)(up - lo);
#pragma unroll 4
      for (int k = lane; k < len; k += 32) s = __dadd_rn(s, __dmul_rn(xc[k], pc[k]));
    }
    for (int o = 16; o; o >>= 1) s = __dadd_rn(s, __shfl_xor_sync(0xffffffffu, s, o));
    if (lane == 0) t[j] = __dadd_rn(s, __dmul_rn(d[dlen == 1 ? 0 : j], p[j]));
  }
}

// chunk sums of p.t
__global__ void __launch_bounds__(CG_DT) k_cg_pt(const double *__restrict__ p, const double *__restrict__ t, int n,
                                                 double *part, const CgState *st) {
  __shared__ double sh[CG_DT];
  if (st->done) return;
  const int i0 = blockIdx.x * CG_CH + threadIdx.x, i1 = i0 + CG_DT;
  const double a = i0 < n ? __dmul_rn(p[i0], t[i0]) : 0, c = i1 < n ? __dmul_rn(p[i1], t[i1]) : 0;
  const double s = cg_chunk_tree(a, c, sh);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}

// alpha = absNew / p.t (every CTA folds the same chunk sums); x += alpha p; r -= alpha t; chunk sums of r.r
__global__ void __launch_bounds__(CG_DT) k_cg_update(const double *__restrict__ p, const double *__restrict__ t, int n,
                                                     double *x, double *r, const double *__restrict__ part_pt, int nch,
                                                     double *part_rr, const CgState *st, int it) {
  __shared__ double sh[CG_DT];
  if (st->done) return;
  const double alpha = __ddiv_rn(st->ab[it & 1], cg_fold(part_pt, nch, sh));
  double v[2] = {0, 0};
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int i = blockIdx.x * CG_CH + threadIdx.x + h * CG_DT;
    if (i < n) {
      x[i] = __dadd_rn(x[i], __dmul_rn(alpha, p[i]));
      const double ri = __dsub_rn(r[i], __dmul_rn(alpha, t[i]));
      r[i] = ri;
      v[h] = __dmul_rn(ri, ri);
    }
  }
  const double s = cg_chunk_tree(v[0], v[1], sh);
  if (threadIdx.x == 0) part_rr[blockIdx.x] = s;
}

// rn2 = r.r; stop when rn2 < threshold; else beta = rn2 / absOld, p = r + beta p
__global__ void __launch_bounds__(CG_DT) k_cg_direction(const double *__restrict__ r, int n, double *p,
                                                        const double *__restrict__ part_rr, int nch, double threshold,
                                                        CgState *st, int it) {
  __shared__ double sh[1];
  if (st->done) return;  // set only by CTA 0 of this launch on convergence, when every CTA returns below anyway
  const double rn2 = cg_fold(part_rr, nch, sh);
  const bool lead = blockIdx.x == 0 && threadIdx.x == 0;
  if (rn2 < threshold) {
    if (lead) st->rn2 = rn2, st->iters = it, st->done = 1;
    return;
  }
  const double beta = __ddiv_rn(rn2, st->ab[it & 1]);
#pragma unroll
  for (int h = 0; h < 2; h++) {
    const int i = blockIdx.x * CG_CH + threadIdx.x + h * CG_DT;
    if (i < n) p[i] = __dadd_rn(r[i], __dmul_rn(beta, p[i]));
  }
  if (lead) st->rn2 = rn2, st->ab[(it + 1) & 1] = rn2;
}

// ---- LDpred2-auto: one CTA per chain -------------------------------------------------------------------------------------

struct LdaArgs {
  const double *beta_hat, *n_vec, *log_var, *p_init;
  const int *ind_sub;
  const uint32_t *rng;  // 6 words per chain
  uint32_t *rng_out;    // 6 words per chain, the state after the last sweep (may be null)
  int m, burn_in, num_iter, report_step, nrep, no_jump_sign, use_mle;
  double h2_init, shrink, p_lo, p_hi, t_lo, t_hi, mean_ld, gap0;
  // outputs, per chain: m (estimates), T = burn_in + num_iter (paths), m x nrep (sample, may be null)
  double *beta_est, *postp_est, *corr_est, *path_p, *path_h2, *path_alpha, *sample;
  // scratch, per chain: ncol (dot), m (the others)
  double *dot, *cb, *avg_b, *avg_p, *avg_bh, *abuf, *bbuf;
  int *causal;
  unsigned long long *ns;
};

// Sum over k < nb of b_k exp(-t a_k) (b non-null) or of a_k, in one fixed order: thread i folds k = i, i + LT, ... from
// 0, then the pairwise tree v[i] += v[i + w], w = LT / 2 .. 1.  Every thread returns the sum.
__device__ double lda_red(const double *__restrict__ a, const double *__restrict__ b, double t, int nb, double *sh) {
  const int tid = threadIdx.x;
  double s = 0;
  for (int k = tid; k < nb; k += LT) s = __dadd_rn(s, b ? __dmul_rn(b[k], lda_exp(__dmul_rn(-t, a[k]))) : a[k]);
  sh[tid] = s;
  __syncthreads();
  for (int w = LT / 2; w >= 32; w >>= 1) {
    if (tid < w) sh[tid] = s = __dadd_rn(s, sh[tid + w]);
    __syncthreads();
  }
  if (tid < 32) {
    for (int w = 16; w; w >>= 1) s = __dadd_rn(s, __shfl_down_sync(0xffffffffu, s, w));
    if (tid == 0) sh[0] = s;
  }
  __syncthreads();
  s = sh[0];
  __syncthreads();
  return s;
}

__global__ void __launch_bounds__(LT) k_ldpred2_auto(const long long *__restrict__ p, const int *__restrict__ rows,
                                                     const int *__restrict__ first_i, const double *__restrict__ x, int ncol,
                                                     const LdaArgs A) {
  __shared__ lda_mat s_pw[32];  // A^(2^i)
  __shared__ lda_mat s_ln[32];  // A^(l + 1): lane l's draw is row 2 of it applied to the state
  __shared__ lda_mat s_adv;     // A^(LT - 1): a bootstrap thread's stride
  __shared__ double s_red[LT];
  __shared__ uint32_t s_rng[6];
  __shared__ int s_cmd, s_nb;
  __shared__ double s_shift, s_p, s_h2, s_par[2], s_cur_h2;
  const int c = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned long long t0 = globaltimer();
  const int m = A.m, T = A.burn_in + A.num_iter;
  double *dp = A.dot + (size_t)c * ncol, *cb = A.cb + (size_t)c * m;
  double *avg_b = A.avg_b + (size_t)c * m, *avg_p = A.avg_p + (size_t)c * m, *avg_bh = A.avg_bh + (size_t)c * m;
  double *abuf = A.abuf + (size_t)c * m, *bbuf = A.bbuf + (size_t)c * m;
  int *causal = A.causal + (size_t)c * m;
  double *path_p = A.path_p + (size_t)c * T, *path_h2 = A.path_h2 + (size_t)c * T, *path_alpha = A.path_alpha + (size_t)c * T;
  double *sample = A.sample ? A.sample + (size_t)c * m * A.nrep : nullptr;
  if (tid == 0) lda_pow2_table(s_pw, 32);
  for (int i = tid; i < ncol; i += LT) dp[i] = 0;
  for (int i = tid; i < m; i += LT) cb[i] = 0, avg_b[i] = 0, avg_p[i] = 0, avg_bh[i] = 0;
  for (int i = tid; i < T; i += LT) path_p[i] = na_real(), path_h2[i] = na_real(), path_alpha[i] = na_real();
  if (sample)
    for (size_t i = tid; i < (size_t)m * A.nrep; i += LT) sample[i] = 0;
  __syncthreads();
  if (tid < 32) s_ln[tid] = lda_mat_pow(s_pw, tid + 1);
  if (tid == 32) s_adv = lda_mat_pow(s_pw, LT - 1);
  if (tid == 0) {  // src/ldpred2-auto.cpp:91-94
    for (int i = 0; i < 6; i++) s_rng[i] = A.rng[6 * c + i];
    const double h2 = A.h2_init < 1e-3 ? 1e-3 : A.h2_init;
    double pp = A.p_lo < A.p_init[c] ? A.p_init[c] : A.p_lo;
    pp = A.p_hi < pp ? A.p_hi : pp;
    s_p = pp, s_h2 = h2, s_cur_h2 = 0;
    s_par[0] = 0, s_par[1] = __ddiv_rn(h2, __dmul_rn((double)m, pp));
  }
  __syncthreads();
  int next_k = A.burn_in + A.report_step - 1, irep = 0;
  // warp 0's sweep state (every lane holds the same values)
  uint32_t st[6];
  double gap = 0, cur_h2 = 0;
  int nb = 0;
  for (int k = 0; k < T; k++) {
    if (warp == 0) {
      for (int i = 0; i < 6; i++) st[i] = s_rng[i];
      cur_h2 = s_cur_h2, gap = 0, nb = 0;
    }
    const double inv_odd_p = __ddiv_rn(__dsub_rn(1.0, s_p), s_p), apo = s_par[0], sigma2 = s_par[1];
    int j = 0;
    for (;;) {
      if (warp == 0) {
        int cmd = CMD_NEXT_SWEEP;
        double shift = 0;
        while (j < m) {
          const int jj = j + lane, nv = min(32, m - j);
          const bool valid = jj < m;
          lda_coord_t co = {0, 0, 0, 0};
          double cur = 0;
          int j2 = 0;
          bool sel = false;
          if (valid) {
            j2 = A.ind_sub[jj];
            cur = cb[jj];
            co = lda_coord(A.beta_hat[jj], dp[j2], cur, A.n_vec[jj], A.log_var[jj], A.shrink, A.use_mle, apo, sigma2,
                           inv_odd_p);
            // the draw lane positions after the state: row 2 of A^(lane + 1) in each component
            const uint32_t p1 = lda_mulmod3(s_ln[lane].a + 6, st, LDA_M1), p2 = lda_mulmod3(s_ln[lane].a + 15, st + 3, LDA_M2);
            sel = co.postp > lda_u01(p1, p2);
          }
          // the first lane that draws a normal or changes beta; the lanes before it consume one uniform each
          const unsigned stop = __ballot_sync(0xffffffffu, valid && (sel || cur != 0));
          const int last = stop ? __ffs(stop) - 1 : nv - 1;
          if (valid && lane <= last && k >= A.burn_in) {
            avg_p[jj] = __dadd_rn(avg_p[jj], co.postp);
            avg_b[jj] = __dadd_rn(avg_b[jj], __dmul_rn(co.C3, co.postp));
            avg_bh[jj] = __dadd_rn(avg_bh[jj], co.dps);
          }
          lda_mat_apply(&s_ln[last], st);
          if (!stop) {
            j += nv;
            continue;
          }
          const bool lsel = __shfl_sync(0xffffffffu, sel, last);
          const double lcur = __shfl_sync(0xffffffffu, cur, last), C3 = __shfl_sync(0xffffffffu, co.C3, last);
          const double C4 = __shfl_sync(0xffffffffu, co.C4, last), dps = __shfl_sync(0xffffffffu, co.dps, last);
          const int lj2 = __shfl_sync(0xffffffffu, j2, last);
          double diff = -lcur, nbeta = 0;
          if (lsel) {  // src/ldpred2-auto.cpp:134-150
            const double samp = lda_rnorm(C3, __dsqrt_rn(C4), st);
            if (!(A.no_jump_sign && __dmul_rn(samp, lcur) < 0)) {
              nbeta = samp;
              diff = __dadd_rn(diff, samp);
              if (lane == 0) causal[nb] = j + last;
              nb++;
              gap = __dadd_rn(gap, __dmul_rn(samp, samp));
            }
          }
          if (lane == 0) cb[j + last] = nbeta;
          j += last + 1;
          if (diff != 0) {
            cur_h2 = __dadd_rn(cur_h2, __dmul_rn(diff, __dadd_rn(__dmul_rn(2.0, dps), diff)));
            cmd = lj2;
            shift = diff;
            break;
          }
        }
        if (lane == 0) {
          s_cmd = cmd;
          s_shift = shift;
        }
      }
      __syncthreads();
      const int cmd = s_cmd;
      if (cmd < 0) break;
      incr_mult_col(p, rows, first_i, x, cmd, s_shift, dp, tid);
      __syncthreads();
    }
    if (tid == 0) {  // src/ldpred2-auto.cpp:161-168
      s_cur_h2 = cur_h2, s_nb = nb;
      if (gap > A.gap0) {
        s_cmd = CMD_DIVERGED;
      } else {
        s_p = lda_draw_p(nb, m, A.mean_ld, A.p_lo, A.p_hi, st);
        s_h2 = cur_h2 < 1e-3 ? 1e-3 : cur_h2;
      }
      for (int i = 0; i < 6; i++) s_rng[i] = st[i];
    }
    __syncthreads();
    if (s_cmd == CMD_DIVERGED) {
      for (int i = tid; i < m; i += LT) avg_b[i] = na_real(), avg_p[i] = na_real(), avg_bh[i] = na_real();
      break;
    }
    const int nbc = s_nb;
    if (A.use_mle) {
      if (nbc > 0) {  // MLE_alpha(par_mle, ind_causal, log_var, curr_beta, alpha_bounds, boot = true)
        uint32_t bs[6];
        for (int i = 0; i < 6; i++) bs[i] = s_rng[i];
        lda_skip(bs, tid, s_pw);
        for (int kk = tid; kk < nbc; kk += LT) {  // draw kk of the bootstrap, by skip-ahead
          const int jc = causal[(int)__dmul_rn((double)nbc, lda_unif(bs))];
          abuf[kk] = A.log_var[jc];
          bbuf[kk] = __dmul_rn(cb[jc], cb[jc]);
          lda_mat_apply(&s_adv, bs);
        }
        __syncthreads();
        if (tid == 0) lda_skip(s_rng, nbc, s_pw);
        const double sum_a = lda_red(abuf, nullptr, 0, nbc, s_red);
        const double s2_lo = __ddiv_rn(s_par[1], 2.0), s2_hi = __dmul_rn(s_par[1], 2.0);
        lda_golden g;
        double t = lda_golden_start(&g, A.t_lo, A.t_hi), s2;
        for (;;) {
          const double C = lda_red(abuf, bbuf, t, nbc, s_red);
          if (!lda_golden_next(&g, lda_mle_profile(t, sum_a, C, nbc, s2_lo, s2_hi, &s2), &t)) break;
        }
        const double C = lda_red(abuf, bbuf, g.best_t, nbc, s_red);
        lda_mle_profile(g.best_t, sum_a, C, nbc, s2_lo, s2_hi, &s2);
        if (tid == 0) s_par[0] = g.best_t, s_par[1] = s2;
      }
    } else if (tid == 0) {
      s_par[1] = __ddiv_rn(s_h2, __dmul_rn((double)m, s_p));
    }
    __syncthreads();
    if (tid == 0) {
      path_p[k] = s_p, path_h2[k] = s_h2;
      if (A.use_mle) path_alpha[k] = __dsub_rn(s_par[0], 1.0);
    }
    if (k == next_k) {  // src/ldpred2-auto.cpp:185-191
      if (sample)
        for (int i = tid; i < nbc; i += LT) sample[causal[i] + (size_t)irep * m] = cb[causal[i]];
      irep++;
      next_k += A.report_step;
    }
    __syncthreads();
  }
  const double inv = (double)A.num_iter;
  for (int i = tid; i < m; i += LT) {  // avg / num_iter, NA_real kept as it is
    const double b = avg_b[i], q = avg_p[i], h = avg_bh[i];
    A.beta_est[(size_t)c * m + i] = b != b ? b : __ddiv_rn(b, inv);
    A.postp_est[(size_t)c * m + i] = q != q ? q : __ddiv_rn(q, inv);
    A.corr_est[(size_t)c * m + i] = h != h ? h : __ddiv_rn(h, inv);
  }
  if (tid == 0 && A.rng_out)
    for (int i = 0; i < 6; i++) A.rng_out[6 * c + i] = s_rng[i];
  if (tid == 0 && A.ns) A.ns[c] = globaltimer() - t0;
}

// ---- LDpred2-grid: one CTA per grid point --------------------------------------------------------------------------------

struct LdgArgs {
  const double *beta_hat, *n_vec, *p, *h2;
  const int *sparse, *ind_sub;
  const uint32_t *rng;  // 6 words per point
  int m, burn_in, num_iter;
  double gap0;
  double *beta_est, *sample;  // m per point; m x num_iter (SAMPLING, one point)
  double *dot, *cb, *avg;     // scratch per point: ncol, m, m
  unsigned long long *ns;
};

// src/ldpred2.cpp:9-69 (SAMPLING false) and src/ldpred2-sampling.cpp:9-59 (SAMPLING true) for point g = blockIdx.x, with
// auto's warp-0 scan: lane l draws the uniform popc(lanes below l that draw) ahead of the state, a sparse point's lanes
// with postp < p draw none, and the scan stops at the first lane that draws a normal or changes beta.
template <bool SAMPLING>
__global__ void __launch_bounds__(LT) k_ldpred2_grid(const long long *__restrict__ p, const int *__restrict__ rows,
                                                     const int *__restrict__ first_i, const double *__restrict__ x, int ncol,
                                                     const LdgArgs A) {
  __shared__ lda_mat s_pw[32];  // A^(2^i)
  __shared__ lda_mat s_ln[32];  // A^(o + 1): the draw o uniforms ahead is row 2 of it applied to the state
  __shared__ int s_cmd;
  __shared__ double s_shift;
  const int g = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const unsigned long long t0 = globaltimer();
  const int m = A.m, T = A.burn_in + A.num_iter;
  double *dp = A.dot + (size_t)g * ncol, *cb = A.cb + (size_t)g * m, *avg = A.avg + (size_t)g * m;
  if (tid == 0) lda_pow2_table(s_pw, 32);
  for (int i = tid; i < ncol; i += LT) dp[i] = 0;
  for (int i = tid; i < m; i += LT) cb[i] = 0, avg[i] = 0;
  if (SAMPLING)
    for (size_t i = tid; i < (size_t)m * A.num_iter; i += LT) A.sample[i] = 0;
  __syncthreads();
  if (tid < 32) s_ln[tid] = lda_mat_pow(s_pw, tid + 1);
  __syncthreads();
  // src/ldpred2.cpp:27-28
  const double pp = A.p[g], h2_per_var = __ddiv_rn(A.h2[g], __dmul_rn((double)m, pp));
  const double inv_odd_p = __ddiv_rn(__dsub_rn(1.0, pp), pp);
  const int sparse = A.sparse[g] != 0;
  // warp 0's chain state (every lane holds the same values)
  uint32_t st[6];
  for (int i = 0; i < 6; i++) st[i] = A.rng[6 * g + i];
  double gap = 0;
  bool diverged = false;
  for (int k = 0; k < T; k++) {
    gap = 0;
    int j = 0;
    for (;;) {
      if (warp == 0) {
        int cmd = CMD_NEXT_SWEEP;
        double shift = 0;
        while (j < m) {
          const int jj = j + lane, nv = min(32, m - j);
          const bool valid = jj < m;
          lda_gcoord_t co = {0, 0, 0};
          double cur = 0;
          int j2 = 0;
          if (valid) {
            j2 = A.ind_sub[jj];
            cur = cb[jj];
            co = lda_grid_coord(lda_grid_res(A.beta_hat[jj], dp[j2], cur, SAMPLING), h2_per_var, A.n_vec[jj], inv_odd_p);
          }
          const bool draws = valid && lda_grid_draws(sparse, co.postp, pp);
          const unsigned dmask = __ballot_sync(0xffffffffu, draws);
          bool sel = false;
          if (draws) {
            const lda_mat *M = &s_ln[lda_grid_offset(dmask, lane)];
            sel = co.postp > lda_u01(lda_mulmod3(M->a + 6, st, LDA_M1), lda_mulmod3(M->a + 15, st + 3, LDA_M2));
          }
          // the first lane that draws a normal or changes beta; the lanes before it only consume their uniforms
          const unsigned stop = __ballot_sync(0xffffffffu, valid && (sel || cur != 0));
          const int last = stop ? __ffs(stop) - 1 : nv - 1;
          if (!SAMPLING && draws && lane <= last && k >= A.burn_in) avg[jj] = __dadd_rn(avg[jj], __dmul_rn(co.C3, co.postp));
          const int used = __popc(dmask & (last == 31 ? 0xffffffffu : (2u << last) - 1));
          if (used) lda_mat_apply(&s_ln[used - 1], st);
          if (!stop) {
            j += nv;
            continue;
          }
          const bool lsel = __shfl_sync(0xffffffffu, sel, last);
          const double lcur = __shfl_sync(0xffffffffu, cur, last), C3 = __shfl_sync(0xffffffffu, co.C3, last);
          const double C4 = __shfl_sync(0xffffffffu, co.C4, last);
          const int lj2 = __shfl_sync(0xffffffffu, j2, last);
          double diff = -lcur, nbeta = 0;
          if (lsel) {  // src/ldpred2.cpp:53-57, src/ldpred2-sampling.cpp:50-52
            nbeta = lda_rnorm(C3, __dsqrt_rn(C4), st);
            diff = __dadd_rn(diff, nbeta);
            if (!SAMPLING) gap = __dadd_rn(gap, __dmul_rn(nbeta, nbeta));
            if (SAMPLING && k >= A.burn_in && lane == 0) A.sample[(size_t)(k - A.burn_in) * m + j + last] = nbeta;
          }
          if (lane == 0) cb[j + last] = nbeta;
          j += last + 1;
          if (diff != 0) {
            cmd = lj2;
            shift = diff;
            break;
          }
        }
        if (!SAMPLING && cmd == CMD_NEXT_SWEEP && gap > A.gap0) cmd = CMD_DIVERGED;  // src/ldpred2.cpp:65
        if (lane == 0) {
          s_cmd = cmd;
          s_shift = shift;
        }
      }
      __syncthreads();
      const int cmd = s_cmd;
      if (cmd < 0) {
        diverged = cmd == CMD_DIVERGED;
        break;
      }
      incr_mult_col(p, rows, first_i, x, cmd, s_shift, dp, tid);
      __syncthreads();
    }
    __syncthreads();  // s_cmd is rewritten by the next sweep
    if (diverged) break;
  }
  if (!SAMPLING) {
    const double inv = (double)A.num_iter;
    for (int i = tid; i < m; i += LT) A.beta_est[(size_t)g * m + i] = diverged ? na_real() : __ddiv_rn(avg[i], inv);
  }
  if (tid == 0 && A.ns) A.ns[g] = globaltimer() - t0;
}

static int bind(const bsg_sfbm *s) {
  BSG_CUDA(cudaSetDevice(s->device));
  return BSG_OK;
}

// MRG32k3a: each component below its modulus and not all zero
static int check_rng(const unsigned *rng_state, int n, const char *what) {
  for (int c = 0; c < n; c++) {
    const unsigned *s = rng_state + 6 * c;
    if (s[0] >= LDA_M1 || s[1] >= LDA_M1 || s[2] >= LDA_M1 || s[3] >= LDA_M2 || s[4] >= LDA_M2 || s[5] >= LDA_M2 ||
        (s[0] | s[1] | s[2]) == 0 || (s[3] | s[4] | s[5]) == 0)
      return fail(BSG_ERR_ARG, "rng_state of %s %d is not a valid MRG32k3a state.", what, c);
  }
  return BSG_OK;
}

static int check_sub(const bsg_sfbm *s, const int *ind_sub, int m) {
  for (int j = 0; j < m; j++)
    if (ind_sub[j] < 0 || ind_sub[j] >= s->ncol) return fail(BSG_ERR_BOUNDS, "Tested subscript out of bounds (ind_sub).");
  return BSG_OK;
}

}  // namespace sparse
}  // namespace bsg

using namespace bsg;
using namespace bsg::sparse;

extern "C" {

int bsg_sfbm_open(int nrow, int ncol, const double *p, const double *data, const int *first_i, int device,
                  bsg_sfbm **out) {
  if (!out) return fail(BSG_ERR_ARG, "null argument");
  *out = nullptr;
  if (nrow < 0 || ncol < 0 || !p) return fail(BSG_ERR_ARG, "bad dimensions or null p");
  // p: non-decreasing integers starting at 0
  if (p[0] != 0) return fail(BSG_ERR_ARG, "p[0] must be 0.");
  std::vector<long long> hp(ncol + 1);
  for (int j = 0; j <= ncol; j++) {
    const double v = p[j];
    if (!(v >= 0) || v != floor(v) || v > 9.0e15 || (j > 0 && v < p[j - 1]))
      return fail(BSG_ERR_ARG, "p must be non-decreasing integers starting at 0 (column %d).", j);
    hp[j] = (long long)v;
  }
  const long long nnz = hp[ncol];
  if (nnz > 0 && !data) return fail(BSG_ERR_ARG, "null data");
  const bool compact = first_i != nullptr;
  std::vector<int> rows;
  std::vector<double> vals((size_t)nnz);
  if (compact) {
    for (int j = 0; j < ncol; j++)
      if (first_i[j] < 0 || (long long)first_i[j] + (hp[j + 1] - hp[j]) > nrow)
        return fail(BSG_ERR_ARG, "compact column %d: rows first_i[j] .. first_i[j] + len - 1 must lie in [0, nrow).", j);
    memcpy(vals.data(), data, (size_t)nnz * sizeof(double));
  } else {
    // rows: integers in [0, nrow), each at most once per column (the device applies a column's updates in parallel)
    rows.resize((size_t)nnz);
    std::vector<int> seen(nrow, -1);
    for (int j = 0; j < ncol; j++)
      for (long long q = hp[j]; q < hp[j + 1]; q++) {
        const double r = data[2 * q];
        if (!(r >= 0 && r < nrow) || r != floor(r))
          return fail(BSG_ERR_ARG, "column %d: row indices must be integers in [0, nrow).", j);
        const int i = (int)r;
        if (seen[i] == j) return fail(BSG_ERR_ARG, "column %d: row %d is stored twice.", j, i);
        seen[i] = j;
        rows[q] = i;
        vals[q] = data[2 * q + 1];
      }
  }
  if (cudaSetDevice(device) != cudaSuccess) {
    cudaGetLastError();
    return fail(BSG_ERR_CUDA, "CUDA device %d is not available (no CPU fallback).", device);
  }
  bsg_sfbm *s = new bsg_sfbm();
  s->device = device;
  s->nrow = nrow;
  s->ncol = ncol;
  s->compact = compact;
  s->nnz = nnz;
  cudaError_t e = cudaStreamCreateWithFlags(&s->stream, cudaStreamNonBlocking);
  const size_t nv = nnz ? (size_t)nnz : 1;
  if (e == cudaSuccess) e = cudaMalloc(&s->p, (ncol + 1) * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&s->x, nv * sizeof(double));
  if (e == cudaSuccess) e = compact ? cudaMalloc(&s->first_i, (ncol ? ncol : 1) * sizeof(int)) : cudaMalloc(&s->rows, nv * sizeof(int));
  if (e != cudaSuccess) {
    bsg_sfbm_close(s);
    return alloc_fail(e, "SFBM does not fit in device memory");
  }
  e = cudaMemcpy(s->p, hp.data(), (ncol + 1) * sizeof(long long), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && nnz) e = cudaMemcpy(s->x, vals.data(), (size_t)nnz * sizeof(double), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && compact && ncol) e = cudaMemcpy(s->first_i, first_i, ncol * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess && !compact && nnz) e = cudaMemcpy(s->rows, rows.data(), (size_t)nnz * sizeof(int), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    bsg_sfbm_close(s);
    return cuda_fail(e, "SFBM upload");
  }
  *out = s;
  return BSG_OK;
}

void bsg_sfbm_close(bsg_sfbm *s) {
  if (!s) return;
  cudaSetDevice(s->device);
  if (s->stream) cudaStreamSynchronize(s->stream);
  void *ptrs[] = {s->p, s->rows, s->first_i, s->x};
  for (void *q : ptrs)
    if (q) cudaFree(q);
  if (s->stream) cudaStreamDestroy(s->stream);
  delete s;
}

int bsg_sfbm_nrow(const bsg_sfbm *s) { return s ? s->nrow : -1; }
int bsg_sfbm_ncol(const bsg_sfbm *s) { return s ? s->ncol : -1; }

int bsg_sfbm_ld_scores(bsg_sfbm *s, const int *ind_sub, int m, double *out) {
  if (!s || m < 0 || (m > 0 && (!ind_sub || !out))) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(check_sub(s, ind_sub, m));
  if (m == 0) return BSG_OK;
  BSG_TRY(bind(s));
  std::vector<uint8_t> use(s->ncol, 0);
  for (int j = 0; j < m; j++) use[ind_sub[j]] = 1;
  if (s->nrow > s->ncol) use.resize(s->nrow, 0);  // rows past the last column are never in ind_sub
  cudaStream_t st = s->stream;
  Bufs b;
  int *d_sub = nullptr;
  uint8_t *d_use = nullptr;
  double *d_out = nullptr;
  BSG_CUDA(b.up(&d_sub, ind_sub, (size_t)m, st));
  BSG_CUDA(b.up(&d_use, use, st));
  BSG_CUDA(b.alloc(&d_out, (size_t)m));
  const int grid = (int)std::min<long long>(((long long)m * 32 + 255) / 256, 132 * 16);
  k_ld_scores_sfbm<<<grid, 256, 0, st>>>(s->p, s->rows, s->first_i, s->x, d_sub, m, d_use, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(cudaMemcpyAsync(out, d_out, (size_t)m * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  return BSG_OK;
}

int bsg_lassosum2(bsg_sfbm *corr, const double *beta_hat, int m, const int *ind_sub, int ngrid, const double *lambda,
                  const double *delta_plus_one, double dfmax, int maxiter, double tol, double *beta_est, int *num_iter,
                  double *seconds) {
  if (!corr || m < 0 || ngrid < 0) return fail(BSG_ERR_ARG, "null argument");
  if (ngrid > 0 && (!num_iter || (m > 0 && (!beta_hat || !ind_sub || !lambda || !delta_plus_one || !beta_est))))
    return fail(BSG_ERR_ARG, "null argument");
  if (corr->nrow != corr->ncol) return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  BSG_TRY(check_sub(corr, ind_sub, m));
  if (ngrid == 0) return BSG_OK;
  BSG_TRY(bind(corr));
  // src/lassosum2.cpp:36-37: 2 * inner_product(beta_hat, beta_hat, 0.0), folded in order
  double ss = 0;
  for (int j = 0; j < m; j++) ss = ss + beta_hat[j] * beta_hat[j];
  const double gap0 = 2 * ss;
  cudaStream_t st = corr->stream;
  const size_t mg = (size_t)m * ngrid;
  Bufs b;
  int *d_sub = nullptr, *d_iter = nullptr;
  double *d_bh = nullptr, *d_lam = nullptr, *d_dp1 = nullptr, *d_beta = nullptr, *d_dot = nullptr;
  unsigned long long *d_ns = nullptr;
  BSG_CUDA(b.up(&d_sub, ind_sub, (size_t)m, st));
  BSG_CUDA(b.up(&d_bh, beta_hat, (size_t)m, st));
  b.up(&d_lam, lambda, mg, st);
  b.up(&d_dp1, delta_plus_one, mg, st);
  b.alloc(&d_beta, mg);
  b.alloc(&d_dot, (size_t)corr->ncol * ngrid);
  BSG_TRY(b.status("lassosum2 state"));
  BSG_CUDA(b.alloc(&d_iter, (size_t)ngrid));
  BSG_CUDA(b.alloc(&d_ns, (size_t)ngrid));
  k_lassosum2<<<ngrid, LT, 0, st>>>(corr->p, corr->rows, corr->first_i, corr->x, corr->ncol, d_bh, m, d_sub, d_lam, d_dp1,
                                    dfmax, maxiter, tol, gap0, d_dot, d_beta, d_iter, d_ns);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  if (m > 0) BSG_CUDA(cudaMemcpyAsync(beta_est, d_beta, mg * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(num_iter, d_iter, (size_t)ngrid * sizeof(int), cudaMemcpyDeviceToHost, st));
  std::vector<unsigned long long> ns(ngrid);
  BSG_CUDA(cudaMemcpyAsync(ns.data(), d_ns, (size_t)ngrid * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  if (seconds)
    for (int g = 0; g < ngrid; g++) seconds[g] = ns[g] * 1e-9;
  return BSG_OK;
}

int bsg_sfbm_solve(bsg_sfbm *A, const double *b, const double *add_to_diag, int diag_len, double tol, int maxiter,
                   double *x, int *iters, double *error) {
  if (!A || !b || !add_to_diag || !x || !iters || !error) return fail(BSG_ERR_ARG, "null argument");
  if (A->nrow != A->ncol) return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  const int n = A->ncol;
  if (diag_len != 1 && diag_len != n) return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  if (!(tol >= 0)) return fail(BSG_ERR_ARG, "'tol' must be non-negative.");
  if (maxiter < 0) return fail(BSG_ERR_ARG, "'maxiter' must be non-negative.");
  A->last_solve_ms = 0;
  if (n == 0) {  // b.b == 0
    *iters = 0, *error = 0;
    return BSG_OK;
  }
  BSG_TRY(bind(A));
  cudaStream_t st = A->stream;
  const int nch = (n + CG_CH - 1) / CG_CH;
  Bufs bf;
  double *d_b = nullptr, *d_d = nullptr, *d_x = nullptr, *d_r = nullptr, *d_p = nullptr, *d_t = nullptr;
  double *d_ppt = nullptr, *d_prr = nullptr;
  CgState *d_st = nullptr;
  bf.up(&d_b, b, (size_t)n, st, A->device);
  bf.up(&d_d, add_to_diag, (size_t)diag_len, st, A->device);
  bf.alloc(&d_x, (size_t)n, A->device, st);
  bf.alloc(&d_r, (size_t)n, A->device, st);
  bf.alloc(&d_p, (size_t)n, A->device, st);
  bf.alloc(&d_t, (size_t)n, A->device, st);
  bf.alloc(&d_ppt, (size_t)nch, A->device, st);
  bf.alloc(&d_prr, (size_t)nch, A->device, st);
  bf.alloc(&d_st, 1, A->device, st);
  if (bf.err != cudaSuccess) {
    cudaStreamSynchronize(st);
    return bf.status("solver state");
  }
  k_cg_init<<<nch, CG_DT, 0, st>>>(d_b, n, d_x, d_r, d_p, d_prr);
  k_cg_init_fold<<<1, 32, 0, st>>>(d_prr, nch, d_st);
  count_launch(2);
  BSG_CUDA(cudaGetLastError());
  CgState hs;
  BSG_CUDA(cudaMemcpyAsync(&hs, d_st, sizeof hs, cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  const double rhs2 = hs.rhs2;
  if (rhs2 == 0) {  // x = 0, no iteration, error 0
    memset(x, 0, (size_t)n * sizeof(double));
    *iters = 0, *error = 0;
    return BSG_OK;
  }
  const double threshold = std::max(tol * tol * rhs2, DBL_MIN);
  int it = 0;
  if (hs.rn2 >= threshold) {
    int nsm = 132;
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, A->device);
    const int mgrid = (int)std::min<long long>(((long long)n * 32 + CG_MT - 1) / CG_MT, (long long)nsm * (2048 / CG_MT));
    CallTimer tm;
    cudaError_t e = tm.start(st);
    while (e == cudaSuccess && it < maxiter && !hs.done) {
      const int end = std::min(maxiter, it + CG_BLOCK);
      count_launch(4 * (end - it));
      for (; it < end; it++) {
        k_cg_matvec<<<mgrid, CG_MT, 0, st>>>(A->p, A->rows, A->first_i, A->x, n, d_d, diag_len, d_p, d_t, d_st);
        k_cg_pt<<<nch, CG_DT, 0, st>>>(d_p, d_t, n, d_ppt, d_st);
        k_cg_update<<<nch, CG_DT, 0, st>>>(d_p, d_t, n, d_x, d_r, d_ppt, nch, d_prr, d_st, it);
        k_cg_direction<<<nch, CG_DT, 0, st>>>(d_r, n, d_p, d_prr, nch, threshold, d_st, it);
      }
      e = cudaGetLastError();
      if (e == cudaSuccess) e = cudaMemcpyAsync(&hs, d_st, sizeof hs, cudaMemcpyDeviceToHost, st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(st);
    }
    if (e == cudaSuccess) e = tm.stop(st);
    float ms = 0;
    if (e == cudaSuccess) e = tm.elapsed(&ms);
    A->last_solve_ms = ms;
    if (e != cudaSuccess) return cuda_fail(e, "conjugate gradient");
  }
  BSG_CUDA(cudaMemcpyAsync(x, d_x, (size_t)n * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  *iters = hs.done ? hs.iters : it;  // maxiter when the threshold was never reached
  *error = sqrt(hs.rn2 / rhs2);
  return BSG_OK;
}

double bsg_sfbm_last_solve_ms(const bsg_sfbm *A) { return A ? A->last_solve_ms : -1.0; }

int bsg_ldpred2_auto(bsg_sfbm *corr, const double *beta_hat, const double *n_vec, const double *log_var, int m,
                     const int *ind_sub, int nchain, const double *p_init, double h2_init, int burn_in, int num_iter,
                     int report_step, int no_jump_sign, double shrink_corr, int use_mle, const double *p_bounds,
                     const double *alpha_bounds, double mean_ld, const unsigned *rng_state, double *beta_est,
                     double *postp_est, double *corr_est, double *path_p, double *path_h2, double *path_alpha,
                     double *sample_beta, double *seconds) {
  return bsg_ldpred2_auto_ex(corr, beta_hat, n_vec, log_var, m, ind_sub, nchain, p_init, h2_init, burn_in, num_iter,
                             report_step, no_jump_sign, shrink_corr, use_mle, p_bounds, alpha_bounds, mean_ld, rng_state,
                             beta_est, postp_est, corr_est, path_p, path_h2, path_alpha, sample_beta, seconds, nullptr);
}

int bsg_ldpred2_auto_ex(bsg_sfbm *corr, const double *beta_hat, const double *n_vec, const double *log_var, int m,
                        const int *ind_sub, int nchain, const double *p_init, double h2_init, int burn_in, int num_iter,
                        int report_step, int no_jump_sign, double shrink_corr, int use_mle, const double *p_bounds,
                        const double *alpha_bounds, double mean_ld, const unsigned *rng_state, double *beta_est,
                        double *postp_est, double *corr_est, double *path_p, double *path_h2, double *path_alpha,
                        double *sample_beta, double *seconds, unsigned *rng_out) {
  if (!corr || m < 1 || nchain < 0) return fail(BSG_ERR_ARG, "null argument, m < 1 or nchain < 0");
  if (!beta_hat || !n_vec || !log_var || !ind_sub || !p_bounds || !alpha_bounds)
    return fail(BSG_ERR_ARG, "null argument");
  if (nchain > 0 && (!p_init || !rng_state || !beta_est || !postp_est || !corr_est || !path_p || !path_h2 || !path_alpha))
    return fail(BSG_ERR_ARG, "null argument");
  if (corr->nrow != corr->ncol) return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  if (burn_in < 0 || num_iter < 1 || report_step < 1 || (long long)burn_in + num_iter > INT_MAX)
    return fail(BSG_ERR_ARG, "burn_in must be >= 0, num_iter and report_step >= 1.");
  if (!(p_bounds[0] <= p_bounds[1]) || !(p_bounds[0] > 0))
    return fail(BSG_ERR_ARG, "p_bounds must satisfy 0 < p_bounds[0] <= p_bounds[1].");
  if (!(alpha_bounds[0] <= alpha_bounds[1]) || !std::isfinite(alpha_bounds[0]) || !std::isfinite(alpha_bounds[1]))
    return fail(BSG_ERR_ARG, "alpha_bounds must be finite with alpha_bounds[0] <= alpha_bounds[1].");
  if (!(mean_ld > 0)) return fail(BSG_ERR_ARG, "mean_ld must be positive.");
  BSG_TRY(check_rng(rng_state, nchain, "chain"));
  BSG_TRY(check_sub(corr, ind_sub, m));
  if (nchain == 0) return BSG_OK;
  BSG_TRY(bind(corr));
  double ss = 0;  // src/ldpred2-auto.cpp:96-97, folded in order
  for (int j = 0; j < m; j++) ss = ss + beta_hat[j] * beta_hat[j];
  const int T = burn_in + num_iter, nrep = num_iter / report_step;
  const size_t mc = (size_t)m * nchain, tc = (size_t)T * nchain;
  cudaStream_t st = corr->stream;
  Bufs b;
  LdaArgs A{};
  A.m = m, A.burn_in = burn_in, A.num_iter = num_iter, A.report_step = report_step;
  A.nrep = sample_beta ? nrep : 0;
  A.no_jump_sign = no_jump_sign != 0, A.use_mle = use_mle != 0;
  A.h2_init = h2_init, A.shrink = shrink_corr, A.p_lo = p_bounds[0], A.p_hi = p_bounds[1];
  A.t_lo = alpha_bounds[0], A.t_hi = alpha_bounds[1], A.mean_ld = mean_ld, A.gap0 = 2 * ss;
  double *d_bh = nullptr, *d_n = nullptr, *d_lv = nullptr, *d_pi = nullptr;
  int *d_sub = nullptr;
  uint32_t *d_rng = nullptr;
  b.up(&d_bh, beta_hat, (size_t)m, st);
  b.up(&d_n, n_vec, (size_t)m, st);
  b.up(&d_lv, log_var, (size_t)m, st);
  b.up(&d_pi, p_init, (size_t)nchain, st);
  b.up(&d_sub, ind_sub, (size_t)m, st);
  b.up(&d_rng, (const uint32_t *)rng_state, (size_t)6 * nchain, st);
  double **outs[] = {&A.beta_est, &A.postp_est, &A.corr_est, &A.cb, &A.avg_b, &A.avg_p, &A.avg_bh, &A.abuf, &A.bbuf};
  for (double **o : outs) b.alloc(o, mc);
  double **paths[] = {&A.path_p, &A.path_h2, &A.path_alpha};
  for (double **o : paths) b.alloc(o, tc);
  b.alloc(&A.dot, (size_t)corr->ncol * nchain);
  b.alloc(&A.causal, mc);
  if (A.nrep) b.alloc(&A.sample, mc * A.nrep);
  b.alloc(&A.ns, (size_t)nchain);
  if (rng_out) b.alloc(&A.rng_out, (size_t)6 * nchain);
  BSG_TRY(b.status("ldpred2_auto state"));
  A.beta_hat = d_bh, A.n_vec = d_n, A.log_var = d_lv, A.p_init = d_pi, A.ind_sub = d_sub, A.rng = d_rng;
  k_ldpred2_auto<<<nchain, LT, 0, st>>>(corr->p, corr->rows, corr->first_i, corr->x, corr->ncol, A);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(cudaMemcpyAsync(beta_est, A.beta_est, mc * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(postp_est, A.postp_est, mc * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(corr_est, A.corr_est, mc * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(path_p, A.path_p, tc * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(path_h2, A.path_h2, tc * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(path_alpha, A.path_alpha, tc * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (A.nrep) BSG_CUDA(cudaMemcpyAsync(sample_beta, A.sample, mc * A.nrep * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (rng_out) BSG_CUDA(cudaMemcpyAsync(rng_out, A.rng_out, (size_t)6 * nchain * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
  std::vector<unsigned long long> ns(nchain);
  BSG_CUDA(cudaMemcpyAsync(ns.data(), A.ns, (size_t)nchain * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  if (seconds)
    for (int c = 0; c < nchain; c++) seconds[c] = ns[c] * 1e-9;
  return BSG_OK;
}

int bsg_ldpred2_grid(bsg_sfbm *corr, const double *beta_hat, const double *n_vec, int m, const int *ind_sub, int npoint,
                     const double *p, const double *h2, const int *sparse, int burn_in, int num_iter, int sampling,
                     const unsigned *rng_state, double *beta_est, double *sample_beta, double *seconds) {
  if (!corr || m < 1 || npoint < 0) return fail(BSG_ERR_ARG, "null argument, m < 1 or npoint < 0");
  if (!beta_hat || !n_vec || !ind_sub) return fail(BSG_ERR_ARG, "null argument");
  if (npoint > 0 && (!p || !h2 || !sparse || !rng_state || (sampling ? !sample_beta : !beta_est)))
    return fail(BSG_ERR_ARG, "null argument");
  if (corr->nrow != corr->ncol) return fail(BSG_ERR_DIM, "Incompatibility between dimensions.");
  if (burn_in < 0 || num_iter < 1 || (long long)burn_in + num_iter > INT_MAX)
    return fail(BSG_ERR_ARG, "burn_in must be >= 0 and num_iter >= 1.");
  if (sampling && npoint != 1)
    return fail(BSG_ERR_ARG, "Only one set of parameters is allowed when using 'return_sampling_betas'.");
  BSG_TRY(check_rng(rng_state, npoint, "point"));
  BSG_TRY(check_sub(corr, ind_sub, m));
  if (npoint == 0) return BSG_OK;
  BSG_TRY(bind(corr));
  double ss = 0;  // src/ldpred2.cpp:29-30, folded in order
  for (int j = 0; j < m; j++) ss = ss + beta_hat[j] * beta_hat[j];
  const size_t mp = (size_t)m * npoint, smp = sampling ? (size_t)m * num_iter : 0;
  size_t fr = 0, tot = 0;
  BSG_CUDA(cudaMemGetInfo(&fr, &tot));
  const size_t need = ((size_t)corr->ncol * npoint + 3 * mp + smp + 2 * (size_t)m + 2 * (size_t)npoint) * sizeof(double) +
                      (size_t)npoint * (sizeof(int) + 6 * sizeof(uint32_t) + sizeof(unsigned long long)) + (size_t)m * sizeof(int);
  if (need > fr)
    return fail(BSG_ERR_ALLOC, "ldpred2_grid needs %.0f bytes of device memory for %d points, %.0f are free.", (double)need,
                npoint, (double)fr);
  cudaStream_t st = corr->stream;
  Bufs b;
  LdgArgs A{};
  A.m = m, A.burn_in = burn_in, A.num_iter = num_iter, A.gap0 = 2 * ss;
  double *d_bh = nullptr, *d_n = nullptr, *d_p = nullptr, *d_h2 = nullptr;
  int *d_sub = nullptr, *d_sp = nullptr;
  uint32_t *d_rng = nullptr;
  b.up(&d_bh, beta_hat, (size_t)m, st);
  b.up(&d_n, n_vec, (size_t)m, st);
  b.up(&d_sub, ind_sub, (size_t)m, st);
  b.up(&d_p, p, (size_t)npoint, st);
  b.up(&d_h2, h2, (size_t)npoint, st);
  b.up(&d_sp, sparse, (size_t)npoint, st);
  b.up(&d_rng, (const uint32_t *)rng_state, (size_t)6 * npoint, st);
  b.alloc(&A.beta_est, mp);
  b.alloc(&A.cb, mp);
  b.alloc(&A.avg, mp);
  b.alloc(&A.dot, (size_t)corr->ncol * npoint);
  if (sampling) b.alloc(&A.sample, smp);
  b.alloc(&A.ns, (size_t)npoint);
  BSG_TRY(b.status("ldpred2_grid state"));
  A.beta_hat = d_bh, A.n_vec = d_n, A.p = d_p, A.h2 = d_h2, A.sparse = d_sp, A.ind_sub = d_sub, A.rng = d_rng;
  if (sampling)
    k_ldpred2_grid<true><<<npoint, LT, 0, st>>>(corr->p, corr->rows, corr->first_i, corr->x, corr->ncol, A);
  else
    k_ldpred2_grid<false><<<npoint, LT, 0, st>>>(corr->p, corr->rows, corr->first_i, corr->x, corr->ncol, A);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  if (sampling)
    BSG_CUDA(cudaMemcpyAsync(sample_beta, A.sample, smp * sizeof(double), cudaMemcpyDeviceToHost, st));
  else
    BSG_CUDA(cudaMemcpyAsync(beta_est, A.beta_est, mp * sizeof(double), cudaMemcpyDeviceToHost, st));
  std::vector<unsigned long long> ns(npoint);
  BSG_CUDA(cudaMemcpyAsync(ns.data(), A.ns, (size_t)npoint * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  if (seconds)
    for (int g = 0; g < npoint; g++) seconds[g] = ns[g] * 1e-9;
  return BSG_OK;
}

}  // extern "C"
