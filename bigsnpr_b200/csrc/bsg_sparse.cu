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
#include <math.h>
#include <string.h>

#include <vector>

#include "bsg_internal.cuh"

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
      {  // sfbm->incr_mult_col(j2, dotprods, shift): each row of a column is stored once, so the updates do not collide
        const double shift = s_shift;
        const long long lo = p[cmd], up = p[cmd + 1];
        if (rows) {
          for (long long q = lo + threadIdx.x; q < up; q += LT) {
            const int i = rows[q];
            dp[i] = __dadd_rn(dp[i], __dmul_rn(x[q], shift));
          }
        } else {
          const int i0 = first_i[cmd];
          for (long long q = lo + threadIdx.x; q < up; q += LT) {
            const int i = i0 + (int)(q - lo);
            dp[i] = __dadd_rn(dp[i], __dmul_rn(x[q], shift));
          }
        }
      }
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

static int bind(const bsg_sfbm *s) {
  BSG_CUDA(cudaSetDevice(s->device));
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
    cudaGetLastError();
    bsg_sfbm_close(s);
    return fail(e == cudaErrorMemoryAllocation ? BSG_ERR_ALLOC : BSG_ERR_CUDA, "SFBM does not fit in device memory (%s)",
                cudaGetErrorString(e));
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
  cudaError_t e = b.up(&d_lam, lambda, mg, st);
  if (e == cudaSuccess) e = b.up(&d_dp1, delta_plus_one, mg, st);
  if (e == cudaSuccess) e = b.alloc(&d_beta, mg);
  if (e == cudaSuccess) e = b.alloc(&d_dot, (size_t)corr->ncol * ngrid);
  if (e != cudaSuccess) {
    cudaGetLastError();
    return fail(e == cudaErrorMemoryAllocation ? BSG_ERR_ALLOC : BSG_ERR_CUDA, "lassosum2 state (%s)", cudaGetErrorString(e));
  }
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

}  // extern "C"
