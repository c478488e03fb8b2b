// bsg_ldsplit.cu -- snp_ldsplit (R/split-LD.R:99-138) on the device: get_L (src/split-LD.cpp:15-61), get_C (:65-145),
// reconstruct_paths (R/split-LD.R:3-40) and get_perc (src/split-LD.cpp:149-182), bit-identical to the reference.
//
// corr is the lower triangle in CSC (Matrix::tril): rows sorted, the diagonal first in each column.
//   L(p, j), j > p: the fold of r^2 over column p's entries with row >= j, in descending row order (an r^2 below thr_r2
//   adds nothing, one above max_r2 makes it +Inf).  k_suffix stores that fold at every stored entry, so L(p, j) is the
//   value at the first entry of column p with row >= j (0 when there is none).  bsg_ldsplit_costs reads L from the CSC
//   the caller passes instead: L(p, j) is then a binary search of row p in column j.
//   E(row, col) = sum of L(p, col + 1) for p = col, col - 1, ..., row, in fp64 in that order, stored as float
//   (k_build_E: one warp per col, lookups in parallel, the fold serial over shuffles, no FMA).  E is laid out per col,
//   contiguous in row offset (row = col - min_size + 1 - t at offset t), sized for the largest max_size, so every smaller
//   max_size reads a prefix of it.
//   Layer k >= 1 (k_layer): a warp takes 32 consecutive rows; its lanes walk the same cols in ascending order, so the E
//   reads are consecutive floats and the C1 / C2(col + 1, k - 1) reads are broadcasts.  Each row keeps, per max_size
//   value, the lexicographic min of (E + C1(col + 1, k - 1), size^2 + C2(col + 1, k - 1)); in ascending order a tie
//   goes to the later col, which is the reference's "first visited in descending col" rule.  A candidate equal to
//   (+Inf, +Inf) never wins, as in the reference, where it never beats the initial (+Inf, +Inf).  col = m - 1 is never
//   a candidate for k >= 1: the reference reads C1(m, k - 1) there, which aliases C1(0, k), still +Inf at that moment.
//   One pass over E serves up to LS max_size values.  After each layer k_stop applies the reference's stopping rule
//   per max_size; a stopped value stays inactive (its later layers remain +Inf / NA).
#include <math.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "bsg_internal.cuh"

struct bsg_ldcorr {
  int device = 0;
  int m = 0;
  long long nnz = 0;
  double sumsq2 = 0;  // 2 * sum(x^2), folded in storage order
  long long *p = nullptr;
  int *i = nullptr;
  double *x = nullptr;
  cudaStream_t stream = nullptr;
};

namespace bsg {
namespace ldsplit {

constexpr int LS = 8;  // max_size values per pass over E
constexpr unsigned FULL = 0xffffffffu;
constexpr int NA_INT = (int)0x80000000;

// first q in [lo, hi) with rows[q] >= v (hi when none)
__device__ __forceinline__ long long lower_bound(const int *__restrict__ rows, long long lo, long long hi, int v) {
  while (lo < hi) {
    const long long mid = lo + ((hi - lo) >> 1);
    if (rows[mid] < v)
      lo = mid + 1;
    else
      hi = mid;
  }
  return lo;
}

// one thread per column: suffix[q] = the fold at entry q (entries below the diagonal); rstar[col] = the largest row j
// with L(col, j) > 0, or col when there is none
__global__ void k_suffix(const long long *__restrict__ p, const int *__restrict__ rows, const double *__restrict__ x, int m,
                         double thr_r2, double max_r2, double *__restrict__ suffix, int *__restrict__ rstar) {
  for (int col = blockIdx.x * blockDim.x + threadIdx.x; col < m; col += gridDim.x * blockDim.x) {
    double l = 0;
    int rs = col;
    for (long long k = p[col + 1] - 1; k > p[col]; k--) {
      const double r2 = __dmul_rn(x[k], x[k]);
      if (r2 >= thr_r2) l = (r2 > max_r2) ? INFINITY : __dadd_rn(l, r2);
      suffix[k] = l;
      if (l > 0 && rs == col) rs = rows[k];
    }
    rstar[col] = rs;
  }
}

__device__ __forceinline__ double L_from_corr(const long long *__restrict__ p, const int *__restrict__ rows,
                                              const double *__restrict__ suffix, int pcol, int j) {
  const long long hi = p[pcol + 1], q = lower_bound(rows, p[pcol] + 1, hi, j);
  return q < hi ? suffix[q] : 0.0;
}

__device__ __forceinline__ double L_from_csc(const long long *__restrict__ lp, const int *__restrict__ li,
                                             const double *__restrict__ lx, int prow, int j) {
  const long long hi = lp[j + 1], q = lower_bound(li, lp[j], hi, prow);
  return (q < hi && li[q] == prow) ? lx[q] : 0.0;
}

// get_L's triplets: one warp per column, rows rstar .. col + 1 descending, at off[col] ...
__global__ void k_get_L(const long long *__restrict__ p, const int *__restrict__ rows, const double *__restrict__ suffix,
                        const int *__restrict__ rstar, const long long *__restrict__ off, int m, int *__restrict__ li,
                        int *__restrict__ lj, double *__restrict__ lx) {
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int col = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; col < m; col += nw) {
    const int n = rstar[col] - col;
    for (int t = lane; t < n; t += 32) {
      const int j = rstar[col] - t;
      const long long o = off[col] + t;
      li[o] = col;
      lj[o] = j;
      lx[o] = L_from_corr(p, rows, suffix, col, j);
    }
  }
}

// E for every col: a (p, rows, vals) source is corr with its suffix folds (FROM_CSC false) or L in CSC (true)
template <bool FROM_CSC>
__global__ void k_build_E(const long long *__restrict__ p, const int *__restrict__ rows, const double *__restrict__ vals,
                          int m, const double *__restrict__ pos, int min_size, int max_size, double max_cost,
                          const long long *__restrict__ eoff, float *__restrict__ E, int *__restrict__ elen) {
  const int lane = threadIdx.x & 31, nw = (gridDim.x * blockDim.x) >> 5;
  for (int col = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; col < m; col += nw) {
    const double pos_min = pos[col] - 1;
    float *Ec = E + eoff[col];
    double e = 0;
    int count = 0;
    bool stop = false;
    for (int base = 0; !stop; base += 32) {
      const int row = col - base - lane;
      const bool brk = row < 0 || pos[row] < pos_min;
      double v = 0;
      if (!brk) v = FROM_CSC ? L_from_csc(p, rows, vals, row, col + 1) : L_from_corr(p, rows, vals, row, col + 1);
      const unsigned bad = __ballot_sync(FULL, brk);
      const int nt = bad ? __ffs(bad) - 1 : 32;
      int mine = -1;
      float mye = 0;
      for (int t = 0; t < nt; t++) {  // uniform: every lane holds the same e
        e = __dadd_rn(e, __shfl_sync(FULL, v, t));
        if (e > max_cost) {
          stop = true;
          break;
        }
        count++;
        if (lane == t && count >= min_size) {
          mye = __double2float_rn(e);
          mine = count - min_size;
        }
        if (count == max_size) {
          stop = true;
          break;
        }
      }
      if (nt < 32) stop = true;
      if (mine >= 0) Ec[mine] = mye;
    }
    if (lane == 0) elen[col] = count >= min_size ? count - min_size + 1 : 0;
  }
}

template <class T>
__global__ void k_fill(T *__restrict__ a, size_t n, T v) {
  for (size_t q = blockIdx.x * (size_t)blockDim.x + threadIdx.x; q < n; q += (size_t)gridDim.x * blockDim.x) a[q] = v;
}

// State s of ns: C1 at C1 + s m max_K (m x max_K), best likewise, C2 at C2 + s 2m (layers k - 1 and k alternate).
// Layer 0 (src/split-LD.cpp:112-120): rows m - size for size = min_size .. min(S, lim0), lim0 the pos_scaled cut.
__global__ void k_layer0(int m, int max_K, int min_size, int lim0, const int *__restrict__ Sv, int ns, double *C1,
                         double *C2, int *best) {
  const int nsz = lim0 - min_size + 1;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < ns * nsz; q += gridDim.x * blockDim.x) {
    const int s = q / nsz, size = min_size + q % nsz;
    if (size > Sv[s]) continue;
    const int row = m - size;
    const size_t mK = (size_t)m * max_K;
    C1[s * mK + row] = 0;
    best[s * mK + row] = m;
    C2[(size_t)s * 2 * m + row] = (double)size * size;
  }
}

__global__ void __launch_bounds__(256) k_layer(const float *__restrict__ E, const long long *__restrict__ eoff,
                                               const int *__restrict__ elen, int m, int min_size, int max_K, int k,
                                               const int *__restrict__ Sv, int s0, int ng, const int *__restrict__ active,
                                               double *C1, double *C2, int *best) {
  const int lane = threadIdx.x & 31;
  const int r0 = ((blockIdx.x * blockDim.x + threadIdx.x) >> 5) * 32;
  if (r0 >= m) return;
  const int r = r0 + lane;
  const size_t mK = (size_t)m * max_K;
  int S[LS];
  int smax = 0;
#pragma unroll
  for (int s = 0; s < LS; s++) {
    S[s] = (s < ng && active[s0 + s]) ? Sv[s0 + s] : 0;  // 0: inactive, never a candidate
    smax = max(smax, S[s]);
  }
  if (smax == 0) return;
  double c1[LS], c2[LS];
  int bi[LS];
#pragma unroll
  for (int s = 0; s < LS; s++) {
    c1[s] = INFINITY;
    c2[s] = INFINITY;
    bi[s] = NA_INT;
  }
  const int prev = (k - 1) & 1;
  const int hi = min(m - 2, r0 + 31 + smax - 1);
  for (int col = r0 + min_size - 1; col <= hi; col++) {
    const int size = col - r + 1, t = size - min_size;
    const bool ok = r < m && t >= 0 && size <= smax && t < elen[col];
    const double e = ok ? (double)E[eoff[col] + t] : 0.0;
    const double sz2 = (double)size * size;
#pragma unroll
    for (int s = 0; s < LS; s++) {
      if (!(ok && size <= S[s])) continue;
      const size_t o = (size_t)(s0 + s);
      const double a = __dadd_rn(e, C1[o * mK + (size_t)(k - 1) * m + col + 1]);
      const double b = __dadd_rn(sz2, C2[o * 2 * m + (size_t)prev * m + col + 1]);
      if (!(a == INFINITY && b == INFINITY) && (a < c1[s] || (a == c1[s] && b <= c2[s]))) {
        c1[s] = a;
        c2[s] = b;
        bi[s] = col + 1;
      }
    }
  }
  if (r >= m) return;
#pragma unroll
  for (int s = 0; s < LS; s++) {
    if (S[s] == 0) continue;
    const size_t o = (size_t)(s0 + s);
    C1[o * mK + (size_t)k * m + r] = c1[s];
    best[o * mK + (size_t)k * m + r] = bi[s];
    C2[o * 2 * m + (size_t)(k & 1) * m + r] = c2[s];
  }
}

// src/split-LD.cpp:141: stop after layer k if C1(0, k) > max_cost && C1(0, k) > C1(0, k - 1)
__global__ void k_stop(const double *__restrict__ C1, int m, int max_K, int k, int ns, double max_cost, int *active,
                       int *layers) {
  for (int s = threadIdx.x; s < ns; s += blockDim.x) {
    if (!active[s]) continue;
    const size_t o = (size_t)s * m * max_K;
    const double c = C1[o + (size_t)k * m], cp = C1[o + (size_t)(k - 1) * m];
    if (c > max_cost && c > cp) {
      active[s] = 0;
      layers[s] = k + 1;
    }
  }
}

// R/split-LD.R:3-40, one thread per K: the sorted max_size positions t in order (uniq[t] its state), prev_costs[K]
// shared across them; kept rows get their path (1-based all_last) and cost2.
__global__ void k_paths(const double *__restrict__ C1, const int *__restrict__ best, int m, int max_K,
                        const int *__restrict__ uniq, int nt, double max_cost, int *__restrict__ kept,
                        double *__restrict__ cost, double *__restrict__ cost2, int *__restrict__ all_last) {
  const int K = blockIdx.x * blockDim.x + threadIdx.x + 1;
  if (K > max_K) return;
  const size_t mK = (size_t)m * max_K, T = (size_t)max_K * (max_K + 1) / 2;
  double prev = INFINITY;
  for (int t = 0; t < nt; t++) {
    const size_t o = (size_t)uniq[t] * mK;
    const double c = C1[o + (size_t)(K - 1) * m];
    const size_t row = (size_t)t * max_K + K - 1;
    kept[row] = 0;
    if (c > max_cost || !(c < prev)) continue;
    prev = c;
    int *path = all_last + t * T + (size_t)K * (K - 1) / 2;
    int j = 0, last = 0, ok = 1;
    double c2 = 0;
    for (int kk = K; kk >= 1; kk--) {
      j = best[o + (size_t)(kk - 1) * m + j];
      if (j <= last || j > m || (kk > 1 && j == m)) {  // a finite cost always has a full path
        ok = 0;
        break;
      }
      path[K - kk] = j;
      c2 = __dadd_rn(c2, (double)(j - last) * (j - last));
      last = j;
    }
    kept[row] = ok ? 1 : -1;
    cost[row] = c;
    cost2[row] = c2;
  }
}

// get_perc (src/split-LD.cpp:149-182) of every kept row: one CTA per (t, K); per column j, the stored entries below the
// last row of j's block, found by binary search
__global__ void __launch_bounds__(256) k_perc(const long long *__restrict__ p, const int *__restrict__ rows, int m,
                                              long long nnz, int max_K, const int *__restrict__ kept,
                                              const int *__restrict__ all_last, double *__restrict__ perc) {
  __shared__ unsigned long long s_out;
  const int t = blockIdx.x / max_K, K = blockIdx.x % max_K + 1;
  const size_t row = (size_t)t * max_K + K - 1;
  if (kept[row] != 1) return;
  const int *path = all_last + (size_t)t * max_K * (max_K + 1) / 2 + (size_t)K * (K - 1) / 2;
  if (threadIdx.x == 0) s_out = 0;
  __syncthreads();
  unsigned long long cnt = 0;
  for (int j = threadIdx.x; j < m; j += blockDim.x) {
    int lo = 0, hi = K - 1;  // the first block whose 1-based last index exceeds j
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (path[mid] > j)
        hi = mid;
      else
        lo = mid + 1;
    }
    const int limit = path[lo] - 1;
    cnt += p[j + 1] - lower_bound(rows, p[j], p[j + 1], limit + 1);
  }
  for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(FULL, cnt, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(&s_out, cnt);
  __syncthreads();
  if (threadIdx.x == 0) {
    const long long all = 2 * nnz - m;
    perc[row] = __ddiv_rn((double)(all - 2 * (long long)s_out), (double)all);
  }
}

static int grid_for(long long work, int per_block) {
  return (int)std::max<long long>(1, std::min<long long>((work + per_block - 1) / per_block, 132LL * 32));
}

// E capacity per col: max(0, min(max_size, col + 1) - min_size + 1) floats
static std::vector<long long> e_offsets(int m, int min_size, int max_size) {
  std::vector<long long> off(m + 1, 0);
  for (int c = 0; c < m; c++) off[c + 1] = off[c] + std::max(0, std::min(max_size, c + 1) - min_size + 1);
  return off;
}

static int check_pos(const double *pos, int m) {
  if (!pos) return fail(BSG_ERR_ARG, "null argument");
  for (int j = 0; j < m; j++)
    if (isnan(pos[j])) return fail(BSG_ERR_ARG, "pos_scaled has missing values.");
  return BSG_OK;
}

static int check_sizes(int m, int min_size, const int *S, int nS, int max_K) {
  if (min_size < 1) return fail(BSG_ERR_ARG, "min_size >= 1 is not TRUE");
  if (max_K < 1) return fail(BSG_ERR_ARG, "max_K must be at least 1.");
  for (int s = 0; s < nS; s++) {
    if (S[s] > m) return fail(BSG_ERR_ARG, "all(max_size <= m) is not TRUE");
    if (S[s] < min_size) return fail(BSG_ERR_ARG, "max_size must be at least min_size.");
  }
  return BSG_OK;
}

struct Timer {
  cudaEvent_t ev[4] = {nullptr, nullptr, nullptr, nullptr};
  Timer() {
    for (auto &e : ev) cudaEventCreate(&e);
  }
  ~Timer() {
    for (auto &e : ev)
      if (e) cudaEventDestroy(e);
  }
};

// The shared driver: E from a source (corr with suffix folds, or L in CSC), then every layer for the unique sorted
// max_size values U.  On return the device holds C1 / best for every state (the caller reads what it needs).
struct Run {
  Bufs b;
  double *C1 = nullptr, *C2 = nullptr;
  int *best = nullptr, *Sv = nullptr, *active = nullptr, *layers = nullptr;
  float ms_E = 0, ms_layers = 0;
};

template <bool FROM_CSC>
static int run_layers(Run &R, int device, cudaStream_t st, const long long *src_p, const int *src_rows, const double *src_vals,
                      int m, const double *pos, int min_size, const std::vector<int> &U, int max_K, double max_cost,
                      size_t extra_bytes) {
  const int ns = (int)U.size(), smax = U.back();
  const std::vector<long long> eoff = e_offsets(m, min_size, smax);
  const size_t mK = (size_t)m * max_K;
  const size_t need = (size_t)eoff[m] * sizeof(float) + (size_t)(m + 1) * sizeof(long long) + (size_t)m * (sizeof(int) + sizeof(double)) +
                      (size_t)ns * (mK * (sizeof(double) + sizeof(int)) + 2 * (size_t)m * sizeof(double)) + extra_bytes;
  size_t fr = 0, tot = 0;
  BSG_CUDA(cudaMemGetInfo(&fr, &tot));
  if (need > fr)
    return fail(BSG_ERR_ALLOC, "snp_ldsplit needs %.0f bytes of device memory (E: %.0f bytes for max_size = %d), %.0f are free.",
                (double)need, (double)eoff[m] * sizeof(float), smax, (double)fr);
  // the pos_scaled cut of layer 0 (src/split-LD.cpp:114-120)
  int lim0 = min_size - 1;
  for (int size = min_size; size <= smax; size++) {
    if (pos[m - size] < pos[m - 1] - 1) break;
    lim0 = size;
  }
  long long *d_eoff = nullptr;
  float *d_E = nullptr;
  int *d_elen = nullptr;
  double *d_pos = nullptr;
  R.b.up(&d_eoff, eoff, st);
  R.b.alloc(&d_E, (size_t)eoff[m]);
  R.b.alloc(&d_elen, (size_t)m);
  R.b.up(&d_pos, pos, (size_t)m, st);
  R.b.alloc(&R.C1, ns * mK);
  R.b.alloc(&R.best, ns * mK);
  R.b.alloc(&R.C2, (size_t)ns * 2 * m);
  R.b.up(&R.Sv, U, st);
  R.b.alloc(&R.active, (size_t)ns);
  R.b.alloc(&R.layers, (size_t)ns);
  BSG_TRY(R.b.status("snp_ldsplit state"));
  Timer tm;
  BSG_CUDA(cudaEventRecord(tm.ev[0], st));
  k_build_E<FROM_CSC><<<grid_for((long long)m * 32, 256), 256, 0, st>>>(src_p, src_rows, src_vals, m, d_pos, min_size, smax,
                                                                       max_cost, d_eoff, d_E, d_elen);
  BSG_CUDA(cudaEventRecord(tm.ev[1], st));
  k_fill<double><<<grid_for(ns * mK, 256), 256, 0, st>>>(R.C1, ns * mK, INFINITY);
  k_fill<int><<<grid_for(ns * mK, 256), 256, 0, st>>>(R.best, ns * mK, NA_INT);
  k_fill<double><<<grid_for((long long)ns * 2 * m, 256), 256, 0, st>>>(R.C2, (size_t)ns * 2 * m, INFINITY);
  k_fill<int><<<1, 32, 0, st>>>(R.active, (size_t)ns, 1);
  k_fill<int><<<1, 32, 0, st>>>(R.layers, (size_t)ns, max_K);
  if (lim0 >= min_size)
    k_layer0<<<grid_for((long long)ns * (lim0 - min_size + 1), 256), 256, 0, st>>>(m, max_K, min_size, lim0, R.Sv, ns, R.C1,
                                                                                  R.C2, R.best);
  count_launch(7);
  BSG_CUDA(cudaGetLastError());
  const int warps = (m + 31) / 32, blocks = (warps + 7) / 8;
  std::vector<int> act(ns);
  for (int k = 1; k < max_K; k++) {
    for (int s0 = 0; s0 < ns; s0 += LS)
      k_layer<<<blocks, 256, 0, st>>>(d_E, d_eoff, d_elen, m, min_size, max_K, k, R.Sv, s0, std::min(LS, ns - s0), R.active,
                                      R.C1, R.C2, R.best);
    k_stop<<<1, 32, 0, st>>>(R.C1, m, max_K, k, ns, max_cost, R.active, R.layers);
    count_launch((ns + LS - 1) / LS + 1);
    BSG_CUDA(cudaGetLastError());
    if (k % 8 == 0) {  // end early once every max_size value has stopped
      BSG_CUDA(cudaMemcpyAsync(act.data(), R.active, ns * sizeof(int), cudaMemcpyDeviceToHost, st));
      BSG_CUDA(cudaStreamSynchronize(st));
      if (std::none_of(act.begin(), act.end(), [](int a) { return a != 0; })) break;
    }
  }
  BSG_CUDA(cudaEventRecord(tm.ev[2], st));
  BSG_CUDA(cudaEventSynchronize(tm.ev[2]));
  cudaEventElapsedTime(&R.ms_E, tm.ev[0], tm.ev[1]);
  cudaEventElapsedTime(&R.ms_layers, tm.ev[1], tm.ev[2]);
  (void)device;
  return BSG_OK;
}

static int suffix_folds(bsg_ldcorr *c, double thr_r2, double max_r2, Bufs &b, double **suffix, int **rstar) {
  BSG_CUDA(b.alloc(suffix, (size_t)c->nnz));
  BSG_CUDA(b.alloc(rstar, (size_t)c->m));
  k_suffix<<<grid_for(c->m, 128), 128, 0, c->stream>>>(c->p, c->i, c->x, c->m, thr_r2, max_r2, *suffix, *rstar);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

static int bind(const bsg_ldcorr *c) {
  BSG_CUDA(cudaSetDevice(c->device));
  return BSG_OK;
}

}  // namespace ldsplit
}  // namespace bsg

using namespace bsg;
using namespace bsg::ldsplit;

extern "C" {

int bsg_ldcorr_open(int m, const long long *p, const int *i, const double *x, int device, bsg_ldcorr **out) {
  if (!out) return fail(BSG_ERR_ARG, "null argument");
  *out = nullptr;
  if (m < 1 || !p || !i || !x) return fail(BSG_ERR_ARG, "bad dimensions or null argument");
  if (p[0] != 0) return fail(BSG_ERR_ARG, "p[0] must be 0.");
  for (int j = 0; j < m; j++) {
    if (p[j + 1] <= p[j]) return fail(BSG_ERR_ARG, "all(Matrix::diag(corr) != 0) is not TRUE");  // an empty column
    if (i[p[j]] != j || x[p[j]] == 0) return fail(BSG_ERR_ARG, "all(Matrix::diag(corr) != 0) is not TRUE");
    for (long long q = p[j] + 1; q < p[j + 1]; q++)
      if (i[q] <= i[q - 1] || i[q] >= m)
        return fail(BSG_ERR_ARG, "column %d: rows must be increasing, in [column, m) (the lower triangle).", j);
  }
  const long long nnz = p[m];
  double ss = 0;
  for (long long q = 0; q < nnz; q++) ss = ss + x[q] * x[q];
  if (cudaSetDevice(device) != cudaSuccess) {
    cudaGetLastError();
    return fail(BSG_ERR_CUDA, "CUDA device %d is not available (no CPU fallback).", device);
  }
  bsg_ldcorr *c = new bsg_ldcorr();
  c->device = device;
  c->m = m;
  c->nnz = nnz;
  c->sumsq2 = ss * 2;
  cudaError_t e = cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking);
  if (e == cudaSuccess) e = cudaMalloc(&c->p, (m + 1) * sizeof(long long));
  if (e == cudaSuccess) e = cudaMalloc(&c->i, nnz * sizeof(int));
  if (e == cudaSuccess) e = cudaMalloc(&c->x, nnz * sizeof(double));
  if (e != cudaSuccess) {
    bsg_ldcorr_close(c);
    return alloc_fail(e, "corr does not fit in device memory");
  }
  e = cudaMemcpy(c->p, p, (m + 1) * sizeof(long long), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(c->i, i, nnz * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(c->x, x, nnz * sizeof(double), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    bsg_ldcorr_close(c);
    return cuda_fail(e, "corr upload");
  }
  *out = c;
  return BSG_OK;
}

void bsg_ldcorr_close(bsg_ldcorr *c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->stream) cudaStreamSynchronize(c->stream);
  void *ptrs[] = {c->p, c->i, c->x};
  for (void *q : ptrs)
    if (q) cudaFree(q);
  if (c->stream) cudaStreamDestroy(c->stream);
  delete c;
}

int bsg_ldcorr_m(const bsg_ldcorr *c) { return c ? c->m : -1; }
double bsg_ldcorr_sumsq2(const bsg_ldcorr *c) { return c ? c->sumsq2 : NAN; }

int bsg_ldcorr_l_triplets(bsg_ldcorr *c, double thr_r2, double max_r2, long long *count, long long cap, int *li, int *lj,
                     double *lx) {
  if (!c || !count || (cap > 0 && (!li || !lj || !lx))) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(bind(c));
  cudaStream_t st = c->stream;
  Bufs b;
  double *d_suf = nullptr;
  int *d_rs = nullptr;
  BSG_TRY(suffix_folds(c, thr_r2, max_r2, b, &d_suf, &d_rs));
  std::vector<int> rs(c->m);
  BSG_CUDA(cudaMemcpyAsync(rs.data(), d_rs, c->m * sizeof(int), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  std::vector<long long> off(c->m + 1, 0);
  for (int j = 0; j < c->m; j++) off[j + 1] = off[j] + (rs[j] - j);
  *count = off[c->m];
  if (cap <= 0) return BSG_OK;
  if (cap < off[c->m]) return fail(BSG_ERR_ARG, "get_L: room for %lld triplets, %lld needed.", cap, off[c->m]);
  const size_t n = (size_t)off[c->m];
  long long *d_off = nullptr;
  int *d_li = nullptr, *d_lj = nullptr;
  double *d_lx = nullptr;
  b.up(&d_off, off, st);
  b.alloc(&d_li, n);
  b.alloc(&d_lj, n);
  b.alloc(&d_lx, n);
  BSG_TRY(b.status("get_L triplets"));
  k_get_L<<<grid_for((long long)c->m * 32, 256), 256, 0, st>>>(c->p, c->i, d_suf, d_rs, d_off, c->m, d_li, d_lj, d_lx);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  if (n) {
    BSG_CUDA(cudaMemcpyAsync(li, d_li, n * sizeof(int), cudaMemcpyDeviceToHost, st));
    BSG_CUDA(cudaMemcpyAsync(lj, d_lj, n * sizeof(int), cudaMemcpyDeviceToHost, st));
    BSG_CUDA(cudaMemcpyAsync(lx, d_lx, n * sizeof(double), cudaMemcpyDeviceToHost, st));
  }
  BSG_CUDA(cudaStreamSynchronize(st));
  return BSG_OK;
}

int bsg_ldsplit(bsg_ldcorr *c, double thr_r2, int min_size, const int *max_size, int n_max_size, int max_K, double max_r2,
                double max_cost, const double *pos_scaled, int *kept, double *cost, double *cost2, double *perc_kept,
                int *all_last, int *layers, double *seconds) {
  if (!c || n_max_size < 1 || !max_size || !kept || !cost || !cost2 || !perc_kept || !all_last)
    return fail(BSG_ERR_ARG, "null argument");
  const int m = c->m;
  BSG_TRY(check_sizes(m, min_size, max_size, n_max_size, max_K));
  BSG_TRY(check_pos(pos_scaled, m));
  BSG_TRY(bind(c));
  max_cost = std::min(max_cost, c->sumsq2);  // R/split-LD.R:111
  std::vector<int> sorted(max_size, max_size + n_max_size);
  std::sort(sorted.begin(), sorted.end());
  std::vector<int> U, uniq(n_max_size);
  for (int t = 0; t < n_max_size; t++) {
    if (U.empty() || U.back() != sorted[t]) U.push_back(sorted[t]);
    uniq[t] = (int)U.size() - 1;
  }
  const size_t nrow = (size_t)n_max_size * max_K, T = (size_t)max_K * (max_K + 1) / 2;
  cudaStream_t st = c->stream;
  Bufs b;
  double *d_suf = nullptr;
  int *d_rs = nullptr;
  BSG_TRY(suffix_folds(c, thr_r2, max_r2, b, &d_suf, &d_rs));
  Run R;
  BSG_TRY(run_layers<false>(R, c->device, st, c->p, c->i, d_suf, m, pos_scaled, min_size, U, max_K, max_cost,
                            nrow * (sizeof(int) + 3 * sizeof(double)) + n_max_size * T * sizeof(int)));
  int *d_uniq = nullptr, *d_kept = nullptr, *d_path = nullptr;
  double *d_cost = nullptr, *d_cost2 = nullptr, *d_perc = nullptr;
  b.up(&d_uniq, uniq, st);
  b.alloc(&d_kept, nrow);
  b.alloc(&d_cost, nrow);
  b.alloc(&d_cost2, nrow);
  b.alloc(&d_perc, nrow);
  b.alloc(&d_path, n_max_size * T);
  BSG_TRY(b.status("snp_ldsplit results"));
  Timer tm;
  BSG_CUDA(cudaEventRecord(tm.ev[0], st));
  BSG_CUDA(cudaMemsetAsync(d_path, 0, n_max_size * T * sizeof(int), st));
  BSG_CUDA(cudaMemsetAsync(d_perc, 0, nrow * sizeof(double), st));
  k_paths<<<(max_K + 127) / 128, 128, 0, st>>>(R.C1, R.best, m, max_K, d_uniq, n_max_size, max_cost, d_kept, d_cost, d_cost2,
                                                d_path);
  k_perc<<<(unsigned)nrow, 256, 0, st>>>(c->p, c->i, m, c->nnz, max_K, d_kept, d_path, d_perc);
  count_launch(2);
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(cudaEventRecord(tm.ev[1], st));
  BSG_CUDA(cudaMemcpyAsync(kept, d_kept, nrow * sizeof(int), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(cost, d_cost, nrow * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(cost2, d_cost2, nrow * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(perc_kept, d_perc, nrow * sizeof(double), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaMemcpyAsync(all_last, d_path, n_max_size * T * sizeof(int), cudaMemcpyDeviceToHost, st));
  std::vector<int> nl(U.size());
  BSG_CUDA(cudaMemcpyAsync(nl.data(), R.layers, U.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  BSG_CUDA(cudaStreamSynchronize(st));
  for (size_t q = 0; q < nrow; q++)
    if (kept[q] < 0) return fail(BSG_ERR_CUDA, "snp_ldsplit: a kept split has an incomplete path.");
  if (layers)
    for (int t = 0; t < n_max_size; t++) layers[t] = nl[uniq[t]];
  if (seconds) {
    float ms = 0;
    cudaEventElapsedTime(&ms, tm.ev[0], tm.ev[1]);
    seconds[0] = R.ms_E * 1e-3;
    seconds[1] = R.ms_layers * 1e-3;
    seconds[2] = ms * 1e-3;
  }
  return BSG_OK;
}

int bsg_ldsplit_costs(int m, const long long *lp, const int *li, const double *lx, int min_size, int max_size, int max_K,
                      double max_cost, const double *pos_scaled, int device, double *C, int *best_ind) {
  if (m < 1 || !lp || !C || !best_ind) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(check_sizes(m, min_size, &max_size, 1, max_K));
  BSG_TRY(check_pos(pos_scaled, m));
  if (lp[0] != 0) return fail(BSG_ERR_ARG, "L: p[0] must be 0.");
  for (int j = 0; j <= m; j++)
    if (lp[j + 1] < lp[j]) return fail(BSG_ERR_ARG, "L: p must be non-decreasing.");
  const long long nl = lp[m + 1];
  if (nl > 0 && (!li || !lx)) return fail(BSG_ERR_ARG, "null argument");
  for (int j = 0; j <= m; j++)
    for (long long q = lp[j]; q < lp[j + 1]; q++)
      if (li[q] < 0 || li[q] >= m || (q > lp[j] && li[q] <= li[q - 1]))
        return fail(BSG_ERR_ARG, "L: column %d: rows must be increasing, in [0, m).", j);
  if (cudaSetDevice(device) != cudaSuccess) {
    cudaGetLastError();
    return fail(BSG_ERR_CUDA, "CUDA device %d is not available (no CPU fallback).", device);
  }
  cudaStream_t st = nullptr;
  BSG_CUDA(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
  struct StreamGuard {
    cudaStream_t s;
    ~StreamGuard() {
      cudaStreamSynchronize(s);
      cudaStreamDestroy(s);
    }
  } guard{st};
  int rc;
  {
    Bufs b;
    long long *d_lp = nullptr;
    int *d_li = nullptr;
    double *d_lx = nullptr;
    b.up(&d_lp, lp, (size_t)m + 2, st);
    b.up(&d_li, li, (size_t)nl, st);
    b.up(&d_lx, lx, (size_t)nl, st);
    BSG_TRY(b.status("L does not fit in device memory"));
    Run R;
    rc = run_layers<true>(R, device, st, d_lp, d_li, d_lx, m, pos_scaled, min_size, std::vector<int>{max_size}, max_K,
                          max_cost, 0);
    if (rc == BSG_OK) {
      const size_t mK = (size_t)m * max_K;
      BSG_CUDA(cudaMemcpyAsync(C, R.C1, mK * sizeof(double), cudaMemcpyDeviceToHost, st));
      BSG_CUDA(cudaMemcpyAsync(best_ind, R.best, mK * sizeof(int), cudaMemcpyDeviceToHost, st));
      BSG_CUDA(cudaStreamSynchronize(st));
    }
  }
  return rc;
}

}  // extern "C"
