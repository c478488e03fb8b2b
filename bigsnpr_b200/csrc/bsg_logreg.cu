// bsg_logreg.cu -- logistic GWAS with covariates (bigstatsr's big_univLogReg / IRLS, not vendored in the reference):
// per selected SNP j the IRLS fit of y01 on A = [U, x_j] from (gamma0, 0), batched over S SNPs per CTA.
//
// One pass over the ind.train observations is one IRLS step for every SNP a CTA holds.  Per chunk of C observations the
// CTA stages the covariate rows (extended by a constant 1) once, then
//   1. pointwise, per (observation, slot): x from the resident line, eta = u.beta_U + x beta_x, p = 1 / (1 + e^-eta),
//      w = p (1 - p), wz = w eta + (y - p) (= w z), and the five right-hand values w, w x, w x^2, wz, wz x;
//   2. the sums, per (entry, slot): entry e is a product of two extended covariate columns (fa, fb) times one of the
//      five values, so H_UU (u_a u_b . w), H_Ux (u_a . wx), H_xx (1 . wx^2), r_U (u_a . wz) and r_x (1 . wz x) all
//      come out of the same 4 entries x 4 slots register tile.
// Each (entry, slot) sum is owned by one thread: a sequential fma chain over the chunk's observations, added to the
// slot's total in shared memory chunk after chunk.  Its order depends only on (nr, K) -- never on the batch, the grid
// or which thread holds it -- so a SNP's bytes do not depend on the other SNPs of the call.  After a pass one thread
// per slot factors H by Cholesky (x last: std.err = 1 / L_xx), solves for beta, tests max |beta_new - beta_old| < tol
// and, when the SNP is done, writes it and takes the next SNP of the call from a queue (an int counter).
// tests/logreg_ref.py restates the algorithm (DESIGN.md section 4.17).
#include <algorithm>
#include <cmath>
#include <math.h>
#include <vector>

#include "bsg_internal.cuh"

namespace bsg {
namespace logreg {

constexpr int LT = 256;  // threads per CTA
constexpr int LC = 32;   // observations per chunk
constexpr int TE = 4;    // entries per register tile
constexpr int TS = 4;    // slots per register tile
constexpr int NG = 5;    // right-hand values: w, w x, w x^2, w z, w z x
constexpr int SMAX = 64;
constexpr int KMAX = 80;  // covariate vectors: H of K + 1 unknowns fits one CTA's shared memory with 4 slots
constexpr size_t SMEM_MAX = 227 * 1024;

struct LArgs {
  const uint8_t *P;     // hard calls: copy A; dosages: the value copy
  int64_t stride;
  double D;             // dosages: x = byte / D; hard calls: 0 (x = the 2-bit code)
  const int *rows;      // [nr] 0-based samples, one per observation
  const double *U;      // [nr][K] row-major
  const double *y;      // [nr] 0 / 1
  const double *gamma0; // [K]
  const int *cols;      // [nc] 0-based lines
  const uint8_t *bad;   // [nc] NA on a training row or constant: NaN, never iterated
  const short2 *ent;    // [E] (fa, fb) of each entry, index K = the constant 1
  const uint8_t *tile_g;// [E / TE] right-hand value of each entry tile
  int *queue;           // next SNP to take
  int nr, nc, K, E, S, maxiter;
  double tol;
  double *estim, *se;
  int *niter;
};

struct Layout {
  int K, P, E, S, KS;
  size_t o_us, o_y, o_r, o_acc, o_beta, o_g0, o_rows, o_slot, o_ent, o_tg, bytes;
};

// offsets in bytes of the shared-memory arrays (doubles first, then ints, shorts, bytes)
static __host__ __device__ inline Layout layout(int K, int E, int S) {
  Layout L;
  L.K = K, L.P = K + 1, L.E = E, L.S = S, L.KS = K + 1;
  size_t o = 0;
  L.o_us = o, o += sizeof(double) * LC * L.KS;
  L.o_y = o, o += sizeof(double) * LC;
  L.o_r = o, o += sizeof(double) * NG * S * LC;
  L.o_acc = o, o += sizeof(double) * E * S;
  L.o_beta = o, o += sizeof(double) * L.P * S;
  L.o_g0 = o, o += sizeof(double) * K;
  L.o_rows = o, o += sizeof(int) * LC;
  L.o_slot = o, o += sizeof(int) * 3 * S;  // column (line), output index (-1 = empty), steps taken
  L.o_ent = o, o += sizeof(short2) * E;
  L.o_tg = o, o += E / TE;
  L.bytes = (o + 15) / 16 * 16;
  return L;
}

// entry index of H(a, b), a <= b <= K (x = K), and of r(a): the pairs of U (column-major upper triangle), H_Ux, r_U,
// H_xx, r_x, each group padded to TE entries (the table entries() builds)
struct Idx {
  int K, b1, b2, b3, b4;
  __host__ __device__ Idx(int K_) : K(K_) {
    const int n0 = K * (K + 1) / 2, pad = TE;
    b1 = (n0 + pad - 1) / pad * pad;
    b2 = b1 + (K + pad - 1) / pad * pad;
    b3 = b2 + (K + pad - 1) / pad * pad;
    b4 = b3 + pad;
  }
  __host__ __device__ int E() const { return b4 + TE; }
  __host__ __device__ int h(int a, int b) const { return b < K ? b * (b + 1) / 2 + a : (a < K ? b1 + a : b3); }
  __host__ __device__ int r(int a) const { return a < K ? b2 + a : b4; }
};

__device__ __forceinline__ double code_of(const LArgs &a, int line, int row) {
  const uint8_t *p = a.P + (int64_t)line * a.stride;
  if (a.D > 0) return __ddiv_rn((double)p[row], a.D);
  return (double)((p[row >> 2] >> (2 * (row & 3))) & 3);
}

// Cholesky H = R'R in place over the slot's column of acc (upper storage, x last), then R'R beta = r.  false: a pivot
// <= 0 or a non-finite value.
__device__ bool chol_solve(double *A, int S, const Idx &ix, int P, double *beta, double &se) {
  for (int j = 0; j < P; j++) {
    double d = A[(int64_t)ix.h(j, j) * S];
    for (int k = 0; k < j; k++) {
      const double t = A[(int64_t)ix.h(k, j) * S];
      d = __fma_rn(-t, t, d);
    }
    if (!(d > 0) || !isfinite(d)) return false;
    const double rjj = __dsqrt_rn(d);
    A[(int64_t)ix.h(j, j) * S] = rjj;
    for (int i = j + 1; i < P; i++) {
      double v = A[(int64_t)ix.h(j, i) * S];
      for (int k = 0; k < j; k++) v = __fma_rn(-A[(int64_t)ix.h(k, j) * S], A[(int64_t)ix.h(k, i) * S], v);
      A[(int64_t)ix.h(j, i) * S] = __ddiv_rn(v, rjj);
    }
  }
  for (int j = 0; j < P; j++) {  // R' t = r
    double v = A[(int64_t)ix.r(j) * S];
    for (int k = 0; k < j; k++) v = __fma_rn(-A[(int64_t)ix.h(k, j) * S], A[(int64_t)ix.r(k) * S], v);
    A[(int64_t)ix.r(j) * S] = __ddiv_rn(v, A[(int64_t)ix.h(j, j) * S]);
  }
  for (int j = P - 1; j >= 0; j--) {  // R beta = t
    double v = A[(int64_t)ix.r(j) * S];
    for (int k = j + 1; k < P; k++) v = __fma_rn(-A[(int64_t)ix.h(j, k) * S], beta[k], v);
    beta[j] = __ddiv_rn(v, A[(int64_t)ix.h(j, j) * S]);
    if (!isfinite(beta[j])) return false;
  }
  se = __ddiv_rn(1.0, A[(int64_t)ix.h(P - 1, P - 1) * S]);
  return true;
}

__global__ void __launch_bounds__(LT) k_logreg(const LArgs a) {
  extern __shared__ __align__(16) uint8_t smem[];
  const Layout L = layout(a.K, a.E, a.S);
  const Idx ix(a.K);
  const int K = a.K, P = L.P, S = a.S, KS = L.KS, E = a.E, NET = E / TE, NST = S / TS;
  double *us = reinterpret_cast<double *>(smem + L.o_us);
  double *ys = reinterpret_cast<double *>(smem + L.o_y);
  double *R = reinterpret_cast<double *>(smem + L.o_r);  // [g][slot][obs]
  double *acc = reinterpret_cast<double *>(smem + L.o_acc);  // [entry][slot]
  double *beta = reinterpret_cast<double *>(smem + L.o_beta);  // [a][slot]
  double *g0 = reinterpret_cast<double *>(smem + L.o_g0);
  int *rows = reinterpret_cast<int *>(smem + L.o_rows);
  int *s_col = reinterpret_cast<int *>(smem + L.o_slot), *s_out = s_col + S, *s_it = s_out + S;
  short2 *ent = reinterpret_cast<short2 *>(smem + L.o_ent);
  uint8_t *tg = smem + L.o_tg;
  const int tid = threadIdx.x;
  const double nan_ = __longlong_as_double(0x7ff8000000000000LL);
  for (int e = tid; e < E; e += LT) ent[e] = a.ent[e];
  for (int t = tid; t < NET; t += LT) tg[t] = a.tile_g[t];
  for (int k = tid; k < K; k += LT) g0[k] = a.gamma0[k];
  __syncthreads();

  // slot s takes the next SNP of the queue; bad columns are written on the way
  auto take = [&](int s) {
    int j = atomicAdd(a.queue, 1);
    while (j < a.nc && a.bad[j]) {
      a.estim[j] = a.se[j] = nan_;
      a.niter[j] = 0;
      j = atomicAdd(a.queue, 1);
    }
    if (j < a.nc) {
      s_col[s] = a.cols[j], s_out[s] = j, s_it[s] = 0;
      for (int k = 0; k < K; k++) beta[k * S + s] = g0[k];
      beta[K * S + s] = 0.0;
    } else {
      s_out[s] = -1;
    }
  };
  if (tid < S) take(tid);
  __syncthreads();

  while (true) {
    if (!__syncthreads_or(tid < S && s_out[tid] >= 0)) break;
    for (int t = tid; t < E * S; t += LT) acc[t] = 0.0;
    for (int r0 = 0; r0 < a.nr; r0 += LC) {
      const int rc = min(LC, a.nr - r0);
      __syncthreads();  // the previous chunk's sums are done with us / R
      for (int t = tid; t < rc * KS; t += LT) {
        const int r = t / KS, k = t - r * KS;
        us[r * KS + k] = k < K ? a.U[(int64_t)(r0 + r) * K + k] : 1.0;
      }
      for (int r = tid; r < rc; r += LT) {
        ys[r] = a.y[r0 + r];
        rows[r] = a.rows[r0 + r];
      }
      __syncthreads();
      // 1. pointwise values, observation-fast (neighbouring threads read neighbouring codes of one line)
      for (int t = tid; t < S * LC; t += LT) {
        const int s = t / LC, r = t - s * LC;
        double v[NG] = {0.0, 0.0, 0.0, 0.0, 0.0};
        if (r < rc && s_out[s] >= 0) {
          const double x = code_of(a, s_col[s], rows[r]);
          const double *u = us + r * KS;
          double eta = 0.0;
          for (int k = 0; k < K; k++) eta = __fma_rn(u[k], beta[k * S + s], eta);
          eta = __fma_rn(x, beta[K * S + s], eta);
          const double p = __ddiv_rn(1.0, __dadd_rn(1.0, exp(-eta)));
          const double w = __dmul_rn(p, __dsub_rn(1.0, p));
          const double wz = __fma_rn(w, eta, __dsub_rn(ys[r], p));
          v[0] = w;
          v[1] = __dmul_rn(w, x);
          v[2] = __dmul_rn(v[1], x);
          v[3] = wz;
          v[4] = __dmul_rn(wz, x);
        }
#pragma unroll
        for (int g = 0; g < NG; g++) R[(g * S + s) * LC + r] = v[g];
      }
      __syncthreads();
      // 2. the sums: tile (entry tile et, slot tile st), a sequential fma chain over the chunk per (entry, slot)
      for (int tile = tid; tile < NET * NST; tile += LT) {
        const int et = tile % NET, st = tile / NET;
        const int s0 = st * TS;
        const double *Rg = R + ((int)tg[et] * S + s0) * LC;
        int fa[TE], fb[TE];
#pragma unroll
        for (int i = 0; i < TE; i++) fa[i] = ent[et * TE + i].x, fb[i] = ent[et * TE + i].y;
        double part[TE][TS];
#pragma unroll
        for (int i = 0; i < TE; i++)
#pragma unroll
          for (int j = 0; j < TS; j++) part[i][j] = 0.0;
        for (int r = 0; r < rc; r++) {
          const double *u = us + r * KS;
          double l[TE], v[TS];
#pragma unroll
          for (int i = 0; i < TE; i++) l[i] = __dmul_rn(u[fa[i]], u[fb[i]]);
#pragma unroll
          for (int j = 0; j < TS; j++) v[j] = Rg[j * LC + r];
#pragma unroll
          for (int i = 0; i < TE; i++)
#pragma unroll
            for (int j = 0; j < TS; j++) part[i][j] = __fma_rn(l[i], v[j], part[i][j]);
        }
#pragma unroll
        for (int i = 0; i < TE; i++)
#pragma unroll
          for (int j = 0; j < TS; j++) {
            double *q = acc + (et * TE + i) * S + s0 + j;
            *q = __dadd_rn(*q, part[i][j]);
          }
      }
    }
    __syncthreads();
    // 3. one thread per slot: solve, test, write, refill
    if (tid < S && s_out[tid] >= 0) {
      const int s = tid, j = s_out[s];
      double bn[KMAX + 1], se = 0.0;
      const bool ok = chol_solve(acc + s, S, ix, P, bn, se);
      const int it = ++s_it[s];
      bool done = true;
      if (!ok) {
        a.estim[j] = a.se[j] = nan_;
        a.niter[j] = 0;
      } else {
        double diff = 0.0;
        for (int k = 0; k < P; k++) {
          diff = fmax(diff, fabs(__dsub_rn(bn[k], beta[k * S + s])));
          beta[k * S + s] = bn[k];
        }
        if (diff < a.tol || it >= a.maxiter) {
          a.estim[j] = bn[K];
          a.se[j] = se;
          a.niter[j] = diff < a.tol ? it : -it;
        } else {
          done = false;
        }
      }
      if (done) take(s);
    }
    __syncthreads();
  }
}

// Dosage handles: per selected column, NA code or constant value over the training rows
__global__ void k_logreg_check_dos(const uint8_t *__restrict__ raw, int n, const int *__restrict__ lut,
                                   const int *__restrict__ cols, const int *__restrict__ rows, int nr,
                                   uint8_t *__restrict__ bad) {
  const int j = blockIdx.x;
  const uint8_t *col = raw + (int64_t)cols[j] * n;
  const int v0 = lut[col[rows[0]]];
  int any_na = 0, any_diff = 0;
  for (int r = threadIdx.x; r < nr; r += blockDim.x) {
    const int v = lut[col[rows[r]]];
    any_na |= v < 0;
    any_diff |= v != v0;
  }
  any_na = __syncthreads_or(any_na);
  any_diff = __syncthreads_or(any_diff);
  if (threadIdx.x == 0) bad[j] = any_na || !any_diff;
}

// Hard calls: the same flags from the code counts of the column over the training rows
__global__ void k_logreg_check_counts(const int32_t *__restrict__ cnt, int nc, int nr, uint8_t *__restrict__ bad) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc) return;
  const int32_t *c = cnt + 4 * (int64_t)j;
  bad[j] = c[3] > 0 || c[0] == nr || c[1] == nr || c[2] == nr;
}

static thread_local double g_last_ms = 0;

// entries in Idx order, each group padded to TE with (K, K) fillers; tile g per TE entries
static void entries(int K, std::vector<short2> &ent, std::vector<uint8_t> &tg) {
  const Idx ix(K);
  ent.assign(ix.E(), make_short2((short)K, (short)K));
  tg.assign(ix.E() / TE, 0);
  for (int b = 0; b < K; b++)
    for (int a0 = 0; a0 <= b; a0++) ent[ix.h(a0, b)] = make_short2((short)a0, (short)b);
  for (int a0 = 0; a0 < K; a0++) {
    ent[ix.h(a0, K)] = make_short2((short)a0, (short)K);
    ent[ix.r(a0)] = make_short2((short)a0, (short)K);
  }
  for (int t = 0; t < ix.E() / TE; t++) {
    const int e = t * TE;
    tg[t] = e < ix.b1 ? 0 : e < ix.b2 ? 1 : e < ix.b3 ? 3 : e < ix.b4 ? 2 : 4;
  }
}

// S: the multiple of TS up to SMAX that keeps two CTAs per SM and fills the most of the LT threads with register
// tiles (ties: the larger S).  K <= KMAX always fits TS slots.  A SNP's sums do not depend on S.
static int pick_slots(int K, int nc) {
  const Idx ix(K);
  const int net = ix.E() / TE;
  int best = 0;
  double best_eff = -1;
  for (int S = TS; S <= SMAX; S += TS) {
    const size_t b = layout(K, ix.E(), S).bytes;
    if (b > SMEM_MAX) break;
    if (S > TS && b > SMEM_MAX / 2) break;
    const int tiles = net * (S / TS), waves = (tiles + LT - 1) / LT;
    const double eff = (double)tiles / ((double)waves * LT);
    if (eff >= best_eff - 1e-12) best = S, best_eff = eff;
    if (S >= nc) break;  // more slots than SNPs would only idle
  }
  return best;
}

}  // namespace logreg
}  // namespace bsg

using namespace bsg;

extern "C" {

int bsg_univlogreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *U, int K,
                   const double *gamma0, const double *y01, double tol, int maxiter, double *estim, double *std_err,
                   int *niter) {
  using namespace logreg;
  if (!h) return fail(BSG_ERR_ARG, "null handle");
  BSG_TRY(genotypes_check(h, "big_univLogReg on the device needs"));
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  if (nr < 1 || nc < 0 || K < 1) return fail(BSG_ERR_ARG, "Incompatibility between dimensions.");
  if (!(tol > 0)) return fail(BSG_ERR_ARG, "'tol' must be positive.");
  if (maxiter < 1) return fail(BSG_ERR_ARG, "'maxiter' must be at least 1.");
  if (!U || !gamma0 || !y01 || (nc > 0 && (!estim || !std_err || !niter))) return fail(BSG_ERR_ARG, "null argument");
  const int n = h->n;
  std::vector<int> row0, col0;
  BSG_TRY(host_index(ind_row, nr, n, "", row0));
  BSG_TRY(host_index(ind_col, nc, h->m, "", col0));
  for (int r = 0; r < nr; r++)
    if (!(y01[r] == 0.0 || y01[r] == 1.0)) return fail(BSG_ERR_ARG, "'y01.train' must be 0 or 1 (entry %d is not).", r + 1);
  for (int64_t t = 0; t < (int64_t)nr * K; t++)
    if (!std::isfinite(U[t])) return fail(BSG_ERR_ARG, "U must be finite.");
  for (int k = 0; k < K; k++)
    if (!std::isfinite(gamma0[k])) return fail(BSG_ERR_ARG, "gamma0 must be finite.");
  if (K > KMAX) return fail(BSG_ERR_ARG, "big_univLogReg on the device takes at most %d covariate vectors (K = %d).", KMAX, K);
  const int S = pick_slots(K, nc);
  const Idx ix(K);
  const int E = ix.E();
  const Layout lay = layout(K, E, S);
  const size_t need = (size_t)nr * (K * 8 + 8 + 4) + (size_t)K * 8 + (size_t)nc * (4 + 1 + 8 + 8 + 4 + 16) +
                      (size_t)E * 5 + 4096 + 1024;
  size_t fr = 0, tot = 0;
  BSG_CUDA(cudaMemGetInfo(&fr, &tot));
  if (need > fr)
    return fail(BSG_ERR_ALLOC, "big_univLogReg needs %.0f bytes of device memory (%d columns, %d observations, K = %d), "
                               "%.0f are free.", (double)need, nc, nr, K, (double)fr);
  g_last_ms = 0;
  if (nc == 0) return BSG_OK;

  cudaStream_t s = h->stream;
  Bufs b;
  Genotypes g;
  BSG_TRY(genotypes(h, b, &g));
  std::vector<double> Ur((size_t)nr * K);  // row-major [nr][K]
  for (int k = 0; k < K; k++)
    for (int r = 0; r < nr; r++) Ur[(size_t)r * K + k] = U[(size_t)k * nr + r];
  std::vector<short2> ent;
  std::vector<uint8_t> tg;
  entries(K, ent, tg);
  double *d_U, *d_y, *d_g0, *d_est, *d_se;
  int *d_rows, *d_cols, *d_it, *d_queue;
  uint8_t *d_bad, *d_tg;
  short2 *d_ent;
  b.up(&d_U, Ur, s);
  b.up(&d_y, y01, (size_t)nr, s);
  b.up(&d_g0, gamma0, (size_t)K, s);
  b.up(&d_rows, row0, s);
  b.up(&d_cols, col0.data(), (size_t)nc, s);
  b.up(&d_ent, ent, s);
  b.up(&d_tg, tg, s);
  b.alloc(&d_bad, (size_t)nc);
  b.alloc(&d_est, (size_t)nc);
  b.alloc(&d_se, (size_t)nc);
  b.alloc(&d_it, (size_t)nc);
  b.alloc(&d_queue, 1);
  BSG_TRY(b.status("big_univLogReg scratch"));
  BSG_CUDA(cudaMemsetAsync(d_queue, 0, sizeof(int), s));
  CallTimer tm;
  BSG_CUDA(cudaStreamSynchronize(s));
  BSG_CUDA(tm.start(s));
  if (g.dosage) {
    k_logreg_check_dos<<<nc, 256, 0, s>>>(g.raw, n, g.lut, d_cols, d_rows, nr, d_bad);
    count_launch();
  } else {
    int32_t *d_cnt = nullptr;
    BSG_TRY(col_counts_dev(h, ind_row, nr, ind_col, nc, &d_cnt));
    k_logreg_check_counts<<<(nc + 255) / 256, 256, 0, s>>>(d_cnt, nc, nr, d_bad);
    count_launch();
  }
  LArgs a;
  a.P = g.P;
  a.stride = g.stride;
  a.D = g.D;
  a.rows = d_rows;
  a.U = d_U;
  a.y = d_y;
  a.gamma0 = d_g0;
  a.cols = d_cols;
  a.bad = d_bad;
  a.ent = d_ent;
  a.tile_g = d_tg;
  a.queue = d_queue;
  a.nr = nr, a.nc = nc, a.K = K, a.E = E, a.S = S, a.maxiter = maxiter;
  a.tol = tol;
  a.estim = d_est, a.se = d_se, a.niter = d_it;
  BSG_CUDA(cudaFuncSetAttribute(k_logreg, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)lay.bytes));
  int nsm = 132, occ = 1;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->device);
  BSG_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, k_logreg, LT, lay.bytes));
  const int grid = (int)std::max<int64_t>(1, std::min<int64_t>((int64_t)nsm * std::max(occ, 1), (nc + S - 1) / S));
  k_logreg<<<grid, LT, lay.bytes, s>>>(a);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(tm.stop(s));
  BSG_CUDA(cudaMemcpyAsync(estim, d_est, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(std_err, d_se, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(niter, d_it, (size_t)nc * sizeof(int), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  g_last_ms = tm.ms();
  return BSG_OK;
}

double bsg_univlogreg_last_ms(void) { return logreg::g_last_ms; }

}  // extern "C"
