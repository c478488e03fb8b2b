// bsg_gwas.cu -- linear GWAS with covariates (bigstatsr's big_univLinReg / univLinReg5, not vendored in the reference):
// every selected SNP column against y and the K orthonormal covariate vectors U in ONE pass over the SNP-major copy.
//
// Per column j the statistic needs the V = K + 1 sums  x_j . v  (v = y and the columns of U) over the ind.train rows, plus
// sum x, sum x^2 and the missing-value flag.  The vectors are quantised once per call on the host (y to 61-bit fixed point,
// 8 signed base-256 digits; the columns of U to 30-bit fixed point, 4 digits), scattered onto the n sample positions (a repeated row
// adds its entries in integers), and their digits become the N dimension of mma.sync.m16n8k32.u8.s8: one 8-wide N tile
// holds 8 (vector, digit) slices, so the code fragments of a word are loaded once and feed 2 x NT MMAs.  Sums of
// codes x digits are exact in int32 per work item and in int64 per line, hence independent of the work split.
// Hard calls: the 2-bit code is the value (field f of a byte is extracted by (w >> 2f) & 0x03030303, all four fields into
// the same accumulator).  Dosage FBMs (bsg_dosage_scale D > 0): the same slice sums over the value bytes D x code by a
// SIMT kernel, divided by D once per sum.  Sums x, x^2 and the NA flag: the column counts (hard calls) or exact integer
// sums of the bytes (dosages).  The epilogue (k_gwas_stats) turns the sums into estim / std.err in fp64 with a fixed
// operation order (explicit _rn intrinsics, no contraction); tests/gwas_ref.py restates every step.
#include <algorithm>
#include <cmath>
#include <math.h>
#include <vector>

#include "bsg_internal.cuh"
#include "bsg_pmv_shared.cuh"

namespace bsg {
namespace gwas {

using pmv::lds128;
using pmv::ldg_stream;
using pmv::mma_u8s8;
using pmv::smem_u32;

constexpr int GW = 8;                 // consumer warps per CTA, 32 lines (two 16-line MMA row tiles) each
constexpr int GLINES = GW * 32;       // lines per work item
constexpr int GSTAGES = 3;            // digit stages in shared memory
constexpr int SEG = 128;              // bytes per line per chunk = 512 codes
constexpr int NTMAX = 8;              // N tiles per pass: 64 slices
constexpr int SMAX = 8 * NTMAX;
constexpr int MAX_CHUNKS_PER_ITEM = 4096;  // |acc| <= 4096 * 512 * 3 * 128 < 2^31
constexpr int Y_BITS = 60, U_BITS = 30;    // |sum of quantised entries| < 2^bits (as pick_e of the matvecs)
constexpr int Y_DIG = 8, U_DIG = 4;

struct GArgs {
  const uint8_t *P;
  int64_t stride;
  const int *lines;  // physical line per logical line (null = identity)
  int nlines, nlines_pad, nchunks, chunks_per_split, ksplit;
  const uint8_t *dig;  // [nchunks][8 words][NT][32 lanes][16 B]
  long long *part;     // [nlines_pad][SMAX]
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

struct Frag {
  uint4 alo, ahi, blo, bhi;  // lines g / g + 8 of the row tile, bytes [16q, 16q + 16) and [64 + 16q, 64 + 16q + 16)
};

__device__ __forceinline__ void frag_load(Frag &f, const uint8_t *pa, const uint8_t *pb, int64_t off) {
  f.alo = ldg_stream(pa + off);
  f.ahi = ldg_stream(pa + off + 64);
  f.blo = ldg_stream(pb + off);
  f.bhi = ldg_stream(pb + off + 64);
}

__device__ __forceinline__ uint32_t word_of(const Frag &f, int w, bool b) {
  const uint4 &v = b ? (w < 4 ? f.blo : f.bhi) : (w < 4 ? f.alo : f.ahi);
  const int k = w & 3;
  return k == 0 ? v.x : (k == 1 ? v.y : (k == 2 ? v.z : v.w));
}

// One work item = 256 lines x a range of chunks.  Lane (g, q) of warp w holds, per 16-line row tile u, the fragment bytes
// of lines g and g + 8; word w of the chunk feeds, for each N tile t, MMA (fields 0, 1) with digit registers x, y and
// MMA (fields 2, 3) with z, w of the 16-byte unit (w, t, lane) -- the layout k_gwas_digits writes.
template <int NT>
__global__ void __launch_bounds__(GW * 32, 1) k_gwas(const GArgs a) {
  constexpr int CH = 4096 * NT;  // digit bytes per chunk
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sbase = smem_u32(smem);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int ngroups = a.nlines_pad / GLINES, nitems = ngroups * a.ksplit;
  for (int item = blockIdx.x; item < nitems; item += gridDim.x) {
    const int group = item / a.ksplit, ks = item - group * a.ksplit;
    const int c0 = ks * a.chunks_per_split, c1 = min(a.nchunks, c0 + a.chunks_per_split);
    const uint8_t *pA[2], *pB[2];
#pragma unroll
    for (int u = 0; u < 2; u++) {
      const int la = min(group * GLINES + warp * 32 + u * 16 + g, a.nlines - 1);
      const int lb = min(group * GLINES + warp * 32 + u * 16 + g + 8, a.nlines - 1);
      pA[u] = a.P + (int64_t)(a.lines ? a.lines[la] : la) * a.stride + 16 * q;
      pB[u] = a.P + (int64_t)(a.lines ? a.lines[lb] : lb) * a.stride + 16 * q;
    }
    int acc[2][NT][4];
#pragma unroll
    for (int u = 0; u < 2; u++)
#pragma unroll
      for (int t = 0; t < NT; t++)
#pragma unroll
        for (int k = 0; k < 4; k++) acc[u][t][k] = 0;
    auto stage_load = [&](int c, int buf) {
      for (int o = threadIdx.x * 16; o < CH; o += GW * 32 * 16)
        cp_async16(sbase + buf * CH + o, a.dig + (int64_t)c * CH + o);
    };
#pragma unroll
    for (int s = 0; s < GSTAGES - 1; s++) {
      if (c0 + s < c1) stage_load(c0 + s, s);
      cp_async_commit();
    }
    Frag cur[2];
#pragma unroll
    for (int u = 0; u < 2; u++) frag_load(cur[u], pA[u], pB[u], (int64_t)c0 * SEG);
    for (int c = c0; c < c1; c++) {
      const int it = c - c0;
      if (c + GSTAGES - 1 < c1) stage_load(c + GSTAGES - 1, (it + GSTAGES - 1) % GSTAGES);
      cp_async_commit();
      Frag nxt[2];
      const bool more = c + 1 < c1;
#pragma unroll
      for (int u = 0; u < 2; u++)
        if (more) frag_load(nxt[u], pA[u], pB[u], (int64_t)(c + 1) * SEG);
      cp_async_wait<GSTAGES - 1>();
      __syncthreads();
      const uint32_t dbase = sbase + (it % GSTAGES) * CH + lane * 16;
#pragma unroll
      for (int w = 0; w < 8; w++) {
        uint32_t A[2][4][2];  // [row tile][field][line g | g + 8]
#pragma unroll
        for (int u = 0; u < 2; u++) {
          const uint32_t wa = word_of(cur[u], w, false), wb = word_of(cur[u], w, true);
#pragma unroll
          for (int f = 0; f < 4; f++) {
            A[u][f][0] = (wa >> (2 * f)) & 0x03030303u;
            A[u][f][1] = (wb >> (2 * f)) & 0x03030303u;
          }
        }
#pragma unroll
        for (int t = 0; t < NT; t++) {
          const uint4 d = lds128(dbase + (uint32_t)((w * NT + t) * 512));
#pragma unroll
          for (int u = 0; u < 2; u++) {
            mma_u8s8(acc[u][t], A[u][0][0], A[u][0][1], A[u][1][0], A[u][1][1], d.x, d.y);
            mma_u8s8(acc[u][t], A[u][2][0], A[u][2][1], A[u][3][0], A[u][3][1], d.z, d.w);
          }
        }
      }
      if (more) {
        cur[0] = nxt[0];
        cur[1] = nxt[1];
      }
      __syncthreads();  // every warp is done with this stage before it is refilled
    }
    cp_async_wait<0>();
    // accumulator k of row tile u, N tile t: line g + 8 (k >> 1), slice 8 t + 2 q + (k & 1)
#pragma unroll
    for (int u = 0; u < 2; u++)
#pragma unroll
      for (int t = 0; t < NT; t++)
#pragma unroll
        for (int k = 0; k < 4; k++) {
          const int line = group * GLINES + warp * 32 + u * 16 + g + 8 * (k >> 1);
          if (acc[u][t][k])
            atomicAdd(reinterpret_cast<unsigned long long *>(a.part) + (int64_t)line * SMAX + 8 * t + 2 * q + (k & 1),
                      (unsigned long long)(long long)acc[u][t][k]);
        }
    __syncthreads();
  }
}

struct SlotMap {
  int vec[SMAX];  // vector (row of Q) of slice s, -1 = padding
  int dig[SMAX];  // its digit index
};

__device__ __forceinline__ int digit_of(long long q, int d) {
  int r = 0;
  for (int i = 0; i <= d; i++) r = pmv::peel(q);
  return r;
}

// Digit layout of k_gwas: one thread per 16-byte unit (chunk, w, t, g, q): register c, byte r = digit of slice 8 t + g of
// code (w < 4 ? 64 q + 16 w : 256 + 64 q + 16 (w - 4)) + 4 r + c of the chunk.
__global__ void k_gwas_digits(const long long *__restrict__ Q, int n, int nchunks, int NT, const SlotMap map,
                              uint8_t *__restrict__ dig) {
  const int64_t total = (int64_t)nchunks * 8 * NT * 32;
  for (int64_t x = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; x < total; x += (int64_t)gridDim.x * blockDim.x) {
    const int lane = (int)(x & 31), g = lane >> 2, q = lane & 3;
    const int64_t wt = x >> 5;
    const int t = (int)(wt % NT), w = (int)((wt / NT) & 7);
    const int64_t chunk = wt / NT / 8;
    const int s = 8 * t + g, v = map.vec[s], d = map.dig[s];
    uint32_t o[4] = {0, 0, 0, 0};
    if (v >= 0) {
#pragma unroll
      for (int c = 0; c < 4; c++)
#pragma unroll
        for (int r = 0; r < 4; r++) {
          const int64_t k = chunk * 512 + (w < 4 ? 64 * q + 16 * w : 256 + 64 * q + 16 * (w - 4)) + 4 * r + c;
          if (k < n) o[c] |= (uint32_t)(digit_of(Q[(int64_t)v * n + k], d) & 0xFF) << (8 * r);
        }
    }
    reinterpret_cast<uint4 *>(dig)[x] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// Dosage handles: digits by sample, [slice][n]
__global__ void k_gwas_digits_rows(const long long *__restrict__ Q, int n, int S, const SlotMap map, int8_t *__restrict__ dig) {
  const int64_t total = (int64_t)S * n;
  for (int64_t x = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; x < total; x += (int64_t)gridDim.x * blockDim.x) {
    const int s = (int)(x / n);
    const int64_t i = x - (int64_t)s * n;
    const int v = map.vec[s];
    dig[x] = v >= 0 ? (int8_t)digit_of(Q[(int64_t)v * n + i], map.dig[s]) : 0;
  }
}

// Dosage handles: one CTA per selected column, exact sums of value byte x digit per slice over every sample (digits of
// unselected samples are 0), and, on the first pass, sum mult x byte, sum mult x byte^2 and the NA count over ind.train.
constexpr int DT = 256;
__global__ void __launch_bounds__(DT) k_gwas_dos(const uint8_t *__restrict__ raw, int n, const int *__restrict__ lut,
                                                 const int *__restrict__ cols, const int *__restrict__ mult,
                                                 const int8_t *__restrict__ dig, int S, long long *__restrict__ part,
                                                 long long *__restrict__ xs) {
  __shared__ int slut[256];
  __shared__ long long red[DT / 32];
  slut[threadIdx.x] = lut[threadIdx.x];
  __syncthreads();
  const int j = blockIdx.x;
  const uint8_t *col = raw + (int64_t)cols[j] * n;
  for (int s0 = 0; s0 < S; s0 += 16) {
    long long acc[16];
#pragma unroll
    for (int k = 0; k < 16; k++) acc[k] = 0;
    for (int i = threadIdx.x; i < n; i += DT) {
      const int v = max(slut[col[i]], 0);
#pragma unroll
      for (int k = 0; k < 16; k++)
        if (s0 + k < S) acc[k] += v * (int)dig[(int64_t)(s0 + k) * n + i];
    }
#pragma unroll
    for (int k = 0; k < 16; k++) {
      long long t = acc[k];
      for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
      __syncthreads();
      if (threadIdx.x == 0 && s0 + k < S) {
        long long tot = 0;
        for (int w = 0; w < DT / 32; w++) tot += red[w];
        part[(int64_t)j * SMAX + s0 + k] = tot;
      }
      __syncthreads();
    }
  }
  if (xs) {
    long long sx = 0, sxx = 0, na = 0;
    for (int i = threadIdx.x; i < n; i += DT) {
      const int m = mult[i];
      if (!m) continue;
      const int v = slut[col[i]];
      if (v < 0) {
        na += m;
      } else {
        sx += (long long)m * v;
        sxx += (long long)m * v * v;
      }
    }
    long long r3[3] = {sx, sxx, na};
    for (int k = 0; k < 3; k++) {
      long long t = r3[k];
      for (int o = 16; o; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
      if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = t;
      __syncthreads();
      if (threadIdx.x == 0) {
        long long tot = 0;
        for (int w = 0; w < DT / 32; w++) tot += red[w];
        xs[(int64_t)j * 3 + k] = tot;
      }
      __syncthreads();
    }
  }
}

// Hard calls: sum x, sum x^2 and the NA count from the column counts
__global__ void k_gwas_xs_counts(const int32_t *__restrict__ cnt, int nc, long long *__restrict__ xs) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc) return;
  const long long c1 = cnt[4 * (int64_t)j + 1], c2 = cnt[4 * (int64_t)j + 2], c3 = cnt[4 * (int64_t)j + 3];
  xs[3 * (int64_t)j + 0] = c1 + 2 * c2;
  xs[3 * (int64_t)j + 1] = c1 + 4 * c2;
  xs[3 * (int64_t)j + 2] = c3;
}

// The slices of one vector -> x . v in fp64: exact integer slice totals, one top-down sum of the scaled totals
// (slice d weighs 2^(8 d - e)), then one division by D.  Out: S[vec][line].
__global__ void k_gwas_combine(const long long *__restrict__ part, int nc, int s0, int nd, int e, double D,
                               double *__restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc) return;
  double acc = 0.0;
  for (int d = nd - 1; d >= 0; d--) acc = __dadd_rn(acc, scalbn((double)part[(int64_t)j * SMAX + s0 + d], 8 * d - e));
  out[j] = __ddiv_rn(acc, D);
}

__device__ __forceinline__ double u128_to_double(unsigned __int128 v) {
  const unsigned long long hi = (unsigned long long)(v >> 64), lo = (unsigned long long)v;
  return __dadd_rn(__dmul_rn(__ull2double_rn(hi), 18446744073709551616.0), __ull2double_rn(lo));
}

// estim / std.err per column.  xs = (sum b, sum b^2, NA count) of the value bytes b = D x (hard calls: D = 1); S[0] = x.y_c,
// S[1 + k] = x.u_k; host scalars hs = (n, D, df, yres) and per k (u1_k = 1'u_k, uy_k = u_k'y_c).
__global__ void k_gwas_stats(const long long *__restrict__ xs, const double *__restrict__ S, int nc, int K,
                             const double *__restrict__ u1, const double *__restrict__ uy, long long n, double D, double df,
                             double yres, double *__restrict__ estim, double *__restrict__ se) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nc) return;
  const long long sx = xs[3 * (int64_t)j], sxx = xs[3 * (int64_t)j + 1], na = xs[3 * (int64_t)j + 2];
  const __int128 num_i = (__int128)n * sxx - (__int128)sx * sx;  // n^2 D^2 var(x), exact
  const double nan_ = __longlong_as_double(0x7ff8000000000000LL);
  if (na > 0 || num_i <= 0) {
    estim[j] = se[j] = nan_;
    return;
  }
  const double nd = __dmul_rn((double)n, D);
  const double ssx = __ddiv_rn(u128_to_double((unsigned __int128)num_i), __dmul_rn(nd, D));
  const double mx = __ddiv_rn((double)sx, nd);
  double qq = 0.0, pp = 0.0;
  for (int k = 0; k < K; k++) {
    const double t = __dsub_rn(S[(int64_t)(1 + k) * nc + j], __dmul_rn(mx, u1[k]));
    qq = __dadd_rn(qq, __dmul_rn(t, t));
    pp = __dadd_rn(pp, __dmul_rn(t, uy[k]));
  }
  const double den = __dsub_rn(ssx, qq), num = __dsub_rn(S[j], pp);
  if (!(den > 0)) {
    estim[j] = se[j] = nan_;
    return;
  }
  const double b = __ddiv_rn(num, den);
  const double rss = __dsub_rn(yres, __dmul_rn(b, num));
  estim[j] = b;
  se[j] = __dsqrt_rn(__ddiv_rn(__ddiv_rn(rss, df), den));
}

static thread_local double g_last_ms = 0;

// e = bits - exponent(max |v|) - hb (pick_e), hb as hb_bits of the matvecs
static int host_pick_e(double m, int hb, int bits) {
  int ex = 0;
  if (m > 0) {
    frexp(m, &ex);
    return bits - ex - hb;
  }
  return 0;
}

template <int NT>
static int launch_gwas(const GArgs &a, int grid, cudaStream_t s) {
  const int smem = GSTAGES * 4096 * NT;
  BSG_CUDA(cudaFuncSetAttribute(k_gwas<NT>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  k_gwas<NT><<<grid, GW * 32, smem, s>>>(a);
  return BSG_OK;
}

}  // namespace gwas
}  // namespace bsg

using namespace bsg;

extern "C" {

int bsg_univlinreg(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *U, int K,
                   const double *y, double *estim, double *std_err) {
  using namespace gwas;
  if (!h) return fail(BSG_ERR_ARG, "null handle");
  const bool dos = h->fbm_generic != 0;
  BSG_TRY(genotypes_check(h, "big_univLinReg on the device needs"));
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  if (nr < 0 || nc < 0 || K < 1) return fail(BSG_ERR_ARG, "Incompatibility between dimensions.");
  if (nr - K - 1 < 1) return fail(BSG_ERR_ARG, "Not enough rows of ind.train for %d covariate vectors.", K);
  if (!U || !y || (nc > 0 && (!estim || !std_err))) return fail(BSG_ERR_ARG, "null argument");
  const int n = h->n;
  std::vector<int> row0, col0;
  int maxmult = 1;
  BSG_TRY(host_index(ind_row, nr, n, "", row0, &maxmult));
  BSG_TRY(host_index(ind_col, nc, h->m, "", col0));
  for (int r = 0; r < nr; r++)
    if (!std::isfinite(y[r])) return fail(BSG_ERR_ARG, "'y.train' must be finite (entry %d is not).", r + 1);
  for (int64_t t = 0; t < (int64_t)nr * K; t++)
    if (!std::isfinite(U[t])) return fail(BSG_ERR_ARG, "U must be finite.");
  // host scalars, sequential sums in index order: y_c = y - mean(y); u1_k = 1'u_k; uy_k = u_k'y_c; yres = |y_c|^2 - |U'y_c|^2
  double ysum = 0.0;
  for (int r = 0; r < nr; r++) ysum += y[r];
  const double ybar = ysum / nr;
  std::vector<double> yc(nr), u1(K), uy(K);
  double yy = 0.0;
  for (int r = 0; r < nr; r++) {
    yc[r] = y[r] - ybar;
    yy += yc[r] * yc[r];
  }
  double uu1 = 0.0, uyy = 0.0;
  for (int k = 0; k < K; k++) {
    double a = 0.0, b = 0.0;
    const double *u = U + (int64_t)k * nr;
    for (int r = 0; r < nr; r++) {
      a += u[r];
      b += u[r] * yc[r];
    }
    u1[k] = a;
    uy[k] = b;
    uu1 += a * a;
    uyy += b * b;
  }
  // the statistic centres x and y, which is the regression of the contract only when the intercept lies in span(U)
  if (!(fabs(uu1 - nr) <= 1e-6 * nr))
    return fail(BSG_ERR_ARG, "U must have orthonormal columns spanning the intercept (|U'1|^2 = %g, n = %d).", uu1, nr);
  const double yres = yy - uyy, df = (double)(nr - K - 1);

  // vectors: 0 = y_c (60 bits, 8 digits), 1 + k = u_k (30 bits, 4 digits); passes of at most SMAX slices
  const int V = K + 1, hb = hb_bits(maxmult);
  std::vector<int> ebits(V), ndig(V), vpass(V), vslot(V);
  std::vector<std::vector<int>> passes;
  int used = SMAX;
  for (int v = 0; v < V; v++) {
    ndig[v] = v == 0 ? Y_DIG : U_DIG;
    const double *x = v == 0 ? yc.data() : U + (int64_t)(v - 1) * nr;
    double m = 0.0;
    for (int r = 0; r < nr; r++) m = std::max(m, fabs(x[r]));
    ebits[v] = host_pick_e(m, hb, v == 0 ? Y_BITS : U_BITS);
    if (used + ndig[v] > SMAX) {
      passes.emplace_back();
      used = 0;
    }
    vpass[v] = (int)passes.size() - 1;
    vslot[v] = used;
    passes.back().push_back(v);
    used += ndig[v];
  }
  int maxvp = 0;
  for (auto &p : passes) maxvp = std::max(maxvp, (int)p.size());
  const int nchunks = dos ? 0 : (int)(h->strideA / SEG);
  const int nlines_pad = (int)round_up(std::max(nc, 1), GLINES);
  const size_t dig_bytes = dos ? (size_t)SMAX * n : (size_t)nchunks * 4096 * NTMAX;
  const size_t need = (size_t)maxvp * n * 8 + dig_bytes + (size_t)nlines_pad * SMAX * 8 + (size_t)V * nc * 8 +
                      (size_t)nc * (3 * 8 + 2 * 8 + 4 * 4 + 4) + (size_t)n * 4 + (size_t)2 * K * 8 + 4096 + 1024;
  size_t fr = 0, tot = 0;
  BSG_CUDA(cudaMemGetInfo(&fr, &tot));
  if (need > fr)
    return fail(BSG_ERR_ALLOC, "big_univLinReg needs %.0f bytes of device memory (%d columns, %d samples, %d vectors), "
                               "%.0f are free.", (double)need, nc, n, V, (double)fr);
  g_last_ms = 0;
  if (nc == 0) return BSG_OK;

  cudaStream_t s = h->stream;
  Bufs b;
  Genotypes g;
  BSG_TRY(genotypes(h, b, &g));
  const double D = g.dosage ? g.D : 1.0;
  long long *d_Q, *d_part, *d_xs;
  uint8_t *d_dig;
  double *d_S, *d_u1, *d_uy, *d_est, *d_se;
  int *d_cols, *d_mult = nullptr;
  b.alloc(&d_Q, (size_t)maxvp * n);
  b.alloc(&d_dig, dig_bytes);
  b.alloc(&d_part, (size_t)nlines_pad * SMAX);
  b.alloc(&d_xs, (size_t)3 * nc);
  b.alloc(&d_S, (size_t)V * nc);
  b.alloc(&d_est, (size_t)nc);
  b.alloc(&d_se, (size_t)nc);
  b.up(&d_u1, u1, s);
  b.up(&d_uy, uy, s);
  b.up(&d_cols, col0.data(), (size_t)nc, s);
  if (g.dosage) {  // how many times ind.train holds each sample
    std::vector<int> mult(n, 0);
    for (int i : row0) mult[i]++;
    b.up(&d_mult, mult, s);
  }
  BSG_TRY(b.status("big_univLinReg scratch"));
  CallTimer tm;
  BSG_CUDA(cudaStreamSynchronize(s));
  if (!g.dosage) {  // sum x, sum x^2, NA count from the column counts over ind.train (multiplicities included)
    int32_t *d_cnt = nullptr;
    BSG_TRY(col_counts_dev(h, ind_row, nr, ind_col, nc, &d_cnt));
    k_gwas_xs_counts<<<(nc + 255) / 256, 256, 0, s>>>(d_cnt, nc, d_xs);
    count_launch();
  }
  // quantise and scatter onto the sample positions (integer adds: a repeated row adds its entries), vector by vector
  std::vector<long long> Qh((size_t)V * n, 0LL);
  for (int v = 0; v < V; v++) {
    const double *x = v == 0 ? yc.data() : U + (int64_t)(v - 1) * nr;
    long long *Q = Qh.data() + (size_t)v * n;
    for (int r = 0; r < nr; r++) Q[row0[r]] += llrint(ldexp(x[r], ebits[v]));
  }
  BSG_CUDA(tm.start(s));
  int nsm = 132;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->device);
  for (size_t p = 0; p < passes.size(); p++) {
    const std::vector<int> &pv = passes[p];
    SlotMap map;
    for (int t = 0; t < SMAX; t++) map.vec[t] = -1, map.dig[t] = 0;
    int S = 0;
    for (size_t a = 0; a < pv.size(); a++) {
      const int v = pv[a];
      for (int d = 0; d < ndig[v]; d++) map.vec[vslot[v] + d] = (int)a, map.dig[vslot[v] + d] = d;
      S = vslot[v] + ndig[v];
    }
    // the pass's vectors are consecutive
    BSG_CUDA(cudaMemcpyAsync(d_Q, Qh.data() + (size_t)pv[0] * n, pv.size() * n * sizeof(long long),
                             cudaMemcpyHostToDevice, s));
    BSG_CUDA(cudaMemsetAsync(d_part, 0, (size_t)nlines_pad * SMAX * sizeof(long long), s));
    if (g.dosage) {
      int8_t *dg = reinterpret_cast<int8_t *>(d_dig);
      k_gwas_digits_rows<<<(int)std::min<int64_t>(((int64_t)S * n + 255) / 256, 4096), 256, 0, s>>>(d_Q, n, S, map, dg);
      k_gwas_dos<<<nc, DT, 0, s>>>(g.raw, n, g.lut, d_cols, d_mult, dg, S, d_part, p == 0 ? d_xs : nullptr);
      count_launch(2);
    } else {
      const int NT = (S + 7) / 8;
      const int64_t units = (int64_t)nchunks * 8 * NT * 32;
      k_gwas_digits<<<(int)std::min<int64_t>((units + 255) / 256, 8192), 256, 0, s>>>(d_Q, n, nchunks, NT, map, d_dig);
      GArgs a;
      a.P = g.P;
      a.stride = g.stride;
      a.lines = d_cols;
      a.nlines = nc;
      a.nlines_pad = nlines_pad;
      a.nchunks = nchunks;
      a.dig = d_dig;
      a.part = d_part;
      const int ngroups = nlines_pad / GLINES;
      int ks = (2 * nsm + ngroups - 1) / ngroups;
      ks = std::min(ks, std::max(1, nchunks / 8));
      ks = std::max(ks, (nchunks + MAX_CHUNKS_PER_ITEM - 1) / MAX_CHUNKS_PER_ITEM);
      ks = std::max(ks, 1);
      a.chunks_per_split = (nchunks + ks - 1) / ks;
      a.ksplit = (nchunks + a.chunks_per_split - 1) / a.chunks_per_split;
      const int grid = std::min(ngroups * a.ksplit, nsm);
      int rc = BSG_OK;
      switch (NT) {
        case 1: rc = launch_gwas<1>(a, grid, s); break;
        case 2: rc = launch_gwas<2>(a, grid, s); break;
        case 3: rc = launch_gwas<3>(a, grid, s); break;
        case 4: rc = launch_gwas<4>(a, grid, s); break;
        case 5: rc = launch_gwas<5>(a, grid, s); break;
        case 6: rc = launch_gwas<6>(a, grid, s); break;
        case 7: rc = launch_gwas<7>(a, grid, s); break;
        default: rc = launch_gwas<8>(a, grid, s); break;
      }
      BSG_TRY(rc);
      count_launch(2);
    }
    for (size_t a = 0; a < pv.size(); a++) {
      const int v = pv[a];
      k_gwas_combine<<<(nc + 255) / 256, 256, 0, s>>>(d_part, nc, vslot[v], ndig[v], ebits[v], D, d_S + (int64_t)v * nc);
    }
    count_launch((int)pv.size());
    BSG_CUDA(cudaGetLastError());
  }
  k_gwas_stats<<<(nc + 255) / 256, 256, 0, s>>>(d_xs, d_S, nc, K, d_u1, d_uy, (long long)nr, D, df, yres, d_est, d_se);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(tm.stop(s));
  BSG_CUDA(cudaMemcpyAsync(estim, d_est, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaMemcpyAsync(std_err, d_se, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  g_last_ms = tm.ms();
  return BSG_OK;
}

double bsg_univlinreg_last_ms(void) { return gwas::g_last_ms; }

}  // extern "C"
