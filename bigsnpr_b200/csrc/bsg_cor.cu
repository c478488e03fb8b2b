// bsg_cor.cu -- windowed pairwise-complete correlations: corMat / ld_scores
// (src/corr.cpp:11-97,102-126 ; src/ld-scores.cpp:11-78,83-105).
//
// Every sum the reference accumulates per pair (nona, xSum, xxSum, ySum, yySum, xySum) is a sum of
// small integers, i.e. a handful of population counts over bit planes of the two packed columns:
//     valid_x = ~(lo&hi), x1 = lo&~hi, x2 = hi&~lo   (staged code: 1 -> 01, 2 -> 10, NA -> 11)
//     nona = |vx & vy|, xSum = |x1&vy| + 2|x2&vy|, xxSum = |x1&vy| + 4|x2&vy|  (same for y),
//     xySum = |x1&y1| + 2|x1&y2| + 2|x2&y1| + 4|x2&y2|.
// They are exact, so the fp64 epilogue below -- written in the reference's operation order
// (src/corr.cpp:77-80) -- returns bit-identical r.  Rows / columns subsets (any multiset) are first
// compacted into a temporary packed matrix so the pair kernel always runs on dense lines.
#include <math.h>
#include <stdlib.h>

#include <algorithm>
#include <thread>

#include <vector>

#include "bsg_gram.cuh"
#include "bsg_internal.cuh"


namespace bsg {

// out line j = codes of (rows[i], cols[j]) for i < nr, packed 16 per word; pads are code 0.
__global__ void k_compact(const uint8_t *__restrict__ A, int64_t strideA, const int *__restrict__ rows, int nr,
                          const int *__restrict__ cols, int nc, uint8_t *__restrict__ out, int64_t stride_out) {
  int64_t words = stride_out / 4;
  int64_t total = (int64_t)nc * words;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    int64_t j = t / words, wq = t - j * words;
    const uint8_t *line = A + (int64_t)(cols ? cols[j] : (int)j) * strideA;
    uint32_t v = 0;
#pragma unroll 4
    for (int p = 0; p < 16; p++) {
      int64_t i = wq * 16 + p;
      if (i < nr) {
        int r = rows ? rows[i] : (int)i;
        v |= (uint32_t)((line[r >> 2] >> (2 * (r & 3))) & 3) << (2 * p);
      }
    }
    reinterpret_cast<uint32_t *>(out + j * stride_out)[wq] = v;
  }
}

// per-line counts of codes {0,1,2,3} over the first L codes (pads are code 0), one warp per line
__global__ void k_line_counts_ext(const uint8_t *__restrict__ P, int64_t stride, int nlines, int L,
                                  int32_t *__restrict__ cnt, uint8_t *__restrict__ na) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nw = (gridDim.x * blockDim.x) >> 5;
  int64_t nvec = ((int64_t)(L + 3) / 4 + 15) / 16;
  for (int l = warp; l < nlines; l += nw) {
    const uint4 *src = reinterpret_cast<const uint4 *>(P + (int64_t)l * stride);
    int c1 = 0, c2 = 0, c3 = 0;
    for (int64_t v = lane; v < nvec; v += 32) {
      uint4 q = __ldg(src + v);
      uint32_t ws[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        uint32_t lo = ws[k] & 0x55555555u, hi = (ws[k] >> 1) & 0x55555555u;
        c3 += __popc(lo & hi);
        c1 += __popc(lo & ~hi);
        c2 += __popc(hi & ~lo);
      }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      c1 += __shfl_xor_sync(0xffffffffu, c1, o);
      c2 += __shfl_xor_sync(0xffffffffu, c2, o);
      c3 += __shfl_xor_sync(0xffffffffu, c3, o);
    }
    if (lane == 0) {
      cnt[4 * (int64_t)l + 0] = L - c1 - c2 - c3;
      cnt[4 * (int64_t)l + 1] = c1;
      cnt[4 * (int64_t)l + 2] = c2;
      cnt[4 * (int64_t)l + 3] = c3;
      na[l] = c3 > 0;
    }
  }
}

// host wrappers (used by the Gram product in bsg_la.cu): out line l = codes (code_idx[k]) of source line
// line_idx[l], packed 16 per word
int compact_lines(const uint8_t *src, int64_t src_stride, const int *code_idx, int ncodes, const int *line_idx,
                  int nlines, uint8_t *out, int64_t out_stride, cudaStream_t s) {
  if (nlines == 0) return BSG_OK;
  int64_t work = (int64_t)nlines * (out_stride / 4);
  k_compact<<<(int)std::min<int64_t>((work + 255) / 256, 132 * 32), 256, 0, s>>>(src, src_stride, code_idx, ncodes, line_idx,
                                                                               nlines, out, out_stride);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int line_counts(const uint8_t *P, int64_t stride, int nlines, int L, int32_t *cnt, uint8_t *na, cudaStream_t s) {
  if (nlines == 0) return BSG_OK;
  k_line_counts_ext<<<(int)std::min<int64_t>(((int64_t)nlines * 32 + 255) / 256, 132 * 32), 256, 0, s>>>(P, stride, nlines, L,
                                                                                                       cnt, na);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

struct PairSums {
  int nona, x1v, x2v, y1v, y2v, c11, c12, c21, c22;
};

__device__ __forceinline__ void pair_accum(uint32_t a, uint32_t b, PairSums &s) {
  const uint32_t M = 0x55555555u;
  uint32_t alo = a & M, ahi = (a >> 1) & M, blo = b & M, bhi = (b >> 1) & M;
  uint32_t av = M & ~(alo & ahi), bv = M & ~(blo & bhi);
  uint32_t a1 = alo & ~ahi, a2 = ahi & ~alo, b1 = blo & ~bhi, b2 = bhi & ~blo;
  s.nona += __popc(av & bv);
  s.x1v += __popc(a1 & bv);
  s.x2v += __popc(a2 & bv);
  s.y1v += __popc(b1 & av);
  s.y2v += __popc(b2 & av);
  s.c11 += __popc(a1 & b1);
  s.c12 += __popc(a1 & b2);
  s.c21 += __popc(a2 & b1);
  s.c22 += __popc(a2 & b2);
}

// one block per column j0; warps take neighbours j = j0-1-k (k < wlen[j0]) round robin; lanes stride
// over the words of the two lines.  band[boff[j0] + k] = r (or r^2 for LD), keep[...] = threshold test.
template <bool LD>
__global__ void __launch_bounds__(256) k_cor_pairs(const uint8_t *__restrict__ M, int64_t stride, int nrow, int ncol,
                                                   const int *__restrict__ wlen, const long long *__restrict__ boff,
                                                   const double *__restrict__ thr, double *__restrict__ band,
                                                   uint8_t *__restrict__ keep) {
  const int j0 = blockIdx.x;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarp = blockDim.x >> 5;
  const int nw = wlen[j0];
  const int nvec = (int)((((int64_t)nrow + 3) / 4 + 15) / 16);
  const uint4 *la = reinterpret_cast<const uint4 *>(M + (int64_t)j0 * stride);
  for (int k = warp; k < nw; k += nwarp) {
    const int j = j0 - 1 - k;
    const uint4 *lb = reinterpret_cast<const uint4 *>(M + (int64_t)j * stride);
    PairSums s = {0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (int v = lane; v < nvec; v += 32) {
      uint4 a = __ldg(la + v), b = __ldg(lb + v);
      pair_accum(a.x, b.x, s);
      pair_accum(a.y, b.y, s);
      pair_accum(a.z, b.z, s);
      pair_accum(a.w, b.w, s);
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
      s.nona += __shfl_xor_sync(0xffffffffu, s.nona, o);
      s.x1v += __shfl_xor_sync(0xffffffffu, s.x1v, o);
      s.x2v += __shfl_xor_sync(0xffffffffu, s.x2v, o);
      s.y1v += __shfl_xor_sync(0xffffffffu, s.y1v, o);
      s.y2v += __shfl_xor_sync(0xffffffffu, s.y2v, o);
      s.c11 += __shfl_xor_sync(0xffffffffu, s.c11, o);
      s.c12 += __shfl_xor_sync(0xffffffffu, s.c12, o);
      s.c21 += __shfl_xor_sync(0xffffffffu, s.c21, o);
      s.c22 += __shfl_xor_sync(0xffffffffu, s.c22, o);
    }
    if (lane == 0) {
      // pads (code 0) count as valid zeros on both sides: remove them from nona
      const int npad = nvec * 64 - nrow;
      const int nona = s.nona - npad;
      const double xSum = (double)s.x1v + 2.0 * (double)s.x2v;
      const double xxSum = (double)s.x1v + 4.0 * (double)s.x2v;
      const double ySum = (double)s.y1v + 2.0 * (double)s.y2v;
      const double yySum = (double)s.y1v + 4.0 * (double)s.y2v;
      const double xySum = (double)s.c11 + 2.0 * (double)s.c12 + 2.0 * (double)s.c21 + 4.0 * (double)s.c22;
      // src/corr.cpp:77-80 / src/ld-scores.cpp:63-66, same operation order
      const double num = xySum - xSum * ySum / nona;
      const double deno_x = xxSum - xSum * xSum / nona;
      const double deno_y = yySum - ySum * ySum / nona;
      const long long o = boff[j0] + k;
      if (LD) {
        band[o] = num * num / (deno_x * deno_y);
      } else {
        double r = num / sqrt(deno_x * deno_y);
        bool kp = isnan(r) || fabs(r) > thr[nona > 0 ? nona - 1 : 0];
        if (r > 1) r = 1; else if (r < -1) r = -1;
        band[o] = r;
        keep[o] = kp;
      }
    }
  }
}

// res[j] = 1 + sum_k band[j][k] + sum_{j0 > j, j in window(j0)} band[j0][j0-1-j]   (NaN skipped)
__global__ void k_ld_reduce(const double *__restrict__ band, const long long *__restrict__ boff,
                            const int *__restrict__ wlen, const int *__restrict__ reach, int ncol,
                            double *__restrict__ res) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= ncol) return;
  double acc = 1.0;
  for (int k = 0; k < wlen[j]; k++) {
    double v = band[boff[j] + k];
    if (!isnan(v)) acc += v;
  }
  for (int j0 = j + 1; j0 <= reach[j]; j0++) {
    int k = j0 - 1 - j;
    if (k < wlen[j0]) {
      double v = band[boff[j0] + k];
      if (!isnan(v)) acc += v;
    }
  }
  res[j] = acc;
}


// ---------------------------------------------------------------------------------------------------
// Tensor-pipe path: integer Gram tiles (bsg_gram.cuh) + per-pair fp64 epilogue.
// ---------------------------------------------------------------------------------------------------
namespace gram {

struct Frag {
  uint4 a[4];  // A lines: (mt 0: g, g+8), (mt 1: g, g+8)
  uint4 b[4];  // B lines: nt 0..3, line g
};

__device__ __forceinline__ void frag_load(Frag &f, const uint8_t *const (&pa)[4], const uint8_t *const (&pb)[4], int64_t off) {
#pragma unroll
  for (int l = 0; l < 4; l++) f.a[l] = ldg128(pa[l] + off);
#pragma unroll
  for (int l = 0; l < 4; l++) f.b[l] = ldg128(pb[l] + off);
}

template <int PA, int PB, bool RAW>
__device__ __forceinline__ void frag_mma(const Frag &f, int (&acc)[2][4][4]) {
  const uint32_t *aw[4] = {&f.a[0].x, &f.a[1].x, &f.a[2].x, &f.a[3].x};
  const uint32_t *bw[4] = {&f.b[0].x, &f.b[1].x, &f.b[2].x, &f.b[3].x};
#pragma unroll
  for (int w = 0; w < 4; w++) {
    uint32_t wa[4], wb[4];
#pragma unroll
    for (int l = 0; l < 4; l++) {
      wa[l] = RAW ? aw[l][w] : plane_word<PA>(aw[l][w]);
      wb[l] = RAW ? bw[l][w] : plane_word<PB>(bw[l][w]);
    }
#pragma unroll
    for (int cp = 0; cp < 2; cp++) {
      const int s0 = 4 * cp, s1 = 4 * cp + 2;
      uint32_t b0[4], b1[4];
#pragma unroll
      for (int nt = 0; nt < 4; nt++) {
        b0[nt] = (wb[nt] >> s0) & 0x03030303u;
        b1[nt] = (wb[nt] >> s1) & 0x03030303u;
      }
#pragma unroll
      for (int mt = 0; mt < 2; mt++) {
        const uint32_t a0 = (wa[2 * mt] >> s0) & 0x03030303u, a1 = (wa[2 * mt + 1] >> s0) & 0x03030303u;
        const uint32_t a2 = (wa[2 * mt] >> s1) & 0x03030303u, a3 = (wa[2 * mt + 1] >> s1) & 0x03030303u;
#pragma unroll
        for (int nt = 0; nt < 4; nt++) mma_u8u8(acc[mt][nt], a0, a1, a2, a3, b0[nt], b1[nt]);
      }
    }
  }
}

// one product over the whole contraction range, double-buffered fragments
template <int PA, int PB, bool RAW>
__device__ __forceinline__ void gram_product(const uint8_t *const (&pa)[4], const uint8_t *const (&pb)[4], int nchunks,
                                             int *__restrict__ out, int row0, int col0, int g, int q) {
  int acc[2][4][4];
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++)
#pragma unroll
      for (int k = 0; k < 4; k++) acc[mt][nt][k] = 0;
  Frag f0, f1;
  frag_load(f0, pa, pb, 0);
  for (int c = 0; c < nchunks; c += 2) {
    if (c + 1 < nchunks) frag_load(f1, pa, pb, (int64_t)(c + 1) * CHUNK);
    frag_mma<PA, PB, RAW>(f0, acc);
    if (c + 2 < nchunks) frag_load(f0, pa, pb, (int64_t)(c + 2) * CHUNK);
    if (c + 1 < nchunks) frag_mma<PA, PB, RAW>(f1, acc);
  }
#pragma unroll
  for (int mt = 0; mt < 2; mt++)
#pragma unroll
    for (int nt = 0; nt < 4; nt++) {
      const int r = row0 + mt * 16 + g, cc = col0 + nt * 8 + 2 * q;
      *reinterpret_cast<int2 *>(out + (int64_t)r * TN + cc) = make_int2(acc[mt][nt][0], acc[mt][nt][1]);
      *reinterpret_cast<int2 *>(out + (int64_t)(r + 8) * TN + cc) = make_int2(acc[mt][nt][2], acc[mt][nt][3]);
    }
}

// grid = tiles; block = 8 warps (4 x 2), each warp a 32 x 32 block of line pairs over the whole k range
__global__ void __launch_bounds__(THREADS, 1) k_gram(const uint8_t *__restrict__ P, int64_t stride, int nlines,
                                                     int nchunks, const Tile *__restrict__ tiles, int *__restrict__ sums) {
  const Tile t = tiles[blockIdx.x];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int wm = warp >> 1, wn = warp & 1;
  const uint8_t *pa[4], *pb[4];
#pragma unroll
  for (int l = 0; l < 4; l++) {
    int la = t.i0 + wm * 32 + (l >> 1) * 16 + g + 8 * (l & 1);
    int lb = t.j0 + wn * 32 + l * 8 + g;
    la = min(max(la, 0), nlines - 1);
    lb = min(max(lb, 0), nlines - 1);
    pa[l] = P + (int64_t)la * stride + 16 * q;
    pb[l] = P + (int64_t)lb * stride + 16 * q;
  }
  int *out = sums + t.out;
  const int row0 = wm * 32, col0 = wn * 32;
  if (t.mode == 0) {
    gram_product<PL_A, PL_A, true>(pa, pb, nchunks, out, row0, col0, g, q);
  } else {
    // products of the pairwise-complete statistics: aa (xySum), bb (nona), ab (xSum over valid y), ba, hb, bh
    gram_product<PL_A, PL_A, false>(pa, pb, nchunks, out + 0 * TM * TN, row0, col0, g, q);
    gram_product<PL_B, PL_B, false>(pa, pb, nchunks, out + 1 * TM * TN, row0, col0, g, q);
    gram_product<PL_A, PL_B, false>(pa, pb, nchunks, out + 2 * TM * TN, row0, col0, g, q);
    gram_product<PL_B, PL_A, false>(pa, pb, nchunks, out + 3 * TM * TN, row0, col0, g, q);
    gram_product<PL_H, PL_B, false>(pa, pb, nchunks, out + 4 * TM * TN, row0, col0, g, q);
    gram_product<PL_B, PL_H, false>(pa, pb, nchunks, out + 5 * TM * TN, row0, col0, g, q);
  }
}

struct RowBlock {
  int first_tile;  // index of the tile holding column block jb0 (relative to the batch)
  int jb0;         // first column block
};

// fp64 epilogue per pair (j0, j0-1-k), same operation order as src/corr.cpp:77-80 / src/ld-scores.cpp:63-66
// KIND 0: correlation (r, keep by threshold) ; 1: LD (r^2) ; 2: clumping conflict flag: the reference's scaled dot
// product r = sum_i x~_ij x~_ij0 with x~ = (g - c) / s, missing -> 0 (src/clumping-bed.cpp:69-75), written from the
// same integer sums: r = (aa - c_j ab - c_j0 ba + c_j0 c_j bb) / (s_j0 s_j); keep = r^2 > thr.
template <int KIND>
__global__ void k_cor_from_sums(const int *__restrict__ sums, const Tile *__restrict__ tiles,
                                const RowBlock *__restrict__ rbs, int ib0, int j0_begin, int j0_end,
                                const int *__restrict__ wlen, const long long *__restrict__ boff,
                                const int32_t *__restrict__ cnt, int nrow, int npad, const double *__restrict__ thr,
                                double *__restrict__ band, uint8_t *__restrict__ keep, int tn,
                                const double *__restrict__ center, const double *__restrict__ scale, double thr_r2,
                                int nlev) {
  const long long first = boff[j0_begin], total = boff[j0_end] - first;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    // locate j0 by binary search on boff
    int lo = j0_begin, hi = j0_end - 1;
    const long long o = first + t;
    while (lo < hi) {
      int mid = (lo + hi + 1) >> 1;
      if (boff[mid] <= o) lo = mid; else hi = mid - 1;
    }
    const int j0 = lo, k = (int)(o - boff[j0]), j = j0 - 1 - k;
    const int ib = j0 / TM - ib0;
    const RowBlock rb = rbs[ib];
    const Tile tl = tiles[rb.first_tile + (j / tn - rb.jb0)];
    const int *sp = sums + tl.out + (int64_t)(j0 - tl.i0) * tn + (j - tl.j0);
    double nona_d, xSum, xxSum, ySum, yySum, xySum;
    int nona;
    if (tl.mode == 0) {
      nona = nrow;
      const int32_t *cx = cnt + 4 * (int64_t)j0, *cy = cnt + 4 * (int64_t)j;
      xSum = (double)cx[1] + 2.0 * (double)cx[2];
      xxSum = (double)cx[1] + 4.0 * (double)cx[2];
      ySum = (double)cy[1] + 2.0 * (double)cy[2];
      yySum = (double)cy[1] + 4.0 * (double)cy[2];
      xySum = (double)sp[0];
    } else {
      const int S = TM * tn;
      const int aa = sp[0], bb = sp[S], ab = sp[2 * S], ba = sp[3 * S], hb = sp[4 * S], bh = sp[5 * S];
      nona = bb - npad;  // pads are valid zeros on both sides
      xSum = (double)ab;
      xxSum = (double)ab + 2.0 * (double)hb;
      ySum = (double)ba;
      yySum = (double)ba + 2.0 * (double)bh;
      xySum = (double)aa;
    }
    (void)nona_d;
    if (KIND == 3 || KIND == 4) {
      // clumping_chr on an FBM.code256 (src/clumping.cpp:66-73): no missing-value handling in the reference -- a
      // missing genotype makes xySum NA and `r2 > thr` false; `center` / `scale` carry the caller's sumX / denoX
      const bool has_na = cnt[4 * (int64_t)j0 + 3] != 0 || cnt[4 * (int64_t)j + 3] != 0;
      const double num = xySum - center[j] * center[j0] / nrow;
      const double r2 = num * num / (scale[j] * scale[j0]);
      if (KIND == 3) {
        keep[o] = (!has_na && r2 > thr_r2) ? 1 : 0;
      } else {  // snp_grid_clumping: how many of the sorted thresholds thr[0..nlev) r2 exceeds
        int l = 0;
        if (!has_na)
          for (int t = 0; t < nlev; t++) l += r2 > thr[t];
        keep[o] = (uint8_t)l;
      }
      continue;
    }
    if (KIND == 2) {
      const double cx = center[j0], cy = center[j];
      const double r = (xySum - cy * xSum - cx * ySum + cx * cy * (double)nona) / (scale[j0] * scale[j]);
      keep[o] = (r * r > thr_r2) ? 1 : 0;
      continue;
    }
    const double num = xySum - xSum * ySum / nona;
    const double deno_x = xxSum - xSum * xSum / nona;
    const double deno_y = yySum - ySum * ySum / nona;
    if (KIND == 1) {
      band[o] = num * num / (deno_x * deno_y);
    } else {
      double r = num / sqrt(deno_x * deno_y);
      bool kp = isnan(r) || fabs(r) > thr[nona > 0 ? nona - 1 : 0];
      if (r > 1) r = 1; else if (r < -1) r = -1;
      band[o] = r;
      keep[o] = kp;
    }
  }
}

}  // namespace gram


// CSC assembly on the device: kept entries per column, then an order-preserving fill (ascending row index,
// diagonal last -- rev() of src/corr.cpp:90-92).
__global__ void k_count_keep(const uint8_t *__restrict__ keep, const long long *__restrict__ boff,
                             const int *__restrict__ wlen, int ncol, int fill_diag, int *__restrict__ cnt) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nw = (gridDim.x * blockDim.x) >> 5;
  for (int j0 = warp; j0 < ncol; j0 += nw) {
    int c = 0;
    for (int k = lane; k < wlen[j0]; k += 32) c += keep[boff[j0] + k];
#pragma unroll
    for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
    if (lane == 0) cnt[j0] = c + (fill_diag ? 1 : 0);
  }
}

__global__ void k_fill_csc(const double *__restrict__ band, const uint8_t *__restrict__ keep,
                           const long long *__restrict__ boff, const int *__restrict__ wlen,
                           const long long *__restrict__ p, int ncol, int fill_diag, int *__restrict__ oi,
                           double *__restrict__ ox) {
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  int nw = (gridDim.x * blockDim.x) >> 5;
  for (int j0 = warp; j0 < ncol; j0 += nw) {
    const int wl = wlen[j0];
    long long o = p[j0];
    for (int base = 0; base < wl; base += 32) {
      const int k = wl - 1 - (base + lane);  // descending k = ascending row index j0-1-k
      const bool kp = (k >= 0) && keep[boff[j0] + k];
      const unsigned m = __ballot_sync(0xffffffffu, kp);
      if (kp) {
        const long long pos = o + __popc(m & ((1u << lane) - 1u));
        oi[pos] = j0 - 1 - k;
        ox[pos] = band[boff[j0] + k];
      }
      o += __popc(m);
    }
    if (fill_diag && lane == 0) {
      oi[o] = j0;
      ox[o] = 1.0;
    }
  }
}

struct Window {
  std::vector<int> wlen, reach;
  std::vector<long long> boff;
  long long total = 0;
};

// window of j0: j = j0-1 downto 0 while pos[j] >= pos[j0] - size   (src/corr.cpp:52-53), literal scan
// `both`: also admit j when pos[j0] <= pos[j] + size -- the clumping sweep tests right-hand neighbours with that expression
// (src/clumping-utils.h:29); for non-integer positions the two roundings can differ at the window edge, so the pair
// statistics are computed for the union and the sweep applies each side's own test.
static void build_window(const double *pos, int nc, double size, Window &w, bool both = false) {
  w.wlen.assign(nc, 0);
  w.reach.assign(nc, 0);
  w.boff.assign(nc + 1, 0);
  for (int j = 0; j < nc; j++) w.reach[j] = j;
  // pos is sorted (checked by the caller), so both tests are monotone in j and the left edge never moves back as j0 grows:
  // a two-pointer walk returns exactly what the reference's downward scan from j0 - 1 returns, in O(nc) instead of
  // O(nc x window) host steps (1e8 for configs[2])
  int left = 0;
  for (int j0 = 0; j0 < nc; j0++) {
    const double pos_min = pos[j0] - size;
    if (left > j0) left = j0;
    while (left < j0 && !(pos[left] >= pos_min || (both && pos[j0] <= pos[left] + size))) left++;
    const int c = j0 - left;
    w.wlen[j0] = c;
    if (c > 0 && w.reach[j0 - c] < j0) w.reach[j0 - c] = j0;
  }
  // reach[j] = largest j0 whose window contains j: windows are contiguous, take a running max from the left
  for (int j = 1; j < nc; j++)
    if (w.reach[j - 1] > w.reach[j] && w.reach[j - 1] > j) w.reach[j] = std::max(w.reach[j], w.reach[j - 1]);
  long long t = 0;
  for (int j = 0; j < nc; j++) {
    w.boff[j] = t;
    t += w.wlen[j];
  }
  w.boff[nc] = t;
  w.total = t;
}

template <class T>
static int to_dev(T **dst, const std::vector<T> &v, cudaStream_t s) {
  BSG_CUDA(cudaMalloc((void **)dst, (v.size() ? v.size() : 1) * sizeof(T)));
  if (v.size()) BSG_CUDA(cudaMemcpyAsync(*dst, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, s));
  return BSG_OK;
}

struct CorScratch {
  uint8_t *M = nullptr;
  bool own_M = true;  // false: M aliases the handle's SNP-major copy (identity rows and columns)
  int *wlen = nullptr, *reach = nullptr;
  long long *boff = nullptr;
  double *thr = nullptr, *band = nullptr, *res = nullptr, *lev = nullptr;
  uint8_t *keep = nullptr;
  ~CorScratch() {
    void *p[] = {own_M ? M : nullptr, wlen, reach, boff, thr, band, res, lev, keep};
    for (void *q : p)
      if (q) cudaFree(q);
  }
};

struct ClumpParams {
  const double *center = nullptr, *scale = nullptr;  // host, per selected column (fbm: sumX / denoX)
  double thr = 0;
  bool fbm = false;  // src/clumping.cpp's statistic instead of src/clumping-bed.cpp's
  const double *levels = nullptr;  // host, nlev sorted thresholds: keep[] receives how many r2 exceeds (fbm only)
  int nlev = 0;
};

static int cor_common(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size,
                      const double *pos, const double *thr, bool ld, Window &w, CorScratch &sc,
                      const ClumpParams *clump = nullptr) {
  cudaStream_t s = h->stream;
  const int *d_row = nullptr, *d_col = nullptr;
  BSG_TRY(upload_index(h, ind_row, nr, h->n, h->w_idx_row, &d_row));
  BSG_TRY(upload_index(h, ind_col, nc, h->m, h->w_idx_col, &d_col));
  for (int j = 1; j < nc; j++)  // the reference asserts this in R (assert_sorted); the C ABI checks it too
    if (pos[j] < pos[j - 1]) return fail(BSG_ERR_ARG, "'pos' is not sorted.");
  build_window(pos, nc, size, w, clump != nullptr);
  if (h->fbm_generic) {
    // dosage FBM: the pair statistics come from fp64 sums over code256[byte] (bsg_generic.cu); thresholds, CSC assembly,
    // LD reduction and the clumping sweep downstream are the same code
    if (clump && !clump->fbm) BSG_PACKED_ONLY(h, "bed_clumping_chr");
    BSG_TRY(to_dev(&sc.wlen, w.wlen, s));
    BSG_TRY(to_dev(&sc.boff, w.boff, s));
    const size_t tot = (size_t)(w.total ? w.total : 1);
    double *d_sx = nullptr, *d_dx = nullptr;
    if (clump) {
      std::vector<double> c(clump->center, clump->center + nc), sv(clump->scale, clump->scale + nc);
      BSG_TRY(to_dev(&d_sx, c, s));
      BSG_TRY(to_dev(&d_dx, sv, s));
      sc.thr = d_sx;  // owned by the scratch (freed with it)
      sc.res = d_dx;
      BSG_CUDA(pool_alloc((void **)&sc.keep, tot, h->device, s));
      if (clump->levels) {
        BSG_TRY(to_dev(&sc.lev, std::vector<double>(clump->levels, clump->levels + clump->nlev), s));
        if (h->dos_scale > 0)  // exact integer pair sums of the D-scaled bytes (bsg_grid.cu)
          BSG_TRY(dosage_pair_levels(h, d_row, nr, d_col, nc, w.wlen, sc.wlen, sc.boff, d_sx, d_dx, sc.lev, clump->nlev,
                                     sc.keep, s));
        else
          BSG_TRY(generic_pairs(h, d_row, nr, d_col, nc, 4, sc.wlen, sc.boff, w.total, sc.lev, nullptr, sc.keep, d_sx, d_dx,
                                (double)clump->nlev, s));
        BSG_CUDA(cudaStreamSynchronize(s));
        return BSG_OK;
      }
    } else {
      BSG_CUDA(pool_alloc((void **)&sc.band, tot * sizeof(double), h->device, s));
      if (!ld) {
        std::vector<double> t(thr, thr + nr);
        if (t.empty()) t.push_back(0.0);
        BSG_TRY(to_dev(&sc.thr, t, s));
        BSG_CUDA(pool_alloc((void **)&sc.keep, tot, h->device, s));
      }
    }
    BSG_TRY(generic_pairs(h, d_row, nr, d_col, nc, clump ? 3 : (ld ? 1 : 0), sc.wlen, sc.boff, w.total, clump ? nullptr : sc.thr,
                          sc.band, sc.keep, d_sx, d_dx, clump ? clump->thr : 0.0, s));
    BSG_CUDA(cudaStreamSynchronize(s));
    return BSG_OK;
  }
  // identity rows and columns: the staged SNP-major copy already is the dense matrix (stride multiple of 128)
  auto ident = [](const int *ind, int len, int lim) {
    if (!ind) return true;
    if (len != lim) return false;
    for (int i = 0; i < len; i++)
      if (ind[i] != i + 1) return false;
    return true;
  };
  const bool direct = ident(ind_row, nr, h->n) && ident(ind_col, nc, h->m);
  int64_t stride = round_up(((int64_t)nr + 3) / 4, 64);
  if (stride < 64) stride = 64;
  if (direct) {
    sc.M = h->A;
    sc.own_M = false;
    stride = h->strideA;
  } else {
    BSG_CUDA(cudaMalloc((void **)&sc.M, (size_t)stride * (nc > 0 ? nc : 1)));
    if (nc > 0) {
      int64_t work = (int64_t)nc * (stride / 4);
      int grid = (int)std::min<int64_t>((work + 255) / 256, 132 * 32);
      k_compact<<<grid, 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, sc.M, stride);
      count_launch();
    }
  }
  BSG_TRY(to_dev(&sc.wlen, w.wlen, s));
  BSG_TRY(to_dev(&sc.boff, w.boff, s));
  double *d_cc = nullptr, *d_cs = nullptr;
  if (clump) {
    std::vector<double> c(clump->center, clump->center + nc), sv(clump->scale, clump->scale + nc);
    BSG_TRY(to_dev(&d_cc, c, s));
    BSG_TRY(to_dev(&d_cs, sv, s));
    sc.thr = d_cc;   // owned by the scratch (freed with it)
    sc.res = d_cs;
    if (clump->levels) BSG_TRY(to_dev(&sc.lev, std::vector<double>(clump->levels, clump->levels + clump->nlev), s));
    BSG_CUDA(pool_alloc((void **)&sc.keep, (size_t)(w.total ? w.total : 1), h->device, s));
  } else {
    BSG_CUDA(pool_alloc((void **)&sc.band, (size_t)(w.total ? w.total : 1) * sizeof(double), h->device, s));
    if (!ld) {
      std::vector<double> t(thr, thr + nr);
      if (t.empty()) t.push_back(0.0);
      BSG_TRY(to_dev(&sc.thr, t, s));
      BSG_CUDA(pool_alloc((void **)&sc.keep, (size_t)(w.total ? w.total : 1), h->device, s));
    }
  }
  static int use_popc = -1;
  if (use_popc < 0) {
    const char *ev = getenv("BSG_COR_POPC");
    use_popc = (ev && ev[0] == '1') ? 1 : 0;
  }
  if (nc > 0 && use_popc && !clump) {
    if (ld)
      k_cor_pairs<true><<<nc, 256, 0, s>>>(sc.M, stride, nr, nc, sc.wlen, sc.boff, nullptr, sc.band, nullptr);
    else
      k_cor_pairs<false><<<nc, 256, 0, s>>>(sc.M, stride, nr, nc, sc.wlen, sc.boff, sc.thr, sc.band, sc.keep);
    count_launch();
  } else if (nc > 0 && w.total > 0) {
    using namespace gram;
    // per-line counts over the selected rows (exact) and missing-value flags
    int32_t *d_cnt = nullptr;
    uint8_t *d_na = nullptr;
    BSG_CUDA(cudaMalloc((void **)&d_cnt, (size_t)nc * 4 * sizeof(int32_t)));
    BSG_CUDA(cudaMalloc((void **)&d_na, (size_t)nc));
    struct Guard {
      void *a, *b, *c, *d, *e;
      ~Guard() {
        void *p[] = {a, b, c, d, e};
        for (void *q : p)
          if (q) cudaFree(q);
      }
    } gd{d_cnt, d_na, nullptr, nullptr, nullptr};
    {
      int grid = (int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 32);
      k_line_counts_ext<<<grid, 256, 0, s>>>(sc.M, stride, nc, nr, d_cnt, d_na);
      count_launch();
    }
    std::vector<uint8_t> na(nc);
    BSG_CUDA(cudaMemcpyAsync(na.data(), d_na, (size_t)nc, cudaMemcpyDeviceToHost, s));
    BSG_CUDA(cudaStreamSynchronize(s));
    const int nchunks = (int)(stride / CHUNK);
    const int npad = nchunks * 256 - nr;  // code-0 slots beyond the last row count as valid on both sides
    const int nib = (nc + TM - 1) / TM;
    // no missing value at all -> 128 x 128 wgmma tiles (bsg_gram5.cu); else 128 x 64 six-plane IMMA tiles
    bool clean = true;
    for (int j = 0; j < nc && clean; j++) clean = na[j] == 0;
    static int use_g5 = -1;
    if (use_g5 < 0) {
      const char *ev = getenv("BSG_GRAM5");
      use_g5 = (ev && ev[0] == '0') ? 0 : 1;
    }
    const bool g5 = use_g5 != 0;  // wgmma tiles (128 x 128): missing-free tiles one product, the others six planes
    (void)clean;
    const int TNv = g5 ? 128 : TN;
    // any-missing flag per column block
    const int njb = (nc + TNv - 1) / TNv;
    std::vector<uint8_t> na_jb(njb, 0);
    for (int j = 0; j < nc; j++) na_jb[j / TNv] |= na[j];
    // tiles, in batches of row blocks bounded by the size of the sums buffer
    const size_t max_sum_ints = (size_t)768 << 20;  // 3 GB of int32
    int ib = 0;
    while (ib < nib) {
      std::vector<Tile> tiles;
      std::vector<RowBlock> rbs;
      size_t used = 0;
      const int ib_start = ib;
      for (; ib < nib; ib++) {
        const int r0 = ib * TM, r1 = std::min(nc, r0 + TM);
        int jmin = r1, jmax = -1;
        for (int j0 = r0; j0 < r1; j0++)
          if (w.wlen[j0] > 0) {
            jmin = std::min(jmin, j0 - w.wlen[j0]);
            jmax = std::max(jmax, j0 - 1);
          }
        RowBlock rb{(int)tiles.size(), 0};
        if (jmax >= jmin) {
          const int jb0 = jmin / TNv, jb1 = jmax / TNv;
          bool na_i = false;
          for (int b = r0 / TNv; b <= (r1 - 1) / TNv; b++) na_i |= na_jb[b] != 0;
          size_t need = 0;
          for (int jb = jb0; jb <= jb1; jb++) need += (size_t)((na_i || na_jb[jb]) ? 6 : 1) * TM * TNv;
          if (used + need > max_sum_ints && ib > ib_start) break;
          rb.jb0 = jb0;
          for (int jb = jb0; jb <= jb1; jb++) {
            const int mode = (na_i || na_jb[jb]) ? 1 : 0;
            tiles.push_back(Tile{r0, jb * TNv, mode, (long long)used});
            used += (size_t)(mode ? 6 : 1) * TM * TNv;
          }
        }
        rbs.push_back(rb);
      }
      const int j0_begin = ib_start * TM, j0_end = std::min(nc, ib * TM);
      if (tiles.empty() || w.boff[j0_end] == w.boff[j0_begin]) continue;
      Tile *d_tiles = nullptr;
      RowBlock *d_rbs = nullptr;
      int *d_sums = nullptr;
      BSG_CUDA(cudaMalloc((void **)&d_tiles, tiles.size() * sizeof(Tile)));
      BSG_CUDA(cudaMalloc((void **)&d_rbs, rbs.size() * sizeof(RowBlock)));
      cudaError_t e = pool_alloc((void **)&d_sums, used * sizeof(int), h->device, s);
      if (e != cudaSuccess) {
        cudaFree(d_tiles);
        cudaFree(d_rbs);
        return cuda_fail(e, "correlation tile sums");
      }
      cudaMemcpyAsync(d_tiles, tiles.data(), tiles.size() * sizeof(Tile), cudaMemcpyHostToDevice, s);
      cudaMemcpyAsync(d_rbs, rbs.data(), rbs.size() * sizeof(RowBlock), cudaMemcpyHostToDevice, s);
      if (g5) {
        bool any0 = false, any1 = false;
        for (const Tile &tl : tiles) (tl.mode ? any1 : any0) = true;
        // TMA-fed wgmma tiles over operands expanded once (bsg_gramt.cu); in-kernel expansion when they do not fit
        bool done = false;
        int rc5 = gramt_enabled() ? gramt_cor(sc.M, stride, nc, tiles.data(), (int)tiles.size(), d_sums, h->device, s, &done) : BSG_OK;
        if (!rc5 && !done) rc5 = gram5_launch(sc.M, stride, nc, stride, d_tiles, (int)tiles.size(), d_sums, any0, any1, s);
        if (rc5) {
          cudaFree(d_tiles);
          cudaFree(d_rbs);
          cudaFree(d_sums);
          return rc5;
        }
      } else {
        k_gram<<<(unsigned)tiles.size(), THREADS, 0, s>>>(sc.M, stride, nc, nchunks, d_tiles, d_sums);
      }
      const long long npairs = w.boff[j0_end] - w.boff[j0_begin];
      const int eg = (int)std::min<long long>((npairs + 255) / 256, 132 * 16);
      if (clump && clump->levels)
        k_cor_from_sums<4><<<eg, 256, 0, s>>>(d_sums, d_tiles, d_rbs, ib_start, j0_begin, j0_end, sc.wlen, sc.boff, d_cnt, nr,
                                              npad, sc.lev, nullptr, sc.keep, TNv, d_cc, d_cs, 0.0, clump->nlev);
      else if (clump && clump->fbm)
        k_cor_from_sums<3><<<eg, 256, 0, s>>>(d_sums, d_tiles, d_rbs, ib_start, j0_begin, j0_end, sc.wlen, sc.boff, d_cnt, nr,
                                              npad, nullptr, nullptr, sc.keep, TNv, d_cc, d_cs, clump->thr, 0);
      else if (clump)
        k_cor_from_sums<2><<<eg, 256, 0, s>>>(d_sums, d_tiles, d_rbs, ib_start, j0_begin, j0_end, sc.wlen, sc.boff, d_cnt, nr,
                                              npad, nullptr, nullptr, sc.keep, TNv, d_cc, d_cs, clump->thr, 0);
      else if (ld)
        k_cor_from_sums<1><<<eg, 256, 0, s>>>(d_sums, d_tiles, d_rbs, ib_start, j0_begin, j0_end, sc.wlen, sc.boff, d_cnt, nr,
                                              npad, nullptr, sc.band, nullptr, TNv, nullptr, nullptr, 0.0, 0);
      else
        k_cor_from_sums<0><<<eg, 256, 0, s>>>(d_sums, d_tiles, d_rbs, ib_start, j0_begin, j0_end, sc.wlen, sc.boff, d_cnt, nr,
                                              npad, sc.thr, sc.band, sc.keep, TNv, nullptr, nullptr, 0.0, 0);
      count_launch(2);
      cudaError_t e2 = cudaStreamSynchronize(s);
      cudaFree(d_tiles);
      cudaFree(d_rbs);
      cudaFree(d_sums);
      if (e2 != cudaSuccess) return cuda_fail(e2, "correlation tiles");
    }
  }
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

LevelBand::~LevelBand() {
  void *p[] = {d_wlen, d_boff, d_lev};
  for (void *q : p)
    if (q) cudaFree(q);
}

int level_band(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size, const double *pos,
               const double *sumX, const double *denoX, const double *levels, int nlev, LevelBand &b) {
  Window w;
  CorScratch sc;
  ClumpParams cp;
  cp.center = sumX;
  cp.scale = denoX;
  cp.fbm = true;
  cp.levels = levels;
  cp.nlev = nlev;
  BSG_TRY(cor_common(h, ind_row, nr, ind_col, nc, size, pos, nullptr, false, w, sc, &cp));
  BSG_CUDA(cudaStreamSynchronize(h->stream));
  b.wlen.swap(w.wlen);
  b.boff.swap(w.boff);
  b.total = w.total;
  std::swap(b.d_wlen, sc.wlen);  // the band and its offsets outlive the scratch
  std::swap(b.d_boff, sc.boff);
  std::swap(b.d_lev, sc.keep);
  return BSG_OK;
}

}  // namespace bsg

using namespace bsg;

extern "C" {

int bsg_cor(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size, const double *thr,
            const double *pos, int fill_diag, int64_t *p, int **pi, double **px) {
  if (!h || !thr || !pos || !p || !pi || !px) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  *pi = nullptr;
  *px = nullptr;
  Window w;
  CorScratch sc;
  BSG_TRY(cor_common(h, ind_row, nr, ind_col, nc, size, pos, thr, false, w, sc));
  cudaStream_t s = h->stream;
  std::vector<int> cnt((size_t)std::max(nc, 1));
  int *d_cnt = nullptr;
  long long *d_p = nullptr;
  BSG_CUDA(cudaMalloc((void **)&d_cnt, (size_t)std::max(nc, 1) * sizeof(int)));
  BSG_CUDA(cudaMalloc((void **)&d_p, (size_t)(nc + 1) * sizeof(long long)));
  struct G2 {
    void *a, *b, *c, *d;
    ~G2() {
      void *q[] = {a, b, c, d};
      for (void *x : q)
        if (x) cudaFree(x);
    }
  } g2{d_cnt, d_p, nullptr, nullptr};
  if (nc > 0) {
    k_count_keep<<<(int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 16), 256, 0, s>>>(sc.keep, sc.boff, sc.wlen, nc,
                                                                                               fill_diag, d_cnt);
    count_launch();
  }
  BSG_CUDA(cudaMemcpyAsync(cnt.data(), d_cnt, (size_t)nc * sizeof(int), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  long long nnz = 0;
  std::vector<long long> hp((size_t)nc + 1);
  for (int j0 = 0; j0 < nc; j0++) {
    hp[j0] = nnz;
    p[j0] = nnz;
    nnz += cnt[j0];
  }
  hp[nc] = nnz;
  p[nc] = nnz;
  int *oi = (int *)malloc((size_t)(nnz ? nnz : 1) * sizeof(int));
  double *ox = (double *)malloc((size_t)(nnz ? nnz : 1) * sizeof(double));
  if (!oi || !ox) {
    free(oi);
    free(ox);
    return fail(BSG_ERR_ALLOC, "cannot allocate the correlation triplets");
  }
  if (nnz > 0) {
    int *d_oi = nullptr;
    double *d_ox = nullptr;
    cudaError_t e = cudaMalloc((void **)&d_oi, (size_t)nnz * sizeof(int));
    g2.c = d_oi;
    if (e == cudaSuccess) e = cudaMalloc((void **)&d_ox, (size_t)nnz * sizeof(double));
    g2.d = d_ox;
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_p, hp.data(), (size_t)(nc + 1) * sizeof(long long), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
      k_fill_csc<<<(int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 16), 256, 0, s>>>(
          sc.band, sc.keep, sc.boff, sc.wlen, d_p, nc, fill_diag, d_oi, d_ox);
      count_launch();
      // The result arrays are fresh malloc memory (configs[2]: 1.2 GB): first touch by one thread runs at ~1.5 GB/s and
      // used to dominate the call.  Touch the pages from several threads while the device assembles the CSC arrays.
      prefault_pages(oi, (size_t)nnz * sizeof(int));
      prefault_pages(ox, (size_t)nnz * sizeof(double));
      e = cudaMemcpyAsync(oi, d_oi, (size_t)nnz * sizeof(int), cudaMemcpyDeviceToHost, s);
    }
    if (e == cudaSuccess) e = cudaMemcpyAsync(ox, d_ox, (size_t)nnz * sizeof(double), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) {
      free(oi);
      free(ox);
      return cuda_fail(e, "correlation CSC assembly");
    }
  }
  *pi = oi;
  *px = ox;
  return BSG_OK;
}

int bsg_ld_scores(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size, const double *pos,
                  double *out) {
  if (!h || !pos || !out) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  Window w;
  CorScratch sc;
  BSG_TRY(cor_common(h, ind_row, nr, ind_col, nc, size, pos, nullptr, true, w, sc));
  if (nc == 0) return BSG_OK;
  BSG_TRY(to_dev(&sc.reach, w.reach, h->stream));
  BSG_CUDA(cudaMalloc((void **)&sc.res, (size_t)nc * sizeof(double)));
  k_ld_reduce<<<(nc + 127) / 128, 128, 0, h->stream>>>(sc.band, sc.boff, sc.wlen, sc.reach, nc, sc.res);
  count_launch();
  BSG_CUDA(cudaMemcpyAsync(out, sc.res, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  BSG_CUDA(cudaStreamSynchronize(h->stream));
  return BSG_OK;
}

}  // extern "C"

// One round of the greedy clumping pass, all undecided variants in parallel (one warp each).  The sequential pass
// (src/clumping-bed.cpp:37-88) visits the variants by decreasing priority and keeps j0 unless an ALREADY KEPT variant of
// its window is correlated with it above the threshold.  Only higher-priority neighbours matter, so j0's fate is known as
// soon as theirs is:  REMOVED if one of its conflicting higher-priority neighbours is KEPT, KEPT if all of them are REMOVED
// (or there is none), otherwise undecided for this round.  By induction on the rank this gives the sequential result; the
// highest-ranked undecided variant is decided in every round, dense LD blocks resolve in two or three rounds.
// Neighbour ranges follow which_to_check (src/clumping-utils.h:12-43) literally: left while pos[j] >= pos[j0] - size, right
// while pos[j] <= pos[j0] + size, each scan stopping at the first failure like the `break` of the sequential loops.
__global__ void k_clump_round(const uint8_t *__restrict__ conflict, const long long *__restrict__ boff, const int *__restrict__ wlen,
                              const double *__restrict__ pos, const int *__restrict__ rank, double size, int nc, int *state,
                              int *n_undecided) {
  const int lane = threadIdx.x & 31;
  const int64_t warp = (blockIdx.x * (int64_t)blockDim.x + threadIdx.x) >> 5, nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t j0l = warp; j0l < nc; j0l += nw) {
    const int j0 = (int)j0l;
    if (state[j0] != -1) continue;  // warp-uniform
    const int k = rank[j0];
    const double pos_min = pos[j0] - size, pos_max = pos[j0] + size;
    int kept = 0, undec = 0;
    const int wl = wlen[j0];
    const long long b0 = boff[j0];
    for (int t0 = 0; t0 < wl; t0 += 32) {  // left neighbours: the pairs of j0's own window
      const int t = t0 + lane;
      bool ok = t < wl;
      int j = j0 - 1 - t;
      if (ok) ok = pos[j] >= pos_min;
      const unsigned stop = __ballot_sync(0xffffffffu, !ok);
      const bool live = stop ? lane < __ffs(stop) - 1 : true;
      if (live && conflict[b0 + t] && rank[j] < k) {
        const int st = state[j];
        kept |= st == 1;
        undec |= st == -1;
      }
      if (stop) break;
    }
    for (int j1 = j0 + 1; j1 < nc; j1 += 32) {  // right neighbours: j0 sits in the window of j
      const int j = j1 + lane, t = j - 1 - j0;
      bool ok = j < nc;
      if (ok) ok = pos[j] <= pos_max && t < wlen[j];
      const unsigned stop = __ballot_sync(0xffffffffu, !ok);
      const bool live = stop ? lane < __ffs(stop) - 1 : true;
      if (live && conflict[boff[j] + t] && rank[j] < k) {
        const int st = state[j];
        kept |= st == 1;
        undec |= st == -1;
      }
      if (stop) break;
    }
    kept = __any_sync(0xffffffffu, kept);
    undec = __any_sync(0xffffffffu, undec);
    if (lane == 0) {
      if (kept)
        state[j0] = 0;
      else if (!undec)
        state[j0] = 1;
      else
        atomicAdd(n_undecided, 1);
    }
  }
}

extern "C" {

// bed_clumping_chr: src/clumping-bed.cpp:11-91 (+ which_to_check, src/clumping-utils.h:12-43).
// ordInd: 1-based column positions by decreasing priority (R: order(S, decreasing = TRUE)); keep[nc] receives 0 / 1.
// All pair statistics inside the window come from the Gram tiles; the greedy pass is resolved on the device in rounds
// (k_clump_round; BSG_CLUMP_HOST=1: the literal sequential pass on the host over the downloaded flags).
static int clumping_common(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *a1,
                           const double *a2, const int *ordInd, const double *pos, double size, double thr, int *keep,
                           bool fbm) {
  if (!h || !a1 || !a2 || !ordInd || !pos || !keep) return fail(BSG_ERR_ARG, "null argument");
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (!ind_col) nc = h->m;
  Window w;
  CorScratch sc;
  ClumpParams cp;
  cp.center = a1;
  cp.scale = a2;
  cp.thr = thr;
  cp.fbm = fbm;
  BSG_TRY(cor_common(h, ind_row, nr, ind_col, nc, size, pos, nullptr, false, w, sc, &cp));
  static int host_sweep = -1;
  if (host_sweep < 0) {
    const char *ev = getenv("BSG_CLUMP_HOST");
    host_sweep = (ev && ev[0] == '1') ? 1 : 0;
  }
  if (!host_sweep) {
    std::vector<int> rank(nc);
    for (int k = 0; k < nc; k++) {
      int j = ordInd[k] - 1;
      if (j < 0 || j >= nc) return fail(BSG_ERR_BOUNDS, "Tested subscript out of bounds (ordInd).");
      rank[j] = k;
    }
    if (nc == 0) return BSG_OK;
    cudaStream_t s = h->stream;
    int *d_rank = nullptr, *d_state = nullptr, *d_cnt = nullptr;
    double *d_pos = nullptr;
    struct G {
      void *p[4];
      ~G() {
        for (void *q : p)
          if (q) cudaFree(q);
      }
    } guard{{nullptr, nullptr, nullptr, nullptr}};
    BSG_CUDA(pool_alloc((void **)&d_rank, (size_t)nc * sizeof(int), h->device, s));
    guard.p[0] = d_rank;
    BSG_CUDA(pool_alloc((void **)&d_state, (size_t)nc * sizeof(int), h->device, s));
    guard.p[1] = d_state;
    BSG_CUDA(pool_alloc((void **)&d_pos, (size_t)nc * sizeof(double), h->device, s));
    guard.p[2] = d_pos;
    BSG_CUDA(pool_alloc((void **)&d_cnt, 64 * sizeof(int), h->device, s));
    guard.p[3] = d_cnt;
    BSG_CUDA(cudaMemcpyAsync(d_rank, rank.data(), (size_t)nc * sizeof(int), cudaMemcpyHostToDevice, s));
    BSG_CUDA(cudaMemcpyAsync(d_pos, pos, (size_t)nc * sizeof(double), cudaMemcpyHostToDevice, s));
    BSG_CUDA(cudaMemsetAsync(d_state, 0xFF, (size_t)nc * sizeof(int), s));  // -1: undecided
    const int grid = (int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 16);
    const int BATCH = 4;  // rounds per host round trip
    int left[BATCH];
    for (int64_t round = 0; round < (int64_t)nc + BATCH; round += BATCH) {
      BSG_CUDA(cudaMemsetAsync(d_cnt, 0, BATCH * sizeof(int), s));
      for (int b = 0; b < BATCH; b++)
        k_clump_round<<<grid, 256, 0, s>>>(sc.keep, sc.boff, sc.wlen, d_pos, d_rank, size, nc, d_state, d_cnt + b);
      count_launch(BATCH);
      BSG_CUDA(cudaMemcpyAsync(left, d_cnt, BATCH * sizeof(int), cudaMemcpyDeviceToHost, s));
      BSG_CUDA(cudaStreamSynchronize(s));
      if (left[BATCH - 1] == 0) break;
    }
    BSG_CUDA(cudaMemcpyAsync(keep, d_state, (size_t)nc * sizeof(int), cudaMemcpyDeviceToHost, s));
    BSG_CUDA(cudaStreamSynchronize(s));
    for (int j = 0; j < nc; j++)
      if (keep[j] != 0 && keep[j] != 1) return fail(BSG_ERR_CUDA, "clumping rounds did not converge.");
    return BSG_OK;
  }
  std::vector<uint8_t> conflict((size_t)w.total);
  if (w.total)
    BSG_CUDA(cudaMemcpyAsync(conflict.data(), sc.keep, (size_t)w.total, cudaMemcpyDeviceToHost, h->stream));
  BSG_CUDA(cudaStreamSynchronize(h->stream));
  std::vector<int> rank(nc);
  for (int k = 0; k < nc; k++) {
    int j = ordInd[k] - 1;
    if (j < 0 || j >= nc) return fail(BSG_ERR_BOUNDS, "Tested subscript out of bounds (ordInd).");
    rank[j] = k;
  }
  for (int j = 0; j < nc; j++) keep[j] = -1;
  for (int k = 0; k < nc; k++) {
    const int j0 = ordInd[k] - 1;
    int keep_j0 = 1;
    // left neighbours: pairs (j0, j) of j0's own window; right neighbours: j0 is in the window of j
    // which_to_check (src/clumping-utils.h:12-43): left while pos[j] >= pos[j0] - size, right while pos[j] <= pos[j0] + size
    const double pos_min = pos[j0] - size, pos_max = pos[j0] + size;
    for (int t = 0; t < w.wlen[j0] && keep_j0; t++) {
      const int j = j0 - 1 - t;
      if (!(pos[j] >= pos_min)) break;
      if (rank[j] < k && keep[j] == 1 && conflict[(size_t)(w.boff[j0] + t)]) keep_j0 = 0;
    }
    for (int j = j0 + 1; j < nc && keep_j0; j++) {
      const int t = j - 1 - j0;
      if (!(pos[j] <= pos_max) || t >= w.wlen[j]) break;  // the union window of j holds every pair either test admits
      if (rank[j] < k && keep[j] == 1 && conflict[(size_t)(w.boff[j] + t)]) keep_j0 = 0;
    }
    keep[j0] = keep_j0;
  }
  return BSG_OK;
}

int bsg_clumping_chr(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *center,
                     const double *scale, const int *ordInd, const double *pos, double size, double thr, int *keep) {
  return clumping_common(h, ind_row, nr, ind_col, nc, center, scale, ordInd, pos, size, thr, keep, false);
}

int bsg_clumping_chr_fbm(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, const double *sumX,
                         const double *denoX, const int *ordInd, const double *pos, double size, double thr,
                         int *keep) {
  return clumping_common(h, ind_row, nr, ind_col, nc, sumX, denoX, ordInd, pos, size, thr, keep, true);
}

}  // extern "C"
