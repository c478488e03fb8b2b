// bsg_cor.cu -- windowed pairwise-complete correlations: corMat / ld_scores
// (src/corr.cpp:11-97,102-126 ; src/ld-scores.cpp:11-78,83-105), and the pair band the clumpings read (bsg_grid.cu).
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
// Integer Gram tiles (bsg_gramt.cu, bsg_gram5.cu: 128 x 128 line pairs) + per-pair fp64 epilogue.
// ---------------------------------------------------------------------------------------------------
namespace gram {

constexpr int CTN = 128;  // columns of a correlation tile

struct RowBlock {
  int first_tile;  // index of the tile holding column block jb0 (relative to the batch)
  int jb0;         // first column block
};

// fp64 epilogue per pair (j0, j0-1-k), same operation order as src/corr.cpp:77-80 / src/ld-scores.cpp:63-66; KIND is a
// BandKind.  BAND_CLUMP: the reference's scaled dot product r = sum_i x~_ij x~_ij0 with x~ = (g - c) / s, missing -> 0
// (src/clumping-bed.cpp:69-75), written from the same integer sums: r = (aa - c_j ab - c_j0 ba + c_j0 c_j bb) / (s_j0 s_j).
template <int KIND>
__global__ void k_cor_from_sums(const int *__restrict__ sums, const Tile *__restrict__ tiles,
                                const RowBlock *__restrict__ rbs, int ib0, int j0_begin, int j0_end,
                                const int *__restrict__ wlen, const long long *__restrict__ boff,
                                const int32_t *__restrict__ cnt, int nrow, int npad, const double *__restrict__ thr,
                                double *__restrict__ band, uint8_t *__restrict__ keep,
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
    const Tile tl = tiles[rb.first_tile + (j / CTN - rb.jb0)];
    const int *sp = sums + tl.out + (int64_t)(j0 - tl.i0) * CTN + (j - tl.j0);
    double xSum, xxSum, ySum, yySum, xySum;
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
      const int S = TM * CTN;
      const int aa = sp[0], bb = sp[S], ab = sp[2 * S], ba = sp[3 * S], hb = sp[4 * S], bh = sp[5 * S];
      nona = bb - npad;  // pads are valid zeros on both sides
      xSum = (double)ab;
      xxSum = (double)ab + 2.0 * (double)hb;
      ySum = (double)ba;
      yySum = (double)ba + 2.0 * (double)bh;
      xySum = (double)aa;
    }
    if (KIND == BAND_LEVELS) {
      // clumping_chr on an FBM.code256 (src/clumping.cpp:66-73): no missing-value handling in the reference -- a
      // missing genotype makes xySum NA and `r2 > thr` false; `center` / `scale` carry the caller's sumX / denoX
      const bool has_na = cnt[4 * (int64_t)j0 + 3] != 0 || cnt[4 * (int64_t)j + 3] != 0;
      const double num = xySum - center[j] * center[j0] / nrow;
      const double r2 = num * num / (scale[j] * scale[j0]);
      int l = 0;  // how many of the sorted thresholds thr[0..nlev) r2 exceeds
      if (!has_na)
        for (int t = 0; t < nlev; t++) l += r2 > thr[t];
      keep[o] = (uint8_t)l;
      continue;
    }
    if (KIND == BAND_CLUMP) {
      const double cx = center[j0], cy = center[j];
      // the numerator's roundings spelled out (the three fused steps ptxas chose), so the flags cannot change with the compiler
      const double num = __fma_rn(__dmul_rn(cx, cy), (double)nona, __fma_rn(cx, -ySum, __fma_rn(cy, -xSum, xySum)));
      const double r = num / (scale[j0] * scale[j]);
      keep[o] = (r * r > thr_r2) ? 1 : 0;
      continue;
    }
    const double num = xySum - xSum * ySum / nona;
    const double deno_x = xxSum - xSum * xSum / nona;
    const double deno_y = yySum - ySum * ySum / nona;
    if (KIND == BAND_LD) {
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

// window of j0: j = j0-1 downto 0 while pos[j] >= pos[j0] - size   (src/corr.cpp:52-53), literal scan
// `both`: also admit j when pos[j0] <= pos[j] + size -- the clumping sweep tests right-hand neighbours with that expression
// (src/clumping-utils.h:29); for non-integer positions the two roundings can differ at the window edge, so the pair
// statistics are computed for the union and the sweep applies each side's own test.
static void build_window(const double *pos, int nc, double size, bool both, PairBand &w) {
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

bool PairBand::col_blocks(int r0, int r1, int tn, int &jb0, int &jb1) const {
  int jmin = r1, jmax = -1;
  for (int j0 = r0; j0 < r1; j0++)
    if (wlen[j0] > 0) {
      jmin = std::min(jmin, j0 - wlen[j0]);
      jmax = std::max(jmax, j0 - 1);
    }
  jb0 = jmin / tn;
  jb1 = jmax / tn;
  return jmax >= jmin;
}

int pair_band(bsg_bed *h, const int *ind_row, int nr, const int *ind_col, int nc, double size, const double *pos, int kind,
              const double *thr, int nthr, const double *center, const double *scale, bool dosage_tiles, PairBand &b) {
  cudaStream_t s = h->stream;
  const int *d_row = nullptr, *d_col = nullptr;
  BSG_TRY(upload_index(h, ind_row, nr, h->n, h->w_idx_row, &d_row));
  BSG_TRY(upload_index(h, ind_col, nc, h->m, h->w_idx_col, &d_col));
  for (int j = 1; j < nc; j++)  // the reference asserts this in R (assert_sorted); the C ABI checks it too
    if (pos[j] < pos[j - 1]) return fail(BSG_ERR_ARG, "'pos' is not sorted.");
  const bool clump = kind == BAND_CLUMP || kind == BAND_LEVELS;
  build_window(pos, nc, size, clump, b);
  if (kind == BAND_CLUMP) BSG_PACKED_ONLY(h, "bed_clumping_chr");
  BSG_CUDA(b.mem.up(&b.d_wlen, b.wlen, s));
  BSG_CUDA(b.mem.up(&b.d_boff, b.boff, s));
  if (kind == BAND_COR || kind == BAND_LEVELS) BSG_CUDA(b.mem.up(&b.d_thr, thr, nthr, s));
  if (clump) {
    BSG_CUDA(b.mem.up(&b.d_center, center, nc, s));
    BSG_CUDA(b.mem.up(&b.d_scale, scale, nc, s));
  }
  if (kind == BAND_COR || kind == BAND_LD) BSG_CUDA(b.mem.alloc(&b.d_band, b.total, h->device, s));
  if (kind != BAND_LD) BSG_CUDA(b.mem.alloc(&b.d_keep, b.total, h->device, s));

  if (h->fbm_generic) {
    // FBM tables other than hard calls: fp64 sums over code256[byte] (bsg_generic.cu), or exact integer sums of the
    // D-scaled dosage bytes (bsg_grid.cu)
    if (dosage_tiles && h->dos_scale > 0)
      BSG_TRY(dosage_pair_levels(h, d_row, nr, d_col, nc, nthr, b));
    else
      BSG_TRY(generic_pairs(h, d_row, nr, d_col, nc, kind, b.d_wlen, b.d_boff, b.total, b.d_thr, nthr, b.d_band, b.d_keep,
                            b.d_center, b.d_scale, s));
    BSG_CUDA(cudaStreamSynchronize(s));
    return BSG_OK;
  }

  // hard calls on the Gram tiles.  Identity rows and columns: the staged SNP-major copy already is the dense matrix (stride
  // multiple of 128); subsets are compacted first
  auto ident = [](const int *ind, int len, int lim) {
    if (!ind) return true;
    if (len != lim) return false;
    for (int i = 0; i < len; i++)
      if (ind[i] != i + 1) return false;
    return true;
  };
  Bufs tmp;
  const uint8_t *M = h->A;
  int64_t stride = h->strideA;
  if (!(ident(ind_row, nr, h->n) && ident(ind_col, nc, h->m))) {
    stride = std::max<int64_t>(round_up(((int64_t)nr + 3) / 4, 64), 64);
    uint8_t *Mc = nullptr;
    BSG_CUDA(tmp.alloc(&Mc, (size_t)stride * nc));
    if (nc > 0) {
      int64_t work = (int64_t)nc * (stride / 4);
      int grid = (int)std::min<int64_t>((work + 255) / 256, 132 * 32);
      k_compact<<<grid, 256, 0, s>>>(h->A, h->strideA, d_row, nr, d_col, nc, Mc, stride);
      count_launch();
    }
    M = Mc;
  }
  BSG_CUDA(cudaGetLastError());
  if (nc == 0 || b.total == 0) return BSG_OK;
  using namespace gram;
  // per-line counts over the selected rows (exact) and missing-value flags
  int32_t *d_cnt = nullptr;
  uint8_t *d_na = nullptr;
  BSG_CUDA(tmp.alloc(&d_cnt, (size_t)nc * 4));
  BSG_CUDA(tmp.alloc(&d_na, (size_t)nc));
  {
    int grid = (int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 32);
    k_line_counts_ext<<<grid, 256, 0, s>>>(M, stride, nc, nr, d_cnt, d_na);
    count_launch();
  }
  std::vector<uint8_t> na(nc);
  BSG_CUDA(cudaMemcpyAsync(na.data(), d_na, (size_t)nc, cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  const int npad = (int)(stride / CHUNK) * 256 - nr;  // code-0 slots beyond the last row count as valid on both sides
  const int nib = (nc + TM - 1) / TM;
  // any-missing flag per column block: a tile touching one takes the six plane products, the others one product
  const int njb = (nc + CTN - 1) / CTN;
  std::vector<uint8_t> na_jb(njb, 0);
  for (int j = 0; j < nc; j++) na_jb[j / CTN] |= na[j];
  const auto epilogue = kind == BAND_COR     ? k_cor_from_sums<BAND_COR>
                        : kind == BAND_LD    ? k_cor_from_sums<BAND_LD>
                        : kind == BAND_CLUMP ? k_cor_from_sums<BAND_CLUMP>
                                             : k_cor_from_sums<BAND_LEVELS>;
  const double thr_r2 = kind == BAND_CLUMP ? thr[0] : 0.0;
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
      RowBlock rb{(int)tiles.size(), 0};
      int jb0, jb1;
      if (b.col_blocks(r0, r1, CTN, jb0, jb1)) {
        bool na_i = false;
        for (int q = r0 / CTN; q <= (r1 - 1) / CTN; q++) na_i |= na_jb[q] != 0;
        size_t need = 0;
        for (int jb = jb0; jb <= jb1; jb++) need += (size_t)((na_i || na_jb[jb]) ? 6 : 1) * TM * CTN;
        if (used + need > max_sum_ints && ib > ib_start) break;
        rb.jb0 = jb0;
        for (int jb = jb0; jb <= jb1; jb++) {
          const int mode = (na_i || na_jb[jb]) ? 1 : 0;
          tiles.push_back(Tile{r0, jb * CTN, mode, (long long)used});
          used += (size_t)(mode ? 6 : 1) * TM * CTN;
        }
      }
      rbs.push_back(rb);
    }
    const int j0_begin = ib_start * TM, j0_end = std::min(nc, ib * TM);
    if (tiles.empty() || b.boff[j0_end] == b.boff[j0_begin]) continue;
    Bufs batch;
    Tile *d_tiles = nullptr;
    RowBlock *d_rbs = nullptr;
    int *d_sums = nullptr;
    BSG_CUDA(batch.up(&d_tiles, tiles, s));
    BSG_CUDA(batch.up(&d_rbs, rbs, s));
    const cudaError_t e = batch.alloc(&d_sums, used, h->device, s);
    if (e != cudaSuccess) return cuda_fail(e, "correlation tile sums");
    bool any0 = false, any1 = false;
    for (const Tile &tl : tiles) (tl.mode ? any1 : any0) = true;
    // TMA-fed wgmma tiles over operands expanded once (bsg_gramt.cu); in-kernel expansion when they do not fit
    bool done = false;
    if (gramt_enabled()) BSG_TRY(gramt_cor(M, stride, nc, tiles.data(), (int)tiles.size(), d_sums, h->device, s, &done));
    if (!done) BSG_TRY(gram5_launch(M, stride, nc, stride, d_tiles, (int)tiles.size(), d_sums, any0, any1, s));
    const long long npairs = b.boff[j0_end] - b.boff[j0_begin];
    const int eg = (int)std::min<long long>((npairs + 255) / 256, 132 * 16);
    epilogue<<<eg, 256, 0, s>>>(d_sums, d_tiles, d_rbs, ib_start, j0_begin, j0_end, b.d_wlen, b.d_boff, d_cnt, nr, npad,
                                b.d_thr, b.d_band, b.d_keep, b.d_center, b.d_scale, thr_r2, nthr);
    count_launch(2);
    const cudaError_t e2 = cudaStreamSynchronize(s);
    if (e2 != cudaSuccess) return cuda_fail(e2, "correlation tiles");
  }
  BSG_CUDA(cudaGetLastError());
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
  PairBand b;
  BSG_TRY(pair_band(h, ind_row, nr, ind_col, nc, size, pos, BAND_COR, thr, nr, nullptr, nullptr, false, b));
  cudaStream_t s = h->stream;
  std::vector<int> cnt((size_t)std::max(nc, 1));
  Bufs tmp;
  int *d_cnt = nullptr;
  long long *d_p = nullptr;
  BSG_CUDA(tmp.alloc(&d_cnt, (size_t)nc));
  BSG_CUDA(tmp.alloc(&d_p, (size_t)nc + 1));
  if (nc > 0) {
    k_count_keep<<<(int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 16), 256, 0, s>>>(b.d_keep, b.d_boff, b.d_wlen, nc,
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
    cudaError_t e = tmp.alloc(&d_oi, (size_t)nnz);
    if (e == cudaSuccess) e = tmp.alloc(&d_ox, (size_t)nnz);
    if (e == cudaSuccess) e = cudaMemcpyAsync(d_p, hp.data(), (size_t)(nc + 1) * sizeof(long long), cudaMemcpyHostToDevice, s);
    if (e == cudaSuccess) {
      k_fill_csc<<<(int)std::min<int64_t>(((int64_t)nc * 32 + 255) / 256, 132 * 16), 256, 0, s>>>(
          b.d_band, b.d_keep, b.d_boff, b.d_wlen, d_p, nc, fill_diag, d_oi, d_ox);
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
  PairBand b;
  BSG_TRY(pair_band(h, ind_row, nr, ind_col, nc, size, pos, BAND_LD, nullptr, 0, nullptr, nullptr, false, b));
  if (nc == 0) return BSG_OK;
  Bufs tmp;
  int *d_reach = nullptr;
  double *d_res = nullptr;
  BSG_CUDA(tmp.up(&d_reach, b.reach, h->stream));
  BSG_CUDA(tmp.alloc(&d_res, (size_t)nc));
  k_ld_reduce<<<(nc + 127) / 128, 128, 0, h->stream>>>(b.d_band, b.d_boff, b.d_wlen, d_reach, nc, d_res);
  count_launch();
  BSG_CUDA(cudaMemcpyAsync(out, d_res, (size_t)nc * sizeof(double), cudaMemcpyDeviceToHost, h->stream));
  BSG_CUDA(cudaStreamSynchronize(h->stream));
  return BSG_OK;
}

}  // extern "C"
