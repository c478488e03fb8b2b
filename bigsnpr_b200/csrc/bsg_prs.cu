// bsg_prs.cu -- C+T scores: snp_PRS with thresholding (R/PRS.R:36-76) for every keep set of one chromosome of
// snp_grid_PRS (R/SCT.R:201-246) in one launch over the SNP-major 2-bit copy.
//
// A keep set's entries are assigned to steps: step k holds the entries whose lpS first exceeds the k-th largest
// threshold (strict >, thresholds in stable decreasing order).  Each set's lines are ordered by step, entries in their
// original order within a step, and every step is padded to a multiple of 32 lines with copies of one of its own lines
// carrying zero digits.  The weights v = (2 same - 1) beta of a set are quantised once (k_prep1 / k_quantT, 61-bit fixed
// point, 8 signed base-256 digits, hb = 0: every entry is its own line), so score(step k) = sum over the lines of steps
// <= k of code x Q plus the reversed-allele constant sum -2 Q over the reversed entries so far, exact per digit slice.
//
// k_prs: one CTA per (set, 512-sample-byte block), eight warps of 64 sample-bytes, the transpose-and-mask fragments and
// per-warp cp.async pipeline of k_pmvT_lines.  The int32 accumulators are cumulative across steps: at each step end
// the warp emits that threshold's column (slice totals + constant, one top-down fp64 sum over the 8 slices with no
// contraction) for its 256 samples.  A set longer than CAP_GROUPS groups drains its accumulators into int64 totals in
// global memory first (int32 head-room: |code 4^c digit| <= 3 x 64 x 128 per line).  A sample whose codes so far hold
// an NA code (3) is NaN from that step on (R: last + NA stays NA); the kernel flags it from the fragments it already
// holds, so the rule needs no second pass and no missing-value list, at any NA rate.
// Dosage tables (CODE_DOSAGE, D > 0) run k_prs_dos instead: the same digits, steps and emits over the raw code bytes, the
// value bytes D x code in int32 slice sums, and one division by D per output.
#include <algorithm>
#include <atomic>
#include <math.h>
#include <numeric>
#include <stdio.h>
#include <string.h>
#include <vector>

#include "bsg_internal.cuh"
#include "bsg_pmv_shared.cuh"

namespace bsg {
namespace prs {
using namespace pmv;

constexpr int TL = 32, TB = 512, WARPS = 8, STG = 6;
constexpr int WSTAGE = TL * 64;                               // one warp's strip of a step: 32 lines x 64 B
constexpr int STAGE_SMEM = WARPS * STG * WSTAGE;              // 96 KB
constexpr int SMEM = STAGE_SMEM + WARPS * 256 * 8;            // + 256 emitted doubles per warp: 112 KB, 2 CTAs per SM
constexpr int CAP_GROUPS = (1 << 16) / TL;                    // 2^16 lines x 3 x 64 x 128 < 2^31
constexpr int PAD = 2;                                        // kind[] of a padding line (0: same, 1: reversed)

struct Args {
  const uint8_t *P;
  int64_t stride;
  int n, nblocks, nthr;
  const int *lines;         // physical line of every padded line, sets concatenated
  const int *grp_off;       // [nsets + 1] first 32-line group of each set
  const int *step_end;      // [nsets][nthr] groups of the set through step k
  const int *col_of;        // [nthr] output column (the caller's threshold order) of step k
  const uint8_t *dig;       // [groups][8][32]
  const long long *kc;      // [nsets][nthr][8] reversed-allele constant added by step k, per slice
  const Scal *sc;           // [nsets]
  const int *long_slot;     // [nsets] slot in `base` of a set longer than CAP_GROUPS groups, else -1
  long long *base;          // [slots][nblocks][64][256] drained totals
  double *S;                // [nsets * nthr][n]
};

__device__ __forceinline__ void cp_async16(uint32_t dst, const void *src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}

template <bool NA>
__global__ void __launch_bounds__(WARPS * 32, 2) k_prs(const Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
  const int set = blockIdx.x / a.nblocks, blk = blockIdx.x % a.nblocks;
  const int g0 = a.grp_off[set], ngrp = a.grp_off[set + 1] - g0;
  const int64_t byte0 = (int64_t)blk * TB + 64 * warp;  // this warp's 64 sample-bytes of every line
  const uint32_t wbase = smem_u32(smem) + warp * (STG * WSTAGE);
  double *ebuf = reinterpret_cast<double *>(smem + STAGE_SMEM) + warp * 256;

  // loader role of the lane and stage layout: as k_pmvT_lines (bsg_pmv.cu)
  const int lrow = lane >> 2, lch = lane & 3;
  const int64_t colb = (byte0 + 16 * lch < a.stride) ? byte0 + 16 * lch : 0;
  uint32_t dst_off[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int row = 8 * i + lrow;
    const int hf = row >> 4, qq = (row >> 2) & 3, r = row & 3, sl = lch >> 1, hc = lch & 1;
    dst_off[i] = (uint32_t)((((((r * 2 + hf) * 2 + sl) * 4 + qq) * 8) + 4 * hc) * 4);
  }
  auto issue = [&](int step, int stage) {
    const uint32_t dst = wbase + stage * WSTAGE;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const int phys = a.lines[(int64_t)(g0 + step) * TL + 8 * i + lrow];
      cp_async16(dst + dst_off[i], a.P + colb + (int64_t)phys * a.stride);
    }
  };

  int acc[4][4][4];
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int c = 0; c < 4; c++)
#pragma unroll
      for (int k = 0; k < 4; k++) acc[j][c][k] = 0;
  uint32_t naw[2][4];  // [slot g / g + 8][byte]: OR of code & (code >> 1) over the lines so far
#pragma unroll
  for (int sl = 0; sl < 2; sl++)
#pragma unroll
    for (int j = 0; j < 4; j++) naw[sl][j] = 0;

  const int *send = a.step_end + (int64_t)set * a.nthr;
  const long long *kc = a.kc + (int64_t)set * a.nthr * 8;
  const int e = a.sc[set].e[0];
  const int slot = a.long_slot[set];
  long long *base = slot >= 0 ? a.base + ((int64_t)slot * a.nblocks + blk) * 64 * 256 : nullptr;
  bool drained = false;
  long long kr0 = 0, kr1 = 0;  // reversed-allele constant so far, slices 2q and 2q + 1
  int k = 0;

  // the column of step k for the warp's 256 samples: lanes q = 3 .. 0 hold slices (7, 6) .. (1, 0) of a sample, so the
  // top-down sum runs along the quad, and lane q = 0 stores the result
  auto emit = [&]() {
    kr0 += kc[k * 8 + 2 * q];
    kr1 += kc[k * 8 + 2 * q + 1];
    uint32_t nam = 0;
    if (NA) {
#pragma unroll
      for (int sl = 0; sl < 2; sl++)
#pragma unroll
        for (int j = 0; j < 4; j++) {
          uint32_t f = naw[sl][j] & 0x55555555u;
          f |= f >> 16;
          f |= f >> 8;
#pragma unroll
          for (int c = 0; c < 4; c++) nam |= ((f >> (2 * c)) & 1u) << ((sl * 4 + j) * 4 + c);
        }
      nam |= __shfl_xor_sync(0xffffffffu, nam, 1);
      nam |= __shfl_xor_sync(0xffffffffu, nam, 2);
    }
#pragma unroll
    for (int sl = 0; sl < 2; sl++)
#pragma unroll
      for (int j = 0; j < 4; j++)
#pragma unroll
        for (int c = 0; c < 4; c++) {
          long long v0 = ((long long)acc[j][c][2 * sl] >> (2 * c)) + kr0;
          long long v1 = ((long long)acc[j][c][2 * sl + 1] >> (2 * c)) + kr1;
          if (drained) {
            const int idx = ((j * 4 + c) * 2 + sl) * 2;
            v0 += base[(int64_t)idx * 256 + tid];
            v1 += base[(int64_t)(idx + 1) * 256 + tid];
          }
          double p = 0.0;
#pragma unroll
          for (int r = 3; r >= 0; r--) {
            const double in = __shfl_down_sync(0xffffffffu, p, 1);
            if (q == r)
              p = __dadd_rn(__dadd_rn(r == 3 ? 0.0 : in, scalbn((double)v1, 8 * (2 * r + 1) - e)),
                            scalbn((double)v0, 16 * r - e));
          }
          if (q == 0) {
            const int bit = (sl * 4 + j) * 4 + c;
            ebuf[4 * (4 * (8 * sl + g) + j) + c] = (NA && ((nam >> bit) & 1u)) ? __longlong_as_double(0x7ff8000000000000LL) : p;
          }
        }
    __syncwarp();
    double *dst = a.S + ((int64_t)set * a.nthr + a.col_of[k]) * a.n + 4 * byte0;
    const int64_t lim = (int64_t)a.n - 4 * byte0;
    for (int i = lane; i < 256; i += 32)
      if (i < lim) dst[i] = ebuf[i];
    __syncwarp();
    k++;
  };
  auto drain = [&]() {
#pragma unroll
    for (int j = 0; j < 4; j++)
#pragma unroll
      for (int c = 0; c < 4; c++)
#pragma unroll
        for (int sl = 0; sl < 2; sl++) {
          const int idx = ((j * 4 + c) * 2 + sl) * 2;
          base[(int64_t)idx * 256 + tid] += (long long)acc[j][c][2 * sl] >> (2 * c);
          base[(int64_t)(idx + 1) * 256 + tid] += (long long)acc[j][c][2 * sl + 1] >> (2 * c);
          acc[j][c][2 * sl] = acc[j][c][2 * sl + 1] = 0;
        }
    drained = true;
  };

  if (base) {  // zero this item's totals (each thread owns its own entries)
    for (int idx = 0; idx < 64; idx++) base[(int64_t)idx * 256 + tid] = 0;
  }
  while (k < a.nthr && send[k] == 0) emit();

#pragma unroll
  for (int st = 0; st < STG - 1; st++) {
    if (st < ngrp) issue(st, st);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  const uint8_t *dg = a.dig + (int64_t)g0 * 256 + g * 32 + 4 * q;  // slice g, lines 4q..4q+3 and 16+4q..16+4q+3
  const uint32_t rd_base = wbase + (uint32_t)((q * 8 + g) * 4);
  uint32_t rd_stage = 0, wr_stage = (STG - 1) * WSTAGE;
  for (int step = 0; step < ngrp; step++) {
    asm volatile("cp.async.wait_group %0;" ::"n"(STG - 2) : "memory");
    __syncwarp();
    {
      const int nxt = step + STG - 1;
      if (nxt < ngrp) issue(nxt, (int)(wr_stage / WSTAGE));
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    const uint32_t b0 = *reinterpret_cast<const uint32_t *>(dg + (int64_t)step * 256);
    const uint32_t b1 = *reinterpret_cast<const uint32_t *>(dg + (int64_t)step * 256 + 16);
    uint32_t W[2][2][4];  // [slot g / g+8][lines lo / hi][byte]
#pragma unroll
    for (int sl = 0; sl < 2; sl++)
#pragma unroll
      for (int hf = 0; hf < 2; hf++) {
        const uint32_t ad = rd_base + rd_stage + (hf * 2 + sl) * 128;
        const uint32_t x0 = lds32(ad), x1 = lds32(ad + 512), x2 = lds32(ad + 1024), x3 = lds32(ad + 1536);
        const uint32_t t0 = prmt(x0, x1, 0x5140), t1 = prmt(x2, x3, 0x5140);
        const uint32_t t2 = prmt(x0, x1, 0x7362), t3 = prmt(x2, x3, 0x7362);
        W[sl][hf][0] = prmt(t0, t1, 0x5410);
        W[sl][hf][1] = prmt(t0, t1, 0x7632);
        W[sl][hf][2] = prmt(t2, t3, 0x5410);
        W[sl][hf][3] = prmt(t2, t3, 0x7632);
      }
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const uint32_t wa = W[0][0][j], wb = W[1][0][j], wc2 = W[0][1][j], wd = W[1][1][j];
      if (NA) {
        naw[0][j] |= (wa & (wa >> 1)) | (wc2 & (wc2 >> 1));
        naw[1][j] |= (wb & (wb >> 1)) | (wd & (wd >> 1));
      }
      mma_u8s8(acc[j][0], wa & 0x03030303u, wb & 0x03030303u, wc2 & 0x03030303u, wd & 0x03030303u, b0, b1);
      mma_u8s8(acc[j][1], wa & 0x0C0C0C0Cu, wb & 0x0C0C0C0Cu, wc2 & 0x0C0C0C0Cu, wd & 0x0C0C0C0Cu, b0, b1);
      mma_u8s8(acc[j][2], wa & 0x30303030u, wb & 0x30303030u, wc2 & 0x30303030u, wd & 0x30303030u, b0, b1);
      mma_u8s8(acc[j][3], wa & 0xC0C0C0C0u, wb & 0xC0C0C0C0u, wc2 & 0xC0C0C0C0u, wd & 0xC0C0C0C0u, b0, b1);
    }
    rd_stage = rd_stage + WSTAGE == STG * WSTAGE ? 0 : rd_stage + WSTAGE;
    wr_stage = wr_stage + WSTAGE == STG * WSTAGE ? 0 : wr_stage + WSTAGE;
    if (base && (step + 1) % CAP_GROUPS == 0) drain();
    while (k < a.nthr && send[k] == step + 1) emit();
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
}

// Reversed-allele constant of every (set, step, slice): sum over the step's reversed entries of -2 x digit, so that with
// the code-times-digit sums it gives prodVecRev's (g - 2) Q exactly.  One thread per (set, step, slice).
__global__ void k_prs_const(int nsets, int nthr, const int *__restrict__ grp_off, const int *__restrict__ step_end,
                            const uint8_t *__restrict__ kind, const uint8_t *__restrict__ dig, long long *__restrict__ kc) {
  const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= (int64_t)nsets * nthr * 8) return;
  const int s = (int)(t & 7), k = (int)((t >> 3) % nthr), set = (int)((t >> 3) / nthr);
  const int *se = step_end + (int64_t)set * nthr;
  const int64_t l0 = (int64_t)(grp_off[set] + (k ? se[k - 1] : 0)) * TL, l1 = (int64_t)(grp_off[set] + se[k]) * TL;
  long long acc = 0;
  for (int64_t l = l0; l < l1; l++)
    if (kind[l] == 1) acc -= 2 * (long long)(int8_t)dig[(l >> 5) * 256 + s * 32 + (l & 31)];
  kc[t] = acc;
}

// A set with a non-finite weight: R's arithmetic element by element (NA code -> NA_real; raw != null: the raw bytes of a
// dosage table through code256), one thread per sample:
// last = last + (sum over the step's entries in order of g v + cst[step]) for every step.
__global__ void k_prs_literal(const uint8_t *__restrict__ P, int64_t stride, const uint8_t *__restrict__ raw,
                              const double *__restrict__ code, int n, int set, int nthr,
                              const int *__restrict__ grp_off, const int *__restrict__ step_end,
                              const int *__restrict__ col_of, const int *__restrict__ lines,
                              const uint8_t *__restrict__ kind, const double *__restrict__ v,
                              const double *__restrict__ cst, double *__restrict__ S) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int *se = step_end + (int64_t)set * nthr;
  double last = 0.0;
  for (int k = 0; k < nthr; k++) {
    const int64_t l0 = (int64_t)(grp_off[set] + (k ? se[k - 1] : 0)) * TL, l1 = (int64_t)(grp_off[set] + se[k]) * TL;
    double inc = 0.0;
    for (int64_t l = l0; l < l1; l++) {
      if (kind[l] == PAD) continue;
      double x;
      if (raw) {  // dosage table: code256 of the raw byte (NA_real for an NA code)
        x = code[raw[(int64_t)lines[l] * n + i]];
      } else {
        const int c = (P[(int64_t)lines[l] * stride + (i >> 2)] >> (2 * (i & 3))) & 3;
        x = c == 3 ? __longlong_as_double(0x7ff8000000000000LL) : (double)c;
      }
      inc = __dadd_rn(inc, __dmul_rn(x, v[l]));
    }
    last = __dadd_rn(last, __dadd_rn(inc, cst[(int64_t)set * nthr + k]));
    S[((int64_t)set * nthr + col_of[k]) * n + i] = last;
  }
}

// out (nr x ncol, column-major, float or double) = S rows `row` (0-based, repeats allowed)
__global__ void k_prs_gather(const double *__restrict__ S, int n, const int *__restrict__ row, int nr, int64_t ncol,
                             int out_double, void *__restrict__ out) {
  const int64_t total = (int64_t)nr * ncol;
  for (int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t col = t / nr;
    const double x = S[col * n + row[t - col * nr]];
    if (out_double)
      reinterpret_cast<double *>(out)[t] = x;
    else
      reinterpret_cast<float *>(out)[t] = __double2float_rn(x);
  }
}

// Dosage tables (bsg_dosage_scale D > 0): every finite code is byte / D with byte = round(D code256[raw]) in 0..255.
// One CTA per (set, 256 samples), one thread per sample reading the raw code bytes of each line (n x m column-major,
// coalesced across the CTA) through a 256-entry table (value byte, or -1 for an NA code).  Per slice the exact int32 sum
// of byte x digit (|byte x digit| <= 255 x 128 per line: CAP_GROUPS groups of head-room, then int64 totals); the step's
// constant is D x (-2 digit) per reversed entry, so a reversed entry adds (byte - 2 D) Q.  Score = the top-down fp64 sum
// of the 8 scaled slice totals, divided by D (one correctly rounded division).
constexpr int DOS_T = 256;
struct DArgs {
  const uint8_t *raw;
  const int *lut;           // [256] value byte of a raw code, -1 for NA
  int n, nsb, nthr;
  double D;
  const int *lines, *grp_off, *step_end, *col_of;
  const uint8_t *dig;
  const long long *kc;
  const Scal *sc;
  double *S;
};

__global__ void __launch_bounds__(DOS_T) k_prs_dos(const DArgs a) {
  __shared__ int lut[256], sdig[256], sline[TL];
  const int tid = threadIdx.x, set = blockIdx.x / a.nsb, sb = blockIdx.x % a.nsb;
  const int64_t i = (int64_t)sb * DOS_T + tid;
  const bool valid = i < a.n;
  const int g0 = a.grp_off[set], ngrp = a.grp_off[set + 1] - g0;
  const int *send = a.step_end + (int64_t)set * a.nthr;
  const long long *kc = a.kc + (int64_t)set * a.nthr * 8;
  const int e = a.sc[set].e[0];
  const long long Di = (long long)a.D;
  lut[tid] = a.lut[tid];
  int acc[8];
  long long tot[8], kr[8];
#pragma unroll
  for (int s = 0; s < 8; s++) acc[s] = 0, tot[s] = 0, kr[s] = 0;
  bool na = false;
  int k = 0;
  auto emit = [&]() {
    double p = 0.0;
#pragma unroll
    for (int s = 7; s >= 0; s--) {
      kr[s] += Di * kc[k * 8 + s];
      p = __dadd_rn(p, scalbn((double)(tot[s] + acc[s] + kr[s]), 8 * s - e));
    }
    if (valid)
      a.S[((int64_t)set * a.nthr + a.col_of[k]) * a.n + i] =
          na ? __longlong_as_double(0x7ff8000000000000LL) : __ddiv_rn(p, a.D);
    k++;
  };
  __syncthreads();
  while (k < a.nthr && send[k] == 0) emit();
  for (int grp = 0; grp < ngrp; grp++) {
    __syncthreads();
    sdig[tid] = (int)(int8_t)a.dig[(int64_t)(g0 + grp) * 256 + tid];  // [slice][line]
    if (tid < TL) sline[tid] = a.lines[(int64_t)(g0 + grp) * TL + tid];
    __syncthreads();
    if (valid) {
#pragma unroll 4
      for (int l = 0; l < TL; l++) {
        int v = lut[a.raw[(int64_t)sline[l] * a.n + i]];
        na |= v < 0;
        v = max(v, 0);
#pragma unroll
        for (int s = 0; s < 8; s++) acc[s] += v * sdig[s * 32 + l];
      }
    }
    if ((grp + 1) % CAP_GROUPS == 0) {
#pragma unroll
      for (int s = 0; s < 8; s++) tot[s] += acc[s], acc[s] = 0;
    }
    while (k < a.nthr && send[k] == grp + 1) emit();
  }
}

static thread_local double g_last_ms = 0;  // of the last call on this thread

}  // namespace prs
}  // namespace bsg

using namespace bsg;

extern "C" {

int bsg_prs_grid(bsg_bed *h, const int *ind_row, int nr, int nsets, const int *set_len, const int *cols,
                 const double *beta, const int *same, const double *lpS, int nthr, const double *thr, int out_double,
                 void *out) {
  using namespace prs;
  if (!h || nsets < 0 || nthr < 1 || (nsets > 0 && !set_len) || (!thr && nthr != 1) || (thr && !lpS))
    return fail(BSG_ERR_ARG, "null argument or bad lengths");
  const bool dos = h->fbm_generic != 0;
  BSG_TRY(genotypes_check(h, "snp_PRS on the device needs"));
  BSG_TRY(bind_device(h));
  if (!ind_row) nr = h->n;
  if (nr < 0) return fail(BSG_ERR_ARG, "bad length of ind.row");
  std::vector<int> row0;
  BSG_TRY(host_index(ind_row, nr, h->n, "", row0));
  // thresholds in stable decreasing order (R's order(thr.list, decreasing = TRUE))
  std::vector<int> ord(nthr);
  std::iota(ord.begin(), ord.end(), 0);
  if (thr) {
    for (int t = 0; t < nthr; t++)
      if (thr[t] != thr[t]) return fail(BSG_ERR_ARG, "'thr.list' must not be NA.");
    std::stable_sort(ord.begin(), ord.end(), [&](int x, int y) { return thr[x] > thr[y]; });
  }
  // steps of every entry, padded line lists
  std::vector<int> grp_off(nsets + 1, 0), step_end((size_t)nsets * nthr), lines;
  std::vector<uint8_t> kind;
  std::vector<double> v, cst((size_t)nsets * nthr, 0.0);
  std::vector<int> long_slot(std::max(nsets, 1), -1);
  int nlong = 0;
  int64_t e0 = 0;
  for (int c = 0; c < nsets; c++) {
    const int L = set_len[c];
    if (L < 0) return fail(BSG_ERR_ARG, "set %d: bad length.", c + 1);
    if (L > 0 && (!cols || !beta)) return fail(BSG_ERR_ARG, "null argument");
    std::vector<std::vector<int>> by_step(nthr);
    for (int i = 0; i < L; i++) {
      const int64_t t = e0 + i;
      if (cols[t] < 1 || cols[t] > h->m) return fail(BSG_ERR_BOUNDS, "ind.keep out of range");
      if (same && same[t] != 0 && same[t] != 1) return fail(BSG_ERR_ARG, "'same.keep' must be TRUE or FALSE.");
      int k = 0;
      if (thr) {
        const double p = lpS[t];
        if (!(p >= 0)) return fail(BSG_ERR_ARG, "'lpS.keep' must be non-negative and not NA.");
        while (k < nthr && !(p > thr[ord[k]])) k++;
      }
      if (k < nthr) by_step[k].push_back(i);
    }
    int grp = grp_off[c];
    for (int k = 0; k < nthr; k++) {
      const auto &ix = by_step[k];
      const int np = (int)round_up((int64_t)ix.size(), TL);
      double sum_rev = 0.0;  // sum(betas[!same]) of the step, in order
      for (int p = 0; p < np; p++) {
        const int i = ix[p < (int)ix.size() ? p : 0];
        const int64_t t = e0 + i;
        const bool rev = same && !same[t];
        lines.push_back(cols[t] - 1);
        kind.push_back(p < (int)ix.size() ? (rev ? 1 : 0) : PAD);
        v.push_back(p < (int)ix.size() ? (rev ? -beta[t] : beta[t]) : 0.0);
        if (p < (int)ix.size() && rev) sum_rev += beta[t];
      }
      cst[(size_t)c * nthr + k] = 2 * sum_rev;
      grp += np / TL;
      step_end[(size_t)c * nthr + k] = grp - grp_off[c];
    }
    grp_off[c + 1] = grp;
    if (!dos && grp - grp_off[c] > CAP_GROUPS) long_slot[c] = nlong++;
    e0 += L;
  }
  std::vector<int> col_of(nthr);
  for (int k = 0; k < nthr; k++) col_of[k] = ord[k];
  const int64_t nl = (int64_t)lines.size(), ngrp = nl / TL;
  const int n = h->n;
  const int64_t ncol = (int64_t)nsets * nthr;
  const int64_t nbytes = ((int64_t)n + 3) / 4;
  const int nblocks = (int)std::max<int64_t>(1, (nbytes + TB - 1) / TB);
  const size_t osz = out_double ? sizeof(double) : sizeof(float);
  if (nr > 0 && ncol > 0 && !out) return fail(BSG_ERR_ARG, "null argument");
  // every device array of the call, before allocating any
  const size_t need = (dos ? (size_t)256 * sizeof(int) : 0) + (size_t)nl * (sizeof(int) + 1 + sizeof(double)) + (size_t)ngrp * 256 +
                      (size_t)ncol * (8 * sizeof(long long) + sizeof(double) + 2 * sizeof(int)) +
                      (size_t)nsets * (sizeof(Scal) + 2 * sizeof(int)) + (size_t)nlong * nblocks * 64 * 256 * 8 +
                      (size_t)ncol * n * sizeof(double) + (size_t)ncol * nr * osz + (size_t)nr * sizeof(int) + 4096;
  size_t fr = 0, tot = 0;
  BSG_CUDA(cudaMemGetInfo(&fr, &tot));
  if (need > fr)
    return fail(BSG_ERR_ALLOC, "snp_grid_PRS needs %.0f bytes of device memory (%lld score columns of %d samples), %.0f "
                               "are free.", (double)need, (long long)ncol, n, (double)fr);
  if (ncol == 0 || nr == 0) return BSG_OK;

  cudaStream_t s = h->stream;
  Bufs b;
  int *d_lut = dos ? dosage_lut(h, b) : nullptr;
  int *d_lines, *d_goff, *d_send, *d_col, *d_slot, *d_row;
  uint8_t *d_kind, *d_dig;
  double *d_v, *d_cst, *d_S;
  long long *d_kc, *d_base = nullptr;
  Scal *d_sc;
  void *d_out;
  b.up(&d_lines, lines, s);
  b.up(&d_goff, grp_off, s);
  b.up(&d_send, step_end, s);
  b.up(&d_col, col_of, s);
  b.up(&d_slot, long_slot, s);
  b.up(&d_row, row0.data(), (size_t)nr, s);
  b.up(&d_kind, kind, s);
  b.up(&d_v, v, s);
  b.up(&d_cst, cst, s);
  b.alloc(&d_dig, (size_t)std::max<int64_t>(ngrp, 1) * 256);
  b.alloc(&d_kc, (size_t)ncol * 8);
  b.alloc(&d_sc, (size_t)std::max(nsets, 1));
  if (nlong) b.alloc(&d_base, (size_t)nlong * nblocks * 64 * 256);
  b.alloc(&d_S, (size_t)ncol * n);
  b.alloc((uint8_t **)&d_out, (size_t)ncol * nr * osz);
  BSG_TRY(b.status("snp_grid_PRS scratch"));
  CallTimer tm;
  BSG_CUDA(tm.start(s));
  BSG_CUDA(cudaMemsetAsync(d_sc, 0, (size_t)std::max(nsets, 1) * sizeof(Scal), s));
  for (int c = 0; c < nsets; c++) {
    const int64_t l0 = (int64_t)grp_off[c] * TL, len = (int64_t)(grp_off[c + 1] - grp_off[c]) * TL;
    if (len) BSG_TRY(prs_prep(d_v + l0, (int)len, d_sc + c, d_dig + l0 / TL * 256, s));
  }
  const int64_t nkc = ncol * 8;
  k_prs_const<<<(int)((nkc + 255) / 256), 256, 0, s>>>(nsets, nthr, d_goff, d_send, d_kind, d_dig, d_kc);
  static std::atomic<unsigned> attr_done{0};  // function attributes are per device
  if (!dos && !(attr_done.load() >> (h->device & 31) & 1u)) {
    BSG_CUDA(cudaFuncSetAttribute(k_prs<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    BSG_CUDA(cudaFuncSetAttribute(k_prs<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
    attr_done.fetch_or(1u << (h->device & 31));
  }
  Args a;
  a.P = h->A;
  a.stride = h->strideA;
  a.n = n;
  a.nblocks = nblocks;
  a.nthr = nthr;
  a.lines = d_lines;
  a.grp_off = d_goff;
  a.step_end = d_send;
  a.col_of = d_col;
  a.dig = d_dig;
  a.kc = d_kc;
  a.sc = d_sc;
  a.long_slot = d_slot;
  a.base = d_base;
  a.S = d_S;
  const int64_t grid = (int64_t)nsets * nblocks;
  if (dos) {
    DArgs d;
    d.raw = h->raw;
    d.lut = d_lut;
    d.n = n;
    d.nsb = (n + DOS_T - 1) / DOS_T;
    d.nthr = nthr;
    d.D = (double)h->dos_scale;
    d.lines = d_lines;
    d.grp_off = d_goff;
    d.step_end = d_send;
    d.col_of = d_col;
    d.dig = d_dig;
    d.kc = d_kc;
    d.sc = d_sc;
    d.S = d_S;
    k_prs_dos<<<(unsigned)((int64_t)nsets * d.nsb), DOS_T, 0, s>>>(d);
  } else if (h->has_na)
    k_prs<true><<<(unsigned)grid, WARPS * 32, SMEM, s>>>(a);
  else
    k_prs<false><<<(unsigned)grid, WARPS * 32, SMEM, s>>>(a);
  count_launch(2);
  BSG_CUDA(cudaGetLastError());
  // sets with a non-finite weight: the literal loop overwrites their columns
  std::vector<Scal> hsc(std::max(nsets, 1));
  BSG_CUDA(cudaMemcpyAsync(hsc.data(), d_sc, (size_t)std::max(nsets, 1) * sizeof(Scal), cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  for (int c = 0; c < nsets; c++)
    if (hsc[c].nonfinite) {
      k_prs_literal<<<(n + 255) / 256, 256, 0, s>>>(h->A, h->strideA, dos ? h->raw : nullptr, h->d_code, n, c, nthr, d_goff, d_send, d_col, d_lines, d_kind,
                                                    d_v, d_cst, d_S);
      count_launch();
    }
  k_prs_gather<<<(int)std::min<int64_t>((ncol * nr + 255) / 256, 132 * 16), 256, 0, s>>>(d_S, n, d_row, nr, ncol,
                                                                                        out_double, d_out);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  BSG_CUDA(tm.stop(s));
  BSG_CUDA(cudaMemcpyAsync(out, d_out, (size_t)ncol * nr * osz, cudaMemcpyDeviceToHost, s));
  BSG_CUDA(cudaStreamSynchronize(s));
  g_last_ms = tm.ms();
  return BSG_OK;
}

double bsg_prs_last_ms(void) { return prs::g_last_ms; }

}  // extern "C"
