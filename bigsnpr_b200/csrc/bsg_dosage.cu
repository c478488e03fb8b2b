// bsg_dosage.cu -- X.y and Xt.y of FBM.code256 dosage matrices (CODE_DOSAGE, R/bigSNP-class.R:13) on the integer tensor pipe.
//
// bigsnpr writes dosages as an FBM.code256 whose table holds 0, 1, 2, NA, 0, 1, 2, seq(0, 2, by = 0.01), NA x 48
// (snp_readBGEN, R/read-bgen.R:184; snp_fastImputeSimple(method = "mean2"), R/impute.R:189-203).  Every finite value is an
// integer multiple of 1/100 in [0, 2], so q = round(100 code256[byte]) is an exact u8 and the products run as
// IMMA.16832.U8.S8 against the same signed base-256 digits of the quantised vector as the 2-bit kernels (bsg_pmv.cu):
// exact integer sums, bit-reproducible whatever the work split.  The general rule: the handle's table qualifies when
// some D in 1..255 makes D v an integer in 0..255 (within 1e-9) for every finite v and every other value is NaN
// (bsg_code256_dosage_scale); D = 1/100 -> 100.  Elements follow SubBMCode256Acc plus bigstatsr's scaling
// ([bigstatsr, unvendored]): (code256[b] - c_j) / s_j = (q / D - c_j) / s_j, and an NA code poisons the outputs it touches.
//
// Operand: the value copy (bsg_bed::dosV), m SNP lines of round_up(n, 128) bytes, built on first use.  Vector: the 61-bit
// fixed point of bsg_pmv.cu (pick_e, peel, k_prep1, k_quantise) in k_quantT's [step][slice][32] layout, which is the
// m16n8k32 B fragment for any contraction index.
//
// Exactness: q <= 255 and |digit| <= 128, so one product is at most 32,640 and an int32 accumulator holds 65,536 of them
// (65,536 x 32,640 = 2,139,095,040 < 2^31): both kernels cap a k-split at 65,536 contraction indices (the 2-bit kernels:
// 262,144).  The exponent rule is unchanged: pick_e bounds |Q| (after a scatter of up to 2^hb duplicates) by 2^60, which
// is what 8 signed base-256 digits represent; the matrix operand enters only through the accumulator bound above.  The
// per-slice int64 totals stay below m x 32,640 < 2^46.  1/D is applied once, in fp64, by the finish kernels.
//
//   k_dmv   Xt.y: lines = selected SNP columns, contraction along a line (samples).  A fragment = one 32-bit word of the
//           line (4 consecutive samples), no unpack.  A row-index multiset is scattered into Q by k_quantise first.
//   k_dmvT  X.y: contraction across lines.  k_pmvT's CTA stage (32 lines x 512 B, 6 stages, full / empty mbarriers); a
//           thread transposes 4 x 4 bytes of 4 consecutive lines with PRMTs and each transposed word is directly the A
//           fragment of one sample.  Identity selection: 2D TMA boxes, 128-byte swizzle.  Column list: one 512-byte
//           cp.async.bulk per selected line into rows of 528 bytes.  Either way the q >= 2 row rotation of k_pmvT keeps
//           every LDS on 32 distinct banks (tests/test_dosage_layout.py replays both layouts).
#include <math.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "bsg_internal.cuh"
#include "bsg_pmv_shared.cuh"

namespace bsg {

int dosage_scale_of(const double *code256) {
  for (int D = 1; D <= 255; D++) {
    bool ok = true;
    for (int k = 0; k < 256 && ok; k++) {
      const double v = code256[k];
      if (v != v) continue;  // NA
      if (!isfinite(v)) ok = false;
      const double t = D * v, r = nearbyint(t);
      ok = ok && fabs(t - r) <= 1e-9 && r >= 0 && r <= 255;
    }
    if (ok) return D;
  }
  return 0;
}

namespace dos {
using namespace pmv;

// ---- staging ---------------------------------------------------------------------------------------------------------
// raw (n x m bytes, column-major) -> value copy; one block per line, NA codes counted per line
__global__ void k_value_copy(const uint8_t *__restrict__ raw, int n, int m, const uint8_t *__restrict__ qmap,
                             const uint8_t *__restrict__ isna, uint8_t *__restrict__ V, int64_t stride,
                             int32_t *__restrict__ nacnt) {
  __shared__ int sh[8];
  const int64_t words = stride / 4;
  for (int j = blockIdx.x; j < m; j += gridDim.x) {
    const uint8_t *src = raw + (int64_t)j * n;
    int cnt = 0;
    for (int64_t w = threadIdx.x; w < words; w += blockDim.x) {
      uint32_t v = 0;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        const int64_t i = 4 * w + k;
        if (i < n) {
          const uint8_t b = src[i];
          cnt += isna[b];
          v |= (uint32_t)qmap[b] << (8 * k);
        }
      }
      reinterpret_cast<uint32_t *>(V + (int64_t)j * stride)[w] = v;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = cnt;
    __syncthreads();
    if (threadIdx.x == 0) {
      int t = 0;
      for (int k = 0; k < (int)(blockDim.x >> 5); k++) t += sh[k];
      nacnt[j] = t;
    }
    __syncthreads();
  }
}

// (line, sample) of every NA code, line by line in sample order (one warp per line holding one)
__global__ void k_na_list(const uint8_t *__restrict__ raw, int n, int m, const uint8_t *__restrict__ isna,
                          const int32_t *__restrict__ nacnt, const long long *__restrict__ off, int2 *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int j = warp; j < m; j += nw) {
    if (nacnt[j] == 0) continue;
    const uint8_t *src = raw + (int64_t)j * n;
    long long pos = off[j];
    for (int i0 = 0; i0 < n; i0 += 32) {
      const int i = i0 + lane;
      const bool na = i < n && isna[src[i]];
      const unsigned b = __ballot_sync(0xffffffffu, na);
      if (na) out[pos + __popc(b & ((1u << lane) - 1u))] = make_int2(j, i);
      pos += __popc(b);
    }
  }
}

__global__ void k_mark(const int *__restrict__ idx, int len, uint8_t *__restrict__ flag) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < len) flag[idx[t]] = 1;
}

// ---- vector layout ---------------------------------------------------------------------------------------------------
// Xt.y digits over the n samples in k_quantT's layout dig[(t / 32) * 256 + slice * 32 + t % 32], t < len_pad (the line
// stride; zero past n), from the integers k_quantise scattered into Q (the only quantisation of the vector).  Publishes
// the exponent and the exact sum of Q (Y = sum y over the selected rows, duplicates included).
__global__ void k_digits_rows(const long long *__restrict__ Q, int n, int len_pad, Scal *sc, uint8_t *__restrict__ dig) {
  if (blockIdx.x == 0 && threadIdx.x == 0) sc->e[0] = pick_e(sc->maxabs[0], sc->hb, 60);
  long long hi = 0, lo = 0;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < len_pad; t += gridDim.x * blockDim.x) {
    long long q = t < n ? Q[t] : 0;
    hi += q >> 32;
    lo += (long long)(unsigned int)(q & 0xFFFFFFFFll);
    const int64_t base = (int64_t)(t >> 5) * 256 + (t & 31);
#pragma unroll
    for (int sl = 0; sl < 8; sl++) dig[base + sl * 32] = (uint8_t)peel(q);
  }
#pragma unroll
  for (int o = 16; o; o >>= 1) {
    hi += __shfl_xor_sync(0xffffffffu, hi, o);
    lo += __shfl_xor_sync(0xffffffffu, lo, o);
  }
  if ((threadIdx.x & 31) == 0 && (hi | lo)) {
    atomicAdd(reinterpret_cast<unsigned long long *>(&sc->sum_hi), (unsigned long long)hi);
    atomicAdd(reinterpret_cast<unsigned long long *>(&sc->sum_lo), (unsigned long long)lo);
  }
}

// any non-finite center or 1 / scale: the _dev forms return all NaN (the host forms re-run the literal loop)
__global__ void k_check_scaling(const double *__restrict__ center, const double *__restrict__ scale, int nc, Scal *sc) {
  int bad = 0;
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < nc; j += gridDim.x * blockDim.x)
    bad |= !isfinite(center[j]) || !isfinite(1.0 / scale[j]);
  if (__any_sync(0xffffffffu, bad) && (threadIdx.x & 31) == 0) atomicOr(&sc->nonfinite, 1);
}

// ---- k_dmv: Xt.y -------------------------------------------------------------------------------------------------------
// A warp owns 32 lines (two 16-line sub-tiles) and walks a range of 64-sample chunks.  Lane (g, q) loads bytes
// [16 q, 16 q + 16) of the chunk from lines g, g + 8, g + 16, g + 24 (every warp load = 8 lines x 64 contiguous bytes) and
// the digit bytes of the same 16 samples, slice g: one 16-byte word at (2 c + q / 2) * 256 + 32 g + 16 (q & 1).  Word w of
// both is k slots 4q..4q+3 (w even) or 16+4q..16+4q+3 (w odd) of IMMA w / 2: two IMMAs per sub-tile and chunk.
constexpr int DW = 8;                                  // warps per CTA
constexpr int DCH = 64;                                // samples per chunk
constexpr int DU = 4;                                  // chunks loaded ahead per warp
constexpr int DMAX_CHUNKS = 65536 / DCH;               // int32 accumulator cap per k-split

struct DArgs {
  const uint8_t *V;
  int64_t stride;
  const int *lines;     // physical line per selected column (null = identity)
  int nlines, nchunks, chunks_per_split, ksplit;
  const uint8_t *dig;   // [stride / 32][8][32]
  long long *part;      // [nlines][16], slices in 0..7
};

__global__ void __launch_bounds__(DW * 32) k_dmv(const DArgs a) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, q = lane & 3;
  const int ngroups = (a.nlines + 32 * DW - 1) / (32 * DW);
  for (int item = blockIdx.x; item < ngroups * a.ksplit; item += gridDim.x) {
    const int grp = item / a.ksplit, ks = item - grp * a.ksplit;
    const int lbase = grp * 32 * DW + warp * 32;
    if (lbase >= a.nlines) continue;  // warp-uniform
    const int c0 = ks * a.chunks_per_split, c1 = min(a.nchunks, c0 + a.chunks_per_split);
    const uint8_t *p[2][2];  // [sub-tile][row g / g + 8]
#pragma unroll
    for (int t = 0; t < 2; t++)
#pragma unroll
      for (int hh = 0; hh < 2; hh++) {
        const int l = min(lbase + 16 * t + 8 * hh + g, a.nlines - 1);
        p[t][hh] = a.V + (int64_t)(a.lines ? a.lines[l] : l) * a.stride + 16 * q;
      }
    const uint8_t *dp = a.dig + (q >> 1) * 256 + g * 32 + 16 * (q & 1);
    int acc[2][2][4];
#pragma unroll
    for (int t = 0; t < 2; t++)
#pragma unroll
      for (int k = 0; k < 4; k++) acc[t][0][k] = acc[t][1][k] = 0;
    for (int c = c0; c < c1; c += DU) {
      uint4 A[DU][2][2], B[DU];
#pragma unroll
      for (int k = 0; k < DU; k++) {
        if (c + k < c1) {
          const int64_t off = (int64_t)(c + k) * DCH;
#pragma unroll
          for (int t = 0; t < 2; t++)
#pragma unroll
            for (int hh = 0; hh < 2; hh++) A[k][t][hh] = ldg_stream(p[t][hh] + off);
          B[k] = __ldg(reinterpret_cast<const uint4 *>(dp + (int64_t)(c + k) * 512));
        } else {
          B[k] = make_uint4(0, 0, 0, 0);
#pragma unroll
          for (int t = 0; t < 2; t++) A[k][t][0] = A[k][t][1] = B[k];
        }
      }
#pragma unroll
      for (int k = 0; k < DU; k++)
#pragma unroll
        for (int t = 0; t < 2; t++) {
          const uint4 &r0 = A[k][t][0], &r1 = A[k][t][1];
          mma_u8s8(acc[t][0], r0.x, r1.x, r0.y, r1.y, B[k].x, B[k].y);
          mma_u8s8(acc[t][1], r0.z, r1.z, r0.w, r1.w, B[k].z, B[k].w);
        }
    }
    // D rows = lines g / g + 8 of the sub-tile, columns = slices 2q, 2q + 1
#pragma unroll
    for (int t = 0; t < 2; t++)
#pragma unroll
      for (int hh = 0; hh < 2; hh++) {
        const int l = lbase + 16 * t + 8 * hh + g;
        if (l < a.nlines) {
          unsigned long long *dst = reinterpret_cast<unsigned long long *>(a.part) + (int64_t)l * 16 + 2 * q;
          const long long v0 = (long long)acc[t][0][2 * hh] + acc[t][1][2 * hh];
          const long long v1 = (long long)acc[t][0][2 * hh + 1] + acc[t][1][2 * hh + 1];
          if (v0) atomicAdd(dst, (unsigned long long)v0);
          if (v1) atomicAdd(dst + 1, (unsigned long long)v1);
        }
      }
  }
}

// ---- k_dmvT: X.y -------------------------------------------------------------------------------------------------------
constexpr int TL = 32, TB = 512, TW = 8, NST = 6;
constexpr int TBOX = 32 * 128;                      // TMA stage: 4 boxes of 32 rows x 128 B, 128-byte swizzle
constexpr int ROWP = 528;                           // line-list stage: one unswizzled 512-byte row per line, 16 B pad
constexpr int STG = 4 * TBOX + 1024;                // both stage kinds (digits at DIG_T / DIG_L), 1 KB aligned
constexpr int DIG_T = 4 * TBOX, DIG_L = TL * ROWP;
constexpr int SMEM_T = NST * STG + 2 * NST * 8 + 1024;
constexpr int MAX_LINES = 65536;                    // int32 accumulator cap per k-split
static_assert(DIG_L + 400 <= STG, "line-list stage overflows");

struct XArgs {
  const uint8_t *V;
  int64_t stride;
  const int *lines;   // physical line of selected column t (null = identity)
  int nlines;
  const uint8_t *dig; // [steps][8][32]
  int lines_per_split, ksplit, nblocks, n;
  long long *part;    // [n][16]
};


template <bool LINES>
__global__ void __launch_bounds__(TW * 32, 2) k_dmvT(const __grid_constant__ CUtensorMap map, const XArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
  const int blk = blockIdx.x % a.nblocks, ks = blockIdx.x / a.nblocks;
  const int l0 = ks * a.lines_per_split, l1 = min(a.nlines, l0 + a.lines_per_split);
  const int nsteps = (l1 - l0 + TL - 1) / TL;
  const uint32_t sbase = (smem_u32(smem) + 1023u) & ~1023u;
  const uint32_t bar_base = sbase + NST * STG;  // full[s] at +8s, empty[s] at +8(NST+s)
  constexpr uint32_t DIG = LINES ? DIG_L : DIG_T;
  // producer: thread 0 (TMA boxes) or warp 0 (one bulk copy per line and lane); + the step's two 128-byte digit halves
  auto fill = [&](int step, int st) {
    const uint32_t full = bar_base + 8 * st, dst = sbase + st * STG;
    const uint8_t *dg = a.dig + (int64_t)(l0 / TL + step) * 256;
    if (LINES) {
      if (lane == 0) mbar_expect_tx(full, TL * TB + 256);
      __syncwarp();
      const int t = min(l0 + step * TL + lane, l1 - 1);  // rows past the split meet zero digits
      bulk_g2s(dst + lane * ROWP, a.V + (int64_t)a.lines[t] * a.stride + (int64_t)blk * TB, TB, full);
    } else {
      mbar_expect_tx(full, 4 * TBOX + 256);
#pragma unroll
      for (int j = 0; j < 4; j++) tma_load_2d(dst + j * TBOX, &map, full, blk * TB + 128 * j, l0 + step * TL);
    }
    if (!LINES || lane == 0) {
      bulk_g2s(dst + DIG, dg, 128, full);
      bulk_g2s(dst + DIG + 144, dg + 128, 128, full);
    }
  };
  if (tid == 0) {
    for (int st = 0; st < NST; st++) {
      mbar_init(bar_base + 8 * st, 1);
      mbar_init(bar_base + 8 * (NST + st), TW);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  const bool producer = LINES ? warp == 0 : tid == 0;
  if (producer)
    for (int st = 0; st < min(NST, nsteps); st++) fill(st, st);
  int stage = 0, pstage = 0;
  uint32_t phase = 0, pphase = 0;

  const int64_t byte0 = (int64_t)blk * TB + 64 * warp;  // this warp's 64 samples of every line
  const int rsw = 2 * (q >> 1);
  // TMA stage: read i of word column 8 sl + g sits at row 4 q + (i ^ rsw), chunk (4 (w & 1) + 2 sl + (g >> 2)) ^ (4 (q & 1)
  // + (i ^ rsw)), word g & 3 of box w >> 1 (k_pmvT).  Line-list stage: row 4 q + (i ^ rsw) at ROWP bytes per row, word
  // 16 w + 8 sl + g: bank = 16 q + 4 (i ^ rsw) + 16 w + 8 sl + g (mod 32), 32 distinct values over the lanes.
  const uint32_t chunk0 = (4 * (warp & 1) + (g >> 2)) ^ (4 * (q & 1) + rsw);
  const uint32_t rd_base = LINES ? sbase + (uint32_t)((4 * q) * ROWP + (16 * warp + g) * 4)
                                 : sbase + (warp >> 1) * TBOX + q * 512 + (rsw << 7) + chunk0 * 16 + 4 * (g & 3);
  const uint32_t dg_base = sbase + DIG + g * 32 + 16 * (g >> 2) + 4 * q;  // slice g, lines 4q..4q+3
  const uint32_t sel_lo = rsw ? 0x1054u : 0x5410u, sel_hi = rsw ? 0x3276u : 0x7632u;

  int acc[4][4];
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int k = 0; k < 4; k++) acc[j][k] = 0;

  for (int step = 0; step < nsteps; step++) {
    const uint32_t full = bar_base + 8 * stage, empty = bar_base + 8 * (NST + stage);
    const uint32_t so = stage * STG;
    const int cstage = stage;
    const uint32_t cphase = phase;
    mbar_wait(full, phase);
    const uint32_t b0 = lds32(dg_base + so), b1 = lds32(dg_base + so + 16);
    uint32_t W[2][2][4];  // [sample word g / g + 8][lines lo / hi][byte]
#pragma unroll
    for (int sl = 0; sl < 2; sl++)
#pragma unroll
      for (int hf = 0; hf < 2; hf++) {
        uint32_t x[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          if (LINES)
            x[i] = lds32(rd_base + so + (uint32_t)((16 * hf + (i ^ rsw)) * ROWP + sl * 32));
          else
            x[i] = lds32(((rd_base + so) ^ TRD(i, sl)) + hf * (16 * 128));
        }
        const uint32_t t0 = prmt(x[0], x[1], 0x5140), t1 = prmt(x[2], x[3], 0x5140);
        const uint32_t t2 = prmt(x[0], x[1], 0x7362), t3 = prmt(x[2], x[3], 0x7362);
        W[sl][hf][0] = prmt(t0, t1, sel_lo);
        W[sl][hf][1] = prmt(t0, t1, sel_hi);
        W[sl][hf][2] = prmt(t2, t3, sel_lo);
        W[sl][hf][3] = prmt(t2, t3, sel_hi);
      }
    __syncwarp();
    if (lane == 0) mbar_arrive(empty);
    if (++stage == NST) {
      stage = 0;
      phase ^= 1;
    }
    // byte r of W[sl][hf][j] = sample byte0 + 4 (8 sl + g) + j of line 16 hf + 4 q + r: the A fragment, no unpack
#pragma unroll
    for (int j = 0; j < 4; j++) mma_u8s8(acc[j], W[0][0][j], W[1][0][j], W[0][1][j], W[1][1][j], b0, b1);
    // refill one step behind (k_pmvT): the previous step's stage, once every warp has released it
    if (producer && step >= 1 && step - 1 + NST < nsteps) {
      mbar_wait(bar_base + 8 * (NST + pstage), pphase);
      fill(step - 1 + NST, pstage);
    }
    __syncwarp();
    pstage = cstage;
    pphase = cphase;
  }
#pragma unroll
  for (int j = 0; j < 4; j++)
#pragma unroll
    for (int sl = 0; sl < 2; sl++) {
      const int64_t sample = byte0 + 4 * (8 * sl + g) + j;
      if (sample < a.n) {
        unsigned long long *dst = reinterpret_cast<unsigned long long *>(a.part) + sample * 16 + 2 * q;
        const long long v0 = acc[j][2 * sl], v1 = acc[j][2 * sl + 1];
        if (v0) atomicAdd(dst, (unsigned long long)v0);
        if (v1) atomicAdd(dst + 1, (unsigned long long)v1);
      }
    }
}

// ---- finish and NA rule ------------------------------------------------------------------------------------------------
// X.y: full_i = R_i / D - C  (C = sum_j c_j z_j), or R_i / D without scaling
__global__ void k_finish_dprod(const long long *__restrict__ part, int n, const Scal *sc, int has_scaling, double D,
                               double *__restrict__ full) {
  const int l = blockIdx.x * blockDim.x + threadIdx.x;
  if (l >= n) return;
  if (sc->nonfinite) {
    full[l] = nan("");
    return;
  }
  const double R = combine<8>(part, l, 0, 1, 0, sc->e[0]) / D;
  if (has_scaling) {
    double C = 0;
    for (int b = 0; b < SUMCZ_BLOCKS; b++) C += sc->cpart[b];
    full[l] = R - C;
  } else {
    full[l] = R;
  }
}

// Xt.y: out_j = (R_j / D - c_j Y) / s_j, or R_j / D
__global__ void k_finish_dcprod(const long long *__restrict__ part, int nlines, const Scal *sc,
                                const double *__restrict__ center, const double *__restrict__ scale, double D,
                                double *__restrict__ out) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= nlines) return;
  if (sc->nonfinite) {
    out[j] = nan("");
    return;
  }
  const int e = sc->e[0];
  const double R = combine<8>(part, j, 0, 1, 0, e) / D;
  if (center) {
    const double Y = scalbn((double)sc->sum_hi, 32 - e) + scalbn((double)sc->sum_lo, -e);
    out[j] = (R - center[j] * Y) / scale[j];
  } else {
    out[j] = R;
  }
}

// X.y: a row holding an NA code in a selected column is NaN (full is indexed by sample)
__global__ void k_na_rows(const int2 *__restrict__ na, long long total, const uint8_t *__restrict__ colsel,
                          double *__restrict__ full) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int2 p = na[t];
    if (!colsel || colsel[p.x]) full[p.y] = nan("");
  }
}

// Xt.y: a line holding an NA code in a selected row is flagged, then every output of a flagged line is NaN
__global__ void k_na_lines(const int2 *__restrict__ na, long long total, const uint8_t *__restrict__ rowsel,
                           uint8_t *__restrict__ bad) {
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
    const int2 p = na[t];
    if (!rowsel || rowsel[p.y]) bad[p.x] = 1;
  }
}
__global__ void k_na_cols(const uint8_t *__restrict__ bad, const int *__restrict__ lines, int nc, double *__restrict__ out) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t < nc && bad[lines ? lines[t] : t]) out[t] = nan("");
}

__global__ void k_gather_rows(const double *__restrict__ full, const int *__restrict__ idx, int len, double *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < len) out[i] = full[idx[i]];
}

// ---- literal loops (host-vector forms with non-finite input): sum of (code256[b] - c) / s * x, element by element ----
__global__ void k_lit_prod(const uint8_t *__restrict__ raw, int n, const double *__restrict__ code, const int *__restrict__ rows,
                           int nr, const int *__restrict__ cols, int nc, const double *__restrict__ center,
                           const double *__restrict__ scale, const double *__restrict__ x, double *__restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  const int r = rows ? rows[i] : i;
  double s = 0;
  for (int t = 0; t < nc; t++) {
    const double c = center ? center[t] : 0.0, sc = scale ? scale[t] : 1.0;
    s += (code[raw[(int64_t)(cols ? cols[t] : t) * n + r]] - c) / sc * x[t];
  }
  out[i] = s;
}

__global__ void k_lit_cprod(const uint8_t *__restrict__ raw, int n, const double *__restrict__ code, const int *__restrict__ rows,
                            int nr, const int *__restrict__ cols, int nc, const double *__restrict__ center,
                            const double *__restrict__ scale, const double *__restrict__ x, double *__restrict__ out) {
  const int lane = threadIdx.x & 31;
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, nw = (gridDim.x * blockDim.x) >> 5;
  for (int t = warp; t < nc; t += nw) {
    const uint8_t *col = raw + (int64_t)(cols ? cols[t] : t) * n;
    const double c = center ? center[t] : 0.0, sc = scale ? scale[t] : 1.0;
    double s = 0;
    for (int i = lane; i < nr; i += 32) s += (code[col[rows ? rows[i] : i]] - c) / sc * x[i];
#pragma unroll
    for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[t] = s;
  }
}

// prod_and_rowSumsSq2 (src/project-utils.cpp:11-43) literally, one thread per selected row in the reference's order:
// x = (code256[b] - c_j) / s_j (NA code: NaN), rss += x^2, XV[, k] += x V[j, k] (K = 0: row sums of squares only).
// BYTES: the code bytes of a dosage handle; else the 2-bit copy A of a hard-call handle (code 3 = NA).  na[i] = 1 when a
// selected column holds an NA code in the row.  HBM-bound byte / bit pass, not a tuned path: x^2 is not linear in the
// code, so the integer kernels do not give it.
template <bool BYTES>
__global__ void k_proj_literal(const uint8_t *__restrict__ P, int64_t stride, const double *__restrict__ code,
                               const int *__restrict__ rows, int nr, const int *__restrict__ cols, int nc,
                               const double *__restrict__ center, const double *__restrict__ scale,
                               const double *__restrict__ V, int K, double *__restrict__ XV, double *__restrict__ rss,
                               uint8_t *__restrict__ na) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nr) return;
  const int r = rows ? rows[i] : i;
  double s2 = 0;
  int any_na = 0;
  for (int j = 0; j < nc; j++) {
    const int64_t col = cols ? cols[j] : j;
    double v;
    if (BYTES) {
      v = code[P[col * stride + r]];
    } else {
      const int g = (P[col * stride + (r >> 2)] >> (2 * (r & 3))) & 3;
      v = g == 3 ? nan("") : (double)g;
    }
    any_na |= v != v;
    const double x = (v - (center ? center[j] : 0.0)) / (scale ? scale[j] : 1.0);
    s2 += x * x;
    for (int k = 0; k < K; k++) XV[(int64_t)k * nr + i] += x * V[(int64_t)k * nc + j];
  }
  rss[i] = s2;
  na[i] = (uint8_t)any_na;
}

__global__ void k_nan_rows(const uint8_t *__restrict__ na, int nr, int K, double *__restrict__ XV) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < nr && na[i])
    for (int k = 0; k < K; k++) XV[(int64_t)k * nr + i] = nan("");
}

static int env_int(const char *name, int dflt) {
  const char *ev = getenv(name);
  return ev ? atoi(ev) : dflt;
}

}  // namespace dos

// ---------------------------------------------------------------------------------------------------------------------
int dosage_build(bsg_bed *h) {
  using namespace dos;
  if (h->dosV) return BSG_OK;
  if (!h->dos_scale || !h->raw) return fail(BSG_ERR_TYPE, "not a dosage handle");
  cudaStream_t s = h->stream;
  const int n = h->n, m = h->m;
  const int64_t stride = round_up(n, 128);
  uint8_t both[2 * 256];  // [0, 256): q of each code (NA -> 0), [256, 512): NA flag
  for (int k = 0; k < 256; k++) {
    const double v = h->code256[k];
    both[256 + k] = v != v;
    both[k] = (v != v) ? 0 : (uint8_t)nearbyint(h->dos_scale * v);
  }
  uint8_t *V = nullptr, *tab = nullptr;
  int32_t *cnt = nullptr;
  long long *d_off = nullptr;
  int2 *na = nullptr;
  const size_t vbytes = (size_t)stride * m + 512;  // slack: a line-list stage loads whole 512-byte segments
  cudaError_t e = cudaMalloc(&V, vbytes);
  if (e == cudaSuccess) e = cudaMalloc(&cnt, (size_t)m * sizeof(int32_t));
  if (e == cudaSuccess) e = cudaMalloc(&tab, sizeof both);
  if (e != cudaSuccess) {
    cudaGetLastError();
    cudaFree(V);
    cudaFree(cnt);
    return fail(BSG_ERR_ALLOC, "cannot allocate the dosage value copy (%.2f GB): %s.", vbytes / 1e9, cudaGetErrorString(e));
  }
  int rc = BSG_OK;
  e = cudaMemcpyAsync(tab, both, sizeof both, cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(V + (size_t)stride * m, 0, 512, s);
  if (e != cudaSuccess) rc = cuda_fail(e, "dosage staging");
  std::vector<int32_t> hc(m);
  if (!rc) {
    dos::k_value_copy<<<std::min(m, 132 * 16), 256, 0, s>>>(h->raw, n, m, tab, tab + 256, V, stride, cnt);
    count_launch();
    e = cudaMemcpyAsync(hc.data(), cnt, (size_t)m * sizeof(int32_t), cudaMemcpyDeviceToHost, s);
    if (e == cudaSuccess) e = cudaStreamSynchronize(s);
    if (e != cudaSuccess) rc = cuda_fail(e, "dosage value copy");
  }
  long long total = 0;
  if (!rc) {
    std::vector<long long> off(m);
    for (int j = 0; j < m; j++) {
      off[j] = total;
      total += hc[j];
    }
    if (total > 0) {
      e = cudaMalloc(&na, (size_t)total * sizeof(int2));
      if (e == cudaSuccess) e = cudaMalloc(&d_off, (size_t)m * sizeof(long long));
      if (e == cudaSuccess) e = cudaMemcpyAsync(d_off, off.data(), (size_t)m * sizeof(long long), cudaMemcpyHostToDevice, s);
      if (e == cudaSuccess) {
        dos::k_na_list<<<std::min((m + 7) / 8, 132 * 16), 256, 0, s>>>(h->raw, n, m, tab + 256, cnt, d_off, na);
        count_launch();
        e = cudaStreamSynchronize(s);
      }
      if (e != cudaSuccess) rc = cuda_fail(e, "dosage NA list");
    }
  }
  cudaFree(d_off);
  cudaFree(tab);
  if (rc) {
    cudaFree(V);
    cudaFree(cnt);
    cudaFree(na);
    return rc;
  }
  h->dosV = V;
  h->dosStride = stride;
  h->dosNaCnt = cnt;
  h->dosNa = na;
  h->dosNaTotal = total;
  return BSG_OK;
}

int dosage_view_masks(bsg_view *v) {
  bsg_bed *h = v->h;
  if (!h->dosNaTotal) return BSG_OK;
  cudaStream_t s = h->stream;
  if (!v->row_identity) {
    BSG_CUDA(cudaMalloc(&v->d_rowsel, (size_t)h->n));
    BSG_CUDA(cudaMemsetAsync(v->d_rowsel, 0, (size_t)h->n, s));
    if (v->nr) dos::k_mark<<<(v->nr + 255) / 256, 256, 0, s>>>(v->d_row, v->nr, v->d_rowsel);
    count_launch();
  }
  if (!v->col_identity) {
    BSG_CUDA(cudaMalloc(&v->d_colsel, (size_t)h->m));
    BSG_CUDA(cudaMemsetAsync(v->d_colsel, 0, (size_t)h->m, s));
    if (v->nc) dos::k_mark<<<(v->nc + 255) / 256, 256, 0, s>>>(v->d_col, v->nc, v->d_colsel);
    count_launch();
  }
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

// X~ x: all n samples from the selected SNP lines (k_dmvT), then the NA rule and the row gather
int dosage_prodvec(bsg_view *v, const double *x_dev, double *out_dev, cudaStream_t s) {
  using namespace dos;
  bsg_bed *h = v->h;
  const int n = h->n, nc = v->nc;
  BSG_TRY(dosage_prep_cols(v, x_dev, s));
  BSG_TRY(v->s_part.ensure((size_t)std::max(n, 1) * 16 * sizeof(long long)));
  long long *part = v->s_part.as<long long>();
  BSG_CUDA(cudaMemsetAsync(part, 0, (size_t)n * 16 * sizeof(long long), s));
  if (nc > 0) {
    XArgs a;
    a.V = h->dosV;
    a.stride = h->dosStride;
    a.lines = v->d_col;
    a.nlines = nc;
    a.dig = v->s_dig1.as<uint8_t>();
    a.n = n;
    a.part = part;
    a.nblocks = (n + TB - 1) / TB;
    int nsm = 132;
    cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->device);
    // k-split: about 4 waves of 2 CTAs per SM, at least 32 steps per split, at most MAX_LINES lines (int32 head-room)
    const int nsteps = (nc + TL - 1) / TL;
    const int lo = (nc + MAX_LINES - 1) / MAX_LINES;
    int ks = std::max(lo, std::min(std::max(1, nsteps / 32), (8 * nsm + a.nblocks - 1) / a.nblocks));
    const int force = env_int("BSG_DMV_KS", 0);
    if (force > 0) ks = std::max(lo, force);
    a.lines_per_split = (int)round_up((nc + ks - 1) / ks, TL);
    a.ksplit = (nc + a.lines_per_split - 1) / a.lines_per_split;
    static unsigned attr_done = 0;
    if (!(attr_done >> (h->device & 31) & 1u)) {
      BSG_CUDA(cudaFuncSetAttribute(k_dmvT<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_T));
      BSG_CUDA(cudaFuncSetAttribute(k_dmvT<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_T));
      attr_done |= 1u << (h->device & 31);
    }
    CUtensorMap map;
    memset(&map, 0, sizeof map);
    const int grid = a.nblocks * a.ksplit;
    if (a.lines) {
      k_dmvT<true><<<grid, TW * 32, SMEM_T, s>>>(map, a);
    } else {
      BSG_TRY(make_map(&map, h->dosV, h->m, h->dosStride, TL));
      k_dmvT<false><<<grid, TW * 32, SMEM_T, s>>>(map, a);
    }
    count_launch();
  }
  double *full = out_dev;
  if (!v->row_identity) {
    BSG_TRY(v->s_full.ensure((size_t)std::max(n, 1) * sizeof(double)));
    full = v->s_full.as<double>();
  }
  Scal *sc = v->s_scal.as<Scal>();
  if (n > 0) {
    k_finish_dprod<<<(n + 255) / 256, 256, 0, s>>>(part, n, sc, v->has_scaling, (double)h->dos_scale, full);
    count_launch();
  }
  if (h->dosNaTotal && nc > 0) {
    k_na_rows<<<(int)std::min<long long>((h->dosNaTotal + 255) / 256, 132 * 16), 256, 0, s>>>(h->dosNa, h->dosNaTotal,
                                                                                            v->d_colsel, full);
    count_launch();
  }
  if (!v->row_identity && v->nr > 0) {
    k_gather_rows<<<(v->nr + 255) / 256, 256, 0, s>>>(full, v->d_row, v->nr, out_dev);
    count_launch();
  }
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

// t(X~) x: one output per selected SNP line (k_dmv), then the NA rule
int dosage_cprodvec(bsg_view *v, const double *x_dev, double *out_dev, cudaStream_t s) {
  using namespace dos;
  bsg_bed *h = v->h;
  const int n = h->n, nc = v->nc;
  const int64_t stride = h->dosStride;
  BSG_TRY(v->s_q0.ensure((size_t)std::max(n, 1) * sizeof(long long)));
  long long *Q = v->s_q0.as<long long>();
  BSG_TRY(dosage_prep_rows(v, x_dev, Q, s));
  Scal *sc = v->s_scal.as<Scal>();
  if (v->has_scaling) {
    k_check_scaling<<<std::max(1, std::min((nc + 255) / 256, 132)), 256, 0, s>>>(v->d_center, v->d_scale, nc, sc);
    count_launch();
  }
  BSG_TRY(v->s_dig1.ensure((size_t)stride * 8));
  uint8_t *dig = v->s_dig1.as<uint8_t>();
  k_digits_rows<<<(int)std::min<int64_t>((stride + 255) / 256, 1184), 256, 0, s>>>(Q, n, (int)stride, sc, dig);
  count_launch();
  DArgs a;
  a.V = h->dosV;
  a.stride = stride;
  a.lines = v->d_col;
  a.nlines = nc;
  a.nchunks = (int)(stride / DCH);
  a.dig = dig;
  const int ngroups = (nc + 32 * DW - 1) / (32 * DW);
  int nsm = 132;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, h->device);
  const int lo = (a.nchunks + DMAX_CHUNKS - 1) / DMAX_CHUNKS;
  int ks = std::max(lo, std::min(std::max(1, a.nchunks / 16), (8 * nsm + ngroups - 1) / ngroups));
  const int force = env_int("BSG_DMV_KS", 0);
  if (force > 0) ks = std::max(lo, force);
  a.chunks_per_split = (a.nchunks + ks - 1) / ks;
  a.ksplit = (a.nchunks + a.chunks_per_split - 1) / a.chunks_per_split;
  BSG_TRY(v->s_part.ensure((size_t)std::max(nc, 1) * 16 * sizeof(long long)));
  a.part = v->s_part.as<long long>();
  BSG_CUDA(cudaMemsetAsync(a.part, 0, (size_t)nc * 16 * sizeof(long long), s));
  const int items = ngroups * a.ksplit;
  k_dmv<<<std::max(1, std::min(items, 4 * nsm)), DW * 32, 0, s>>>(a);
  k_finish_dcprod<<<(nc + 255) / 256, 256, 0, s>>>(a.part, nc, sc, v->has_scaling ? v->d_center : nullptr, v->d_scale,
                                                   (double)h->dos_scale, out_dev);
  count_launch(2);
  if (h->dosNaTotal) {
    BSG_TRY(v->s_q1.ensure((size_t)h->m));
    uint8_t *bad = v->s_q1.as<uint8_t>();
    BSG_CUDA(cudaMemsetAsync(bad, 0, (size_t)h->m, s));
    k_na_lines<<<(int)std::min<long long>((h->dosNaTotal + 255) / 256, 132 * 16), 256, 0, s>>>(h->dosNa, h->dosNaTotal,
                                                                                             v->d_rowsel, bad);
    k_na_cols<<<(nc + 255) / 256, 256, 0, s>>>(bad, v->d_col, nc, out_dev);
    count_launch(2);
  }
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int fbm_proj_literal(bsg_view *v, const double *d_V, int K, double *d_XV, double *d_rss, uint8_t *d_na, cudaStream_t s) {
  using namespace dos;
  bsg_bed *h = v->h;
  const double *c = v->has_scaling ? v->d_center : nullptr, *sc = v->has_scaling ? v->d_scale : nullptr;
  if (v->nr == 0) return BSG_OK;
  const int grid = (v->nr + 127) / 128;
  if (h->fbm_generic)
    k_proj_literal<true><<<grid, 128, 0, s>>>(h->raw, h->n, h->d_code, v->d_row, v->nr, v->d_col, v->nc, c, sc, d_V, K, d_XV,
                                             d_rss, d_na);
  else
    k_proj_literal<false><<<grid, 128, 0, s>>>(h->A, h->strideA, nullptr, v->d_row, v->nr, v->d_col, v->nc, c, sc, d_V, K,
                                              d_XV, d_rss, d_na);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int fbm_nan_rows(const uint8_t *d_na, int nr, int K, double *d_XV, cudaStream_t s) {
  if (nr == 0 || K == 0) return BSG_OK;
  dos::k_nan_rows<<<(nr + 255) / 256, 256, 0, s>>>(d_na, nr, K, d_XV);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

int dosage_literal(bsg_view *v, bool cprod, const double *x_dev, double *out_dev, cudaStream_t s) {
  using namespace dos;
  bsg_bed *h = v->h;
  const double *c = v->has_scaling ? v->d_center : nullptr, *sc = v->has_scaling ? v->d_scale : nullptr;
  if (cprod) {
    if (v->nc > 0)
      k_lit_cprod<<<std::min((v->nc + 7) / 8, 132 * 16), 256, 0, s>>>(h->raw, h->n, h->d_code, v->d_row, v->nr, v->d_col,
                                                                       v->nc, c, sc, x_dev, out_dev);
  } else if (v->nr > 0) {
    k_lit_prod<<<(v->nr + 255) / 256, 256, 0, s>>>(h->raw, h->n, h->d_code, v->d_row, v->nr, v->d_col, v->nc, c, sc, x_dev,
                                                   out_dev);
  }
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

}  // namespace bsg

extern "C" {

int bsg_code256_dosage_scale(const double *code256) { return code256 ? bsg::dosage_scale_of(code256) : 0; }

int bsg_dosage_scale(const bsg_bed *h) { return h ? h->dos_scale : 0; }

}  // extern "C"
