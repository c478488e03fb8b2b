// bsg_gramt.cu -- integer Gram tiles fed by TMA, issued as wgmma from two consumer warpgroups (the dense contractions of
// the path: bed_tcrossprodSelf, R/bed-tcrossprodSelf.R:21-52, and the windowed X^T X of snp_cor / snp_ld_scores /
// clumping, src/corr.cpp:11-97).
//
// Expanding the 2-bit codes to bytes inside the Gram kernels keeps SIMT warps writing shared memory for every tile, and
// the tensor pipe waits on them and on the shared-memory port they compete for.  Here the expansion happens ONCE per
// call, into plain K-major uint8 operand buffers in HBM (k_expand_*: HBM-bound, a few milliseconds), and the Gram kernel
// touches no genotype byte with a SIMT instruction:
//
//   * TMA (cp.async.bulk.tensor.2d, tensor maps with the 128-byte swizzle) moves 128 x 128-byte operand boxes into a
//     shared-memory ring; one elected thread per CTA runs it.
//   * a work item is a 256-row A tile and up to four 128-row B tiles; the two CTAs of an item each own one 128-row half
//     of A.  A CTA walks its B tiles in two passes of two: per pass the two consumer warpgroups (64 A rows each) issue
//     wgmma.m64n128k32.s32.u8.u8 against both B tiles, 2 x 64 int32 accumulators per thread in registers.
//   * the four B tiles are, for the GRM, the four base-128 digit slices of the per-SNP weight, and for the correlations
//     four neighbouring column blocks of the band.  Per 128-byte k-block and pass a CTA pulls 16 KB of A and 2 x 16 KB
//     of B for 2 x 2 x 4 MMAs of 64 x 128 x 32.
//   * tiles are launched in super-tile order so that the CTAs running together share operand rows and walk K in step:
//     the re-reads hit L2, not HBM.
//   * integer accumulation is exact; the epilogue either stores the int32 sums of the 128 x 128 sub-tiles
//     (correlations) or folds the slices into K in fp64 (GRM).
#include <cuda.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <vector>

#include "bsg_gram.cuh"
#include "bsg_internal.cuh"

namespace bsg {
namespace gt {

constexpr int BM = 128;   // A rows per CTA (a work item has 256)
constexpr int BN = 128;   // B rows per tile = accumulator width
constexpr int BK = 128;   // bytes (= u8 elements) per k-block: one 128-byte swizzle row
constexpr int A_BYTES = BM * BK, B_BYTES = BN * BK;
constexpr int NBMAX = 4;  // B tiles per work item
constexpr int NBP = 2;    // B tiles per pass
constexpr int MMA_WARPS = 8;
constexpr int THREADS = (MMA_WARPS + 4) * 32;  // warps 0..7 two consumer warpgroups, warps 8..11 the TMA warpgroup
// registers per thread after the split: the producer warpgroup needs few, the accumulators (2 x 64 per thread) many
constexpr int PROD_REGS = 40, MMA_REGS = 232;
constexpr int STAGE = A_BYTES + NBP * B_BYTES;
constexpr int NST = 4;
constexpr int SMEM = NST * STAGE + 1024 /* alignment slack */ + 256 /* barriers */;

struct GtTile {
  int arow;             // first row of the 256-row A tile in the A tensor map
  int brow[NBMAX];      // first row of B tile b in the B tensor map (< 0: tile unused)
  int i0, j0;           // GRM: first output row / column
  long long out[2][NBMAX];  // sums epilogue: int32 offset of the 128 x 128 sub-tile (half, b), < 0 = discard
};

struct GtArgs {
  const GtTile *tiles;
  int nkb;             // k-blocks per tile
  int *sums;           // EPI 0
  double *K;           // EPI 1: K[j * ldk + i] += sum_b scale[b] * S_b[i][j] for i >= j
  int64_t ldk;
  int nlines;
  double scale[NBMAX];
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}" ::"r"(bar),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void tma_load(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// K-major operand, 128-byte swizzle: 8-row groups 1024 B apart (SBO), LBO unused
__device__ __forceinline__ uint64_t sw128_desc(uint32_t saddr) { return wg::desc(saddr, 16, 1024, 1); }

// B tiles of pass p, in the order the GRM epilogue wants them: the most significant digit slices first
__device__ __forceinline__ int pass_tile(int p, int q) { return NBMAX - NBP * (p + 1) + q; }

template <int EPI>
__global__ void __launch_bounds__(THREADS, 1)
    k_gramt(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB, const GtArgs a) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t sbase = (smem_u32(smem_raw) + 1023u) & ~1023u;  // swizzle atoms are 1024-byte aligned
  const uint32_t bars = sbase + NST * STAGE;                      // full[s] +8s | empty[s] +8(NST+s)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int half = blockIdx.x & 1;
  const GtTile &t = a.tiles[blockIdx.x >> 1];

  if (threadIdx.x == 0) {
    for (int s = 0; s < NST; s++) {
      mbar_init(bars + 8 * s, 1);                   // the producer's arrive.expect_tx
      mbar_init(bars + 8 * (NST + s), MMA_WARPS);   // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp >= MMA_WARPS) {
    // ================= TMA producer =================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    if (warp == MMA_WARPS && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int p = 0; p < NBMAX / NBP; p++) {
        int nact = 0;
#pragma unroll
        for (int q = 0; q < NBP; q++) nact += t.brow[pass_tile(p, q)] >= 0 ? 1 : 0;
        if (nact == 0) continue;
        for (int kb = 0; kb < a.nkb; kb++) {
          mbar_wait(bars + 8 * (NST + stage), phase ^ 1);
          const uint32_t full = bars + 8 * stage, dst = sbase + stage * STAGE;
          mbar_expect_tx(full, (uint32_t)(A_BYTES + nact * B_BYTES));
          tma_load(dst, &tmA, full, kb * BK, t.arow + half * BM);
#pragma unroll
          for (int q = 0; q < NBP; q++) {
            const int br = t.brow[pass_tile(p, q)];
            if (br >= 0) tma_load(dst + A_BYTES + q * B_BYTES, &tmB, full, kb * BK, br);
          }
          if (++stage == NST) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ================= consumer warpgroups: rows [64 cw, 64 cw + 64) of this CTA's 128 =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(MMA_REGS));
    const int cw = warp >> 2, wq = warp & 3;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t d[NBP][64];
    for (int p = 0; p < NBMAX / NBP; p++) {
      bool act[NBP];
      int nact = 0;
#pragma unroll
      for (int q = 0; q < NBP; q++) {
        act[q] = t.brow[pass_tile(p, q)] >= 0;
        nact += act[q] ? 1 : 0;
      }
      if (nact == 0) continue;
      int prev = -1;
      for (int kb = 0; kb < a.nkb; kb++) {
        mbar_wait(bars + 8 * stage, phase);
        wg::fence();
        const uint32_t a0 = sbase + stage * STAGE + cw * 64 * BK;
#pragma unroll
        for (int q = 0; q < NBP; q++) {
          if (!act[q]) continue;
          const uint32_t b0 = sbase + stage * STAGE + A_BYTES + q * B_BYTES;
#pragma unroll
          for (int k4 = 0; k4 < BK / 32; k4++)
            wg::mma_u8_n128(d[q], sw128_desc(a0 + k4 * 32), sw128_desc(b0 + k4 * 32), (kb | k4) ? 1u : 0u);
        }
        wg::commit();
        wg::wait<1>();  // the stage before this one has been read
        if (prev >= 0 && lane == 0) mbar_arrive(bars + 8 * (NST + prev));
        prev = stage;
        if (++stage == NST) {
          stage = 0;
          phase ^= 1;
        }
      }
      wg::wait<0>();
      if (prev >= 0 && lane == 0) mbar_arrive(bars + 8 * (NST + prev));

      if (EPI == 0) {
#pragma unroll
        for (int q = 0; q < NBP; q++) {
          const long long off = t.out[half][pass_tile(p, q)];
          if (!act[q] || off < 0) continue;  // warp-uniform
          int *dst = a.sums + off;
#pragma unroll
          for (int j = 0; j < 64; j += 2) {
            const int r = 64 * cw + wg::acc_row(wq, lane, j), c = wg::acc_col(lane, j);
            *reinterpret_cast<int2 *>(dst + (int64_t)r * BN + c) = make_int2((int)d[q][j], (int)d[q][j + 1]);
          }
        }
      } else {
        const double s0 = act[0] ? a.scale[pass_tile(p, 0)] : 0.0, s1 = act[1] ? a.scale[pass_tile(p, 1)] : 0.0;
#pragma unroll
        for (int j = 0; j < 64; j++) {
          const int i = t.i0 + half * BM + 64 * cw + wg::acc_row(wq, lane, j), jj = t.j0 + wg::acc_col(lane, j);
          // the two slices of this pass (the more significant pair is folded into K first); the sum is exact in fp64:
          // both terms are integers below 2^28 at power-of-two scales 2^7 apart
          const double v = (act[0] ? s0 * (double)(int)d[0][j] : 0.0) + (act[1] ? s1 * (double)(int)d[1][j] : 0.0);
          if (i < a.nlines && jj < a.nlines && i >= jj) a.K[(int64_t)jj * a.ldk + i] += v;
        }
      }
    }
  }
}

// ---- expansion of the packed 2-bit lines to K-major uint8 operands ------------------------------------------------
// plane: 0 = a (genotype, missing -> 0), 1 = n (missing indicator), 2 = b (valid indicator), 3 = h ([genotype == 2]),
//        4 = raw code (lines known to hold no missing value)
__device__ __forceinline__ uint32_t plane_of(uint32_t x, int plane) {
  const uint32_t n = x & (x >> 1) & 0x55555555u;
  if (plane == 4) return x;
  if (plane == 1) return n;
  if (plane == 2) return ~n & 0x55555555u;
  const uint32_t av = x & ~(n | (n << 1));
  return plane == 0 ? av : ((av >> 1) & 0x55555555u);
}
// the 16 codes of a packed word -> 16 bytes in code order
__device__ __forceinline__ uint4 bytes_of(uint32_t x) {
  uint32_t c[4];  // class c: byte r = code 4r + c
#pragma unroll
  for (int k = 0; k < 4; k++) c[k] = (x >> (2 * k)) & 0x03030303u;
  // transpose classes -> natural order: out word w holds codes 4w .. 4w+3 = (c0.byte w, c1.byte w, c2.byte w, c3.byte w)
  uint4 o;
  uint32_t *ow = &o.x;
#pragma unroll
  for (int w = 0; w < 4; w++)
    ow[w] = ((c[0] >> (8 * w)) & 0xFFu) | (((c[1] >> (8 * w)) & 0xFFu) << 8) | (((c[2] >> (8 * w)) & 0xFFu) << 16) |
            (((c[3] >> (8 * w)) & 0xFFu) << 24);
  return o;
}

// out[(row_off + line) * pitch + k] = plane(code(line, k0 + k)), k < pitch (zero beyond the line's packed bytes)
__global__ void k_expand_plane(const uint8_t *__restrict__ P, int64_t stride, int nlines, int64_t k0, int64_t pitch, int plane,
                               uint8_t *__restrict__ out, int64_t row_off) {
  const int64_t wpl = pitch / 16;
  const int64_t total = (int64_t)nlines * wpl;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = t / wpl, w = t - l * wpl;
    const int64_t byte = (k0 >> 2) + 4 * w;
    uint32_t x = 0;
    bool inside = byte + 4 <= stride;
    if (inside) x = *reinterpret_cast<const uint32_t *>(P + l * stride + byte);
    uint4 o = make_uint4(0, 0, 0, 0);
    if (inside) o = bytes_of(plane_of(x, plane));
    *reinterpret_cast<uint4 *>(out + (row_off + l) * pitch + 16 * w) = o;
  }
}

// out[(s * lines_pad + line) * pitch + k] = plane(code(line, k0 + k)) * digit_s[k0 + k]; digits beyond `klen` are 0
__global__ void k_expand_weighted(const uint8_t *__restrict__ P, int64_t stride, int nlines, int64_t lines_pad, int64_t k0,
                                  int64_t klen, int64_t pitch, int plane, const uint8_t *__restrict__ dig, int64_t dig_stride,
                                  int nslices, uint8_t *__restrict__ out) {
  const int64_t wpl = pitch / 16;
  const int64_t total = (int64_t)nlines * wpl;
  for (int64_t t = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; t < total; t += (int64_t)gridDim.x * blockDim.x) {
    const int64_t l = t / wpl, w = t - l * wpl;
    const int64_t byte = (k0 >> 2) + 4 * w;
    uint4 codes = make_uint4(0, 0, 0, 0);
    if (byte + 4 <= stride) codes = bytes_of(plane_of(*reinterpret_cast<const uint32_t *>(P + l * stride + byte), plane));
    const bool have = 16 * w < klen;  // klen is a multiple of 16 except at the very end, where the digits are zero-padded
    for (int s = 0; s < nslices; s++) {
      uint4 o = make_uint4(0, 0, 0, 0);
      if (have) {
        const uint4 d = *reinterpret_cast<const uint4 *>(dig + (int64_t)s * dig_stride + k0 + 16 * w);
        const uint32_t cw[4] = {codes.x, codes.y, codes.z, codes.w}, dw[4] = {d.x, d.y, d.z, d.w};
        uint32_t ow[4];
#pragma unroll
        for (int q = 0; q < 4; q++) {  // per byte: code in {0,1,2} times digit <= 127 -> (bit0 ? d : 0) + (bit1 ? 2d : 0) <= 254
          const uint32_t m1 = (cw[q] & 0x01010101u) * 0xFFu, m2 = ((cw[q] >> 1) & 0x01010101u) * 0xFFu;
          ow[q] = (m1 & dw[q]) | (m2 & (dw[q] << 1));
        }
        o = make_uint4(ow[0], ow[1], ow[2], ow[3]);
      }
      *reinterpret_cast<uint4 *>(out + ((int64_t)s * lines_pad + l) * pitch + 16 * w) = o;
    }
  }
}

// digits in plain order: dig[s * dig_stride + k] = digit s (dbits wide) of rint(W[k] * 2^e); zero outside [lo, hi)
__global__ void k_weight_digits_plain(const double *__restrict__ W, int64_t lo, int64_t hi, int64_t dig_stride, int nslices, int e,
                                      int dbits, uint8_t *__restrict__ dig) {
  for (int64_t k = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; k < dig_stride; k += (int64_t)gridDim.x * blockDim.x) {
    unsigned long long v = 0;
    if (k >= lo && k < hi) v = (unsigned long long)__double2ll_rn(scalbn(W[k], e));
    for (int s = 0; s < nslices; s++) {
      dig[(int64_t)s * dig_stride + k] = (uint8_t)(v & ((1ull << dbits) - 1ull));
      v >>= dbits;
    }
  }
}

// ---- host side ---------------------------------------------------------------------------------------------------------
template <int EPI>
static int launch(const CUtensorMap &mA, const CUtensorMap &mB, const GtArgs &a, int ntiles, cudaStream_t s) {
  BSG_CUDA(cudaFuncSetAttribute(k_gramt<EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM));
  k_gramt<EPI><<<2 * ntiles, THREADS, SMEM, s>>>(mA, mB, a);
  count_launch();
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}

static int grid_cap(int64_t work) { return (int)std::max<int64_t>(1, std::min<int64_t>((work + 255) / 256, 132 * 32)); }

}  // namespace gt

// ---- tensor maps ---------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                             const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeFn encode_fn() {
  static EncodeFn fn = nullptr;
  if (!fn) {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) == cudaSuccess && qr == cudaDriverEntryPointSuccess)
      fn = (EncodeFn)p;
  }
  return fn;
}
// rows x pitch bytes, row-major, box = 128 bytes x box_rows rows, 128-byte swizzle, L2 promotion to 256 B; boxes
// reaching past `rows` or `pitch` read as zero.  Shared by the Gram tiles and k_pmvT (bsg_pmv.cu).
int make_map(CUtensorMap *m, const uint8_t *base, int64_t rows, int64_t pitch, int box_rows) {
  EncodeFn f = encode_fn();
  if (!f) return fail(BSG_ERR_CUDA, "cuTensorMapEncodeTiled is not available from this driver.");
  cuuint64_t gdim[2] = {(cuuint64_t)pitch, (cuuint64_t)rows}, gstr[1] = {(cuuint64_t)pitch};
  cuuint32_t box[2] = {128, (cuuint32_t)box_rows}, estr[2] = {1, 1};
  CUresult r = f(m, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, (void *)base, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                 CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(BSG_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d).", (int)r);
  return BSG_OK;
}

bool gramt_enabled() {
  static int on = -1;
  if (on < 0) {
    const char *ev = getenv("BSG_GRAM_TMA");
    on = (ev && ev[0] == '0') ? 0 : 1;
  }
  return on != 0;
}

// ---------------------------------------------------------------------------------------------------------------------------
// GRM: K (pre-zeroed, nr x nr column-major, filled for i >= j) += sum_k w-weighted integer Grams of the packed sample-major
// lines P.  Ws = {W1, W2', W3} (device, length nc), wmax their maxima over [klo, khi), na[i] = 1 if line i holds a missing
// value.  Only the weights of the columns [klo, khi) (one weight class, tcrossprod_impl) are quantised; the contraction runs
// over that range rounded out to whole 128-code k-blocks, where the digits of the neighbouring columns are zero.
// Columns are processed in blocks of at most KBLK codes: expand -> one launch per plane product -> K accumulates in fp64.
// ---------------------------------------------------------------------------------------------------------------------------
int gramt_grm(const uint8_t *P, int64_t stride, int nr, int nc, const double *const Ws[3], const double wmax[3],
              const uint8_t *na, int nslices, double *K, int64_t ldk, int device, cudaStream_t s, int64_t klo, int64_t khi) {
  using namespace gt;
  if (nslices > NBMAX) nslices = NBMAX;
  const int dbits = 7;
  const int64_t KBLK = 262144;  // 2 * 254 * 262144 < 2^31: int32 accumulators cannot overflow within a block
  const int64_t kb0 = klo / BK * BK, kb1 = std::min<int64_t>(nc, round_up(khi, BK));
  const int64_t kblk = std::min<int64_t>(KBLK, round_up(kb1 - kb0, BK));
  const int64_t lines_pad = round_up(nr, 256);
  bool any_na = false;
  for (int i = 0; i < nr; i++) any_na |= na[i] != 0;
  // buffers: A planes (a, n) and the weighted B of the current product
  uint8_t *Aa = nullptr, *An = nullptr, *Bw = nullptr, *dig[3] = {nullptr, nullptr, nullptr};
  GtTile *d_tiles = nullptr;
  struct Free {
    std::vector<void *> p;
    ~Free() {
      for (void *q : p)
        if (q) cudaFree(q);
    }
  } fr;
  auto alloc = [&](void **q, size_t bytes) -> int {
    cudaError_t e = pool_alloc(q, bytes, device, s);
    if (e != cudaSuccess) return cuda_fail(e, "cudaMalloc(Gram operand buffers)");
    fr.p.push_back(*q);
    return BSG_OK;
  };
  BSG_TRY(alloc((void **)&Aa, (size_t)lines_pad * kblk));
  if (any_na) BSG_TRY(alloc((void **)&An, (size_t)lines_pad * kblk));
  BSG_TRY(alloc((void **)&Bw, (size_t)nslices * lines_pad * kblk));
  const int64_t dig_stride = round_up(nc, 256) + 256;
  double scale[3][NBMAX];
  for (int wv = 0; wv < (any_na ? 3 : 1); wv++) {
    BSG_TRY(alloc((void **)&dig[wv], (size_t)nslices * dig_stride));
    int ex = 0;
    if (wmax[wv] > 0) frexp(wmax[wv], &ex);
    const int e = dbits * nslices - 1 - ex;
    k_weight_digits_plain<<<grid_cap(dig_stride), 256, 0, s>>>(Ws[wv], klo, khi, dig_stride, nslices, e, dbits, dig[wv]);
    count_launch();
    for (int sl = 0; sl < NBMAX; sl++) scale[wv][sl] = sl < nslices ? ldexp(1.0, dbits * sl - e) : 0.0;
  }
  // tiles of the lower triangle (256 x 128), in super-tile order: blocks of 8 x 8 tiles share their operand rows in L2
  const int nI = (nr + 255) / 256, nJ = (nr + 127) / 128;
  std::vector<uint8_t> na_j(nJ, 0);
  for (int i = 0; i < nr; i++) na_j[i / 128] |= na[i];
  std::vector<GtTile> tiles_all, tiles_na;
  const int SI = 8, SJ = 8;
  for (int I0 = 0; I0 < nI; I0 += SI)
    for (int J0 = 0; J0 < nJ; J0 += SJ)
      for (int I = I0; I < std::min(nI, I0 + SI); I++)
        for (int J = J0; J < std::min(nJ, J0 + SJ); J++) {
          if (J * 128 > I * 256 + 255) continue;  // entirely above the diagonal
          GtTile t;
          memset(&t, 0, sizeof t);
          t.arow = I * 256;
          for (int b = 0; b < NBMAX; b++) t.brow[b] = b < nslices ? (int)(b * lines_pad + J * 128) : -1;
          t.i0 = I * 256;
          t.j0 = J * 128;
          tiles_all.push_back(t);
          const bool na_i = na_j[std::min(nJ - 1, 2 * I)] || na_j[std::min(nJ - 1, 2 * I + 1)];
          if (na_i || na_j[J]) tiles_na.push_back(t);
        }
  const size_t nt_all = tiles_all.size(), nt_na = tiles_na.size();
  BSG_TRY(alloc((void **)&d_tiles, (nt_all + nt_na) * sizeof(GtTile)));
  BSG_CUDA(cudaMemcpyAsync(d_tiles, tiles_all.data(), nt_all * sizeof(GtTile), cudaMemcpyHostToDevice, s));
  if (nt_na) BSG_CUDA(cudaMemcpyAsync(d_tiles + nt_all, tiles_na.data(), nt_na * sizeof(GtTile), cudaMemcpyHostToDevice, s));
  BSG_CUDA(cudaStreamSynchronize(s));  // host vectors go out of scope at return; also orders the tile upload

  for (int64_t k0 = kb0; k0 < kb1; k0 += kblk) {
    const int64_t klen = std::min<int64_t>(kblk, kb1 - k0);
    const int64_t pitch = round_up(klen, BK);
    CUtensorMap mAa, mAn, mB;
    BSG_TRY(make_map(&mAa, Aa, lines_pad, pitch, BM));
    if (any_na) BSG_TRY(make_map(&mAn, An, lines_pad, pitch, BM));
    BSG_TRY(make_map(&mB, Bw, (int64_t)nslices * lines_pad, pitch, BM));
    k_expand_plane<<<grid_cap((int64_t)nr * (pitch / 16)), 256, 0, s>>>(P, stride, nr, k0, pitch, any_na ? 0 : 4, Aa, 0);
    if (any_na) k_expand_plane<<<grid_cap((int64_t)nr * (pitch / 16)), 256, 0, s>>>(P, stride, nr, k0, pitch, 1, An, 0);
    count_launch(any_na ? 2 : 1);
    GtArgs a;
    memset(&a, 0, sizeof a);
    a.nkb = (int)(pitch / BK);
    a.K = K;
    a.ldk = ldk;
    a.nlines = nr;
    // products: aa (W1) on every tile; an, na (W2'), nn (W3) on tiles touching a line with missing values
    const int nprod = any_na ? 4 : 1;
    for (int prod = 0; prod < nprod; prod++) {
      const int wsel = prod == 0 ? 0 : (prod == 3 ? 2 : 1);
      const bool a_is_n = prod >= 2, b_is_n = prod == 1 || prod == 3;
      k_expand_weighted<<<grid_cap((int64_t)nr * (pitch / 16)), 256, 0, s>>>(P, stride, nr, lines_pad, k0, klen, pitch,
                                                                             b_is_n ? 1 : (any_na ? 0 : 4), dig[wsel], dig_stride,
                                                                             nslices, Bw);
      count_launch();
      for (int b = 0; b < NBMAX; b++) a.scale[b] = scale[wsel][b];
      a.tiles = prod == 0 ? d_tiles : d_tiles + nt_all;
      const int nt = prod == 0 ? (int)nt_all : (int)nt_na;
      if (nt > 0) BSG_TRY((launch<1>(a_is_n ? mAn : mAa, mB, a, nt, s)));
    }
  }
  BSG_CUDA(cudaStreamSynchronize(s));  // operand buffers are freed on return
  return BSG_OK;
}

// ---------------------------------------------------------------------------------------------------------------------------
// Correlation tiles: sums[tile.out + prod * 128 * 128 + row * 128 + col] for the 128 x 128 tiles of `tiles` (host copy of the
// list the epilogue kernels use; mode 0: product aa only, mode 1: the six plane products).  M = packed SNP-major lines.
// Returns BSG_OK with *done = false when the operand buffers do not fit (the caller then runs the in-kernel-expansion path).
// ---------------------------------------------------------------------------------------------------------------------------
int gramt_cor(const uint8_t *M, int64_t stride, int nlines, const gram::Tile *tiles, int ntiles, int *d_sums, int device,
              cudaStream_t s, bool *done) {
  using namespace gt;
  *done = false;
  if (ntiles == 0) {
    *done = true;
    return BSG_OK;
  }
  bool any_na = false;
  int lmin = nlines, lmax = 0;
  for (int t = 0; t < ntiles; t++) {
    any_na |= tiles[t].mode != 0;
    lmin = std::min(lmin, std::min(tiles[t].i0, tiles[t].j0));
    lmax = std::max(lmax, std::max(tiles[t].i0, tiles[t].j0) + 128);
  }
  lmin = std::max(0, lmin) / 256 * 256;
  lmax = std::min(nlines, lmax);
  const int nl = lmax - lmin;
  const int64_t lines_pad = round_up(nl, 256);
  const int64_t pitch = stride * 4;  // every code slot of the line, pads included (they count as valid on both sides)
  const int nplanes = any_na ? 3 : 1;  // a, b, h (or the raw codes alone)
  const size_t need = (size_t)nplanes * lines_pad * pitch;
  uint8_t *E = nullptr;
  GtTile *d_gt = nullptr;
  if (pool_alloc((void **)&E, need, device, s) != cudaSuccess) {  // not enough room: the caller falls back
    cudaGetLastError();
    return BSG_OK;
  }
  struct Free {
    void *a, *b;
    ~Free() {
      if (a) cudaFree(a);
      if (b) cudaFree(b);
    }
  } frg{E, nullptr};
  const int plane_ids[3] = {any_na ? 0 : 4, 2, 3};
  for (int p = 0; p < nplanes; p++) {
    k_expand_plane<<<grid_cap((int64_t)nl * (pitch / 16)), 256, 0, s>>>(M + (int64_t)lmin * stride, stride, nl, 0, pitch, plane_ids[p],
                                                                        E, (int64_t)p * lines_pad);
    count_launch();
  }
  CUtensorMap mE;  // A and B tiles are both rows of the expanded planes
  BSG_TRY(make_map(&mE, E, (int64_t)nplanes * lines_pad, pitch, BM));
  // group the 128 x 128 tiles: pairs of row blocks (256 rows) x runs of up to four column blocks.  The list is ordered by
  // row block, then column block (bsg_cor.cu), so a row block's tiles are consecutive.
  struct Key { int i0, j0, idx; };
  std::vector<GtTile> gts[6];
  {
    // index tiles by (row block, column block)
    std::vector<Key> keys(ntiles);
    for (int t = 0; t < ntiles; t++) keys[t] = Key{tiles[t].i0, tiles[t].j0, t};
    std::sort(keys.begin(), keys.end(), [](const Key &x, const Key &y) { return x.i0 != y.i0 ? x.i0 < y.i0 : x.j0 < y.j0; });
    size_t p0 = 0;
    while (p0 < keys.size()) {
      const int ipair = keys[p0].i0 / 256 * 256;  // rows [ipair, ipair + 256)
      size_t p1 = p0;
      while (p1 < keys.size() && keys[p1].i0 < ipair + 256) p1++;
      // column blocks present in either half
      std::vector<int> cols;
      for (size_t q = p0; q < p1; q++) cols.push_back(keys[q].j0);
      std::sort(cols.begin(), cols.end());
      cols.erase(std::unique(cols.begin(), cols.end()), cols.end());
      auto find = [&](int i0, int j0) -> int {
        for (size_t q = p0; q < p1; q++)
          if (keys[q].i0 == i0 && keys[q].j0 == j0) return keys[q].idx;
        return -1;
      };
      for (size_t c0 = 0; c0 < cols.size(); c0 += NBMAX) {
        for (int prod = 0; prod < (any_na ? 6 : 1); prod++) {
          // planes per product: A = {a, b, a, b, h, b}, B = {a, b, b, a, b, h}  (plane buffer index: a 0, b 1, h 2)
          const int pa = (0x121010 >> (4 * prod)) & 0xF, pb = (0x210110 >> (4 * prod)) & 0xF;
          GtTile g;
          memset(&g, 0, sizeof g);
          g.arow = (int)(pa * lines_pad + (ipair - lmin));
          bool any = false;
          for (int b = 0; b < NBMAX; b++) {
            g.brow[b] = -1;
            g.out[0][b] = g.out[1][b] = -1;
            if (c0 + b >= cols.size()) continue;
            const int j0 = cols[c0 + b];
            for (int half = 0; half < 2; half++) {
              const int ti = find(ipair + 128 * half, j0);
              if (ti < 0) continue;
              if (prod > 0 && tiles[ti].mode == 0) continue;  // missing-free tile: xySum is the only pair-specific sum
              g.out[half][b] = tiles[ti].out + (long long)prod * 128 * 128;
              g.brow[b] = (int)(pb * lines_pad + (j0 - lmin));
              any = true;
            }
          }
          if (any) gts[prod].push_back(g);
        }
      }
      p0 = p1;
    }
  }
  size_t ngt = 0;
  for (int p = 0; p < 6; p++) ngt += gts[p].size();
  BSG_CUDA(cudaMalloc((void **)&d_gt, ngt * sizeof(GtTile)));
  frg.b = d_gt;
  size_t off = 0;
  for (int p = 0; p < 6; p++) {
    if (gts[p].empty()) continue;
    BSG_CUDA(cudaMemcpyAsync(d_gt + off, gts[p].data(), gts[p].size() * sizeof(GtTile), cudaMemcpyHostToDevice, s));
    GtArgs a;
    memset(&a, 0, sizeof a);
    a.tiles = d_gt + off;
    a.nkb = (int)(pitch / BK);
    a.sums = d_sums;
    BSG_TRY((launch<0>(mE, mE, a, (int)gts[p].size(), s)));
    off += gts[p].size();
  }
  BSG_CUDA(cudaStreamSynchronize(s));  // host tile vectors and the operand buffer are released on return
  *done = true;
  return BSG_OK;
}

}  // namespace bsg
