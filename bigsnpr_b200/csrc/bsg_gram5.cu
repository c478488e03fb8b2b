// bsg_gram5.cu -- the integer Gram tile on the Hopper tensor cores (wgmma, register accumulators).
//
//   S[i][j] = sum_k code(i, k) * code(j, k)      for a 128 x 128 tile of lines, exact int32
//
// Used for the windowed correlations when the tile holds no missing value (only xySum is pair specific then,
// src/corr.cpp:58-75); tiles with missing values take k_wgram5<1> below (six plane products, same pipeline).
//
// Pipeline per CTA (one 128 x 128 tile, whole contraction range):
//   8 producer warps : stream the packed lines (2 x LDG.128 = 128 codes per line and stage, register prefetch),
//                      expand 2-bit codes to bytes with the class masks (w >> 2c) & 0x03030303 -- any fixed
//                      permutation of k inside a 16-byte row is fine for a Gram product because both operands
//                      use the same one -- and STS.128 them into shared memory in the wgmma K-major
//                      no-swizzle layout: core matrix = 8 rows x 16 B, SBO = 128 B between 8-row groups,
//                      LBO = 2048 B between core matrices along K; fence.proxy.async + mbarrier arrive.
//   2 consumer warpgroups: wait for the stage, each issues 4 x wgmma.m64n128k32.s32.u8.u8 on its 64 rows of the
//                      tile (int32 accumulators in registers), and hands the stage back once those MMAs completed;
//                      the tile sums are stored from the registers.
#include <stdint.h>
#include <string.h>

#include "bsg_gram.cuh"
#include "bsg_internal.cuh"

namespace bsg {
namespace gram5 {

constexpr int T5M = 128, T5N = 128;      // tile of line pairs
constexpr int KSTAGE = 128;              // codes per line per stage (32 packed bytes) = 4 MMAs of K = 32
constexpr int SBYTES = KSTAGE / 4;       // packed bytes per line per stage
constexpr int NW = KSTAGE / 16;          // packed words (= core matrices along K) per line per stage
constexpr int STAGES = 3;
constexpr int PF = 2;                    // stages of register prefetch per producer thread
constexpr int PROD_WARPS = 8;            // 256 producer threads: thread t expands line t (0..127 A, 128..255 B)
constexpr int MMA_WARPS = 8;             // two consumer warpgroups, 64 tile rows each
// registers per thread after the split (65,536 in all): the consumers hold 64 int32 accumulators each
constexpr int PROD_REGS = 96, MMA_REGS = 160;
constexpr int THREADS = (PROD_WARPS + MMA_WARPS) * 32;
constexpr int OPER_BYTES = 128 * KSTAGE;  // 16 KB per operand and stage
constexpr int STAGE_BYTES = 2 * OPER_BYTES;
constexpr int LBO = 2048, SBO = 128;     // bytes: next core matrix along K / along M
constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 256;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
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
__device__ __forceinline__ void sts128(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}

using Tile5 = gram::Tile;  // {i0, j0, mode, out}: out = offset (int32) of the 128 x 128 sums of this tile

// consumer side of one pass over the contraction: warpgroup cw (0, 1) multiplies rows [64 cw, 64 cw + 64) of the A
// stage by the 128 B rows; each stage is handed back to the producers once the MMAs reading it have completed
__device__ __forceinline__ void consume_pass(uint32_t (&d)[64], uint32_t sbase, uint32_t bar, int nsteps, int cw, int lane,
                                             int &stage, uint32_t &phase) {
  int prev = -1;
  for (int st = 0; st < nsteps; st++) {
    mbar_wait(bar + 8 * stage, phase);
    wg::fence();
    const uint32_t a0 = sbase + stage * STAGE_BYTES + cw * 8 * SBO, b0 = sbase + stage * STAGE_BYTES + OPER_BYTES;
#pragma unroll
    for (int kk = 0; kk < KSTAGE / 32; kk++)
      wg::mma_u8_n128(d, wg::desc(a0 + kk * 2 * LBO, LBO, SBO, 0), wg::desc(b0 + kk * 2 * LBO, LBO, SBO, 0), (st | kk) ? 1u : 0u);
    wg::commit();
    wg::wait<1>();  // the stage before this one has been read
    if (prev >= 0 && lane == 0) mbar_arrive(bar + 8 * (STAGES + prev));
    prev = stage;
    if (++stage == STAGES) {
      stage = 0;
      phase ^= 1;
    }
  }
  wg::wait<0>();
  if (prev >= 0 && lane == 0) mbar_arrive(bar + 8 * (STAGES + prev));
}

__global__ void __launch_bounds__(THREADS, 1) k_gram5(const uint8_t *__restrict__ P, int64_t stride, int nlines,
                                                     int nsteps, const Tile5 *__restrict__ tiles,
                                                     int *__restrict__ sums) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const Tile5 t = tiles[blockIdx.x];
  if (t.mode != 0) return;  // tiles with missing values are done by the six-plane kernel
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar = sbase + STAGES * STAGE_BYTES;  // full[s] +8s, empty[s] +8(STAGES+s)

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar + 8 * s, PROD_WARPS);            // one arrive per producer warp
      mbar_init(bar + 8 * (STAGES + s), MMA_WARPS);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < PROD_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    // ================= producers: packed line -> bytes in the K-major core-matrix layout =================
    const int row = threadIdx.x & 127;         // row of the operand tile
    const int oper = threadIdx.x >> 7;         // 0: A lines (i0 + row), 1: B lines (j0 + row)
    int line = (oper ? t.j0 : t.i0) + row;
    line = min(max(line, 0), nlines - 1);
    const uint8_t *src = P + (int64_t)line * stride;
    // byte offset of this row inside an operand stage: (row / 8) * SBO + (row % 8) * 16; core matrix k16 at + k16 * LBO
    const uint32_t row_off = (uint32_t)oper * OPER_BYTES + (row >> 3) * SBO + (row & 7) * 16;
    // register prefetch ring: PF stages of this line in flight (2 x LDG.128 each)
    uint4 pf[PF][NW / 4];
#pragma unroll
    for (int u = 0; u < PF; u++) {
#pragma unroll
      for (int v = 0; v < NW / 4; v++)
        pf[u][v] = u < nsteps ? *reinterpret_cast<const uint4 *>(src + (int64_t)u * SBYTES + 16 * v) : make_uint4(0, 0, 0, 0);
    }
    int stage = 0;
    uint32_t phase = 0;
    for (int st0 = 0; st0 < nsteps; st0 += PF) {
#pragma unroll
      for (int u = 0; u < PF; u++) {
        const int st = st0 + u;
        if (st >= nsteps) break;
        uint32_t w[NW];
#pragma unroll
        for (int v = 0; v < NW / 4; v++) {
          w[4 * v] = pf[u][v].x; w[4 * v + 1] = pf[u][v].y; w[4 * v + 2] = pf[u][v].z; w[4 * v + 3] = pf[u][v].w;
        }
        if (st + PF < nsteps) {
#pragma unroll
          for (int v = 0; v < NW / 4; v++)
            pf[u][v] = *reinterpret_cast<const uint4 *>(src + (int64_t)(st + PF) * SBYTES + 16 * v);
        }
        mbar_wait(bar + 8 * (STAGES + stage), phase ^ 1);
        const uint32_t dst = sbase + stage * STAGE_BYTES + row_off;
#pragma unroll
        for (int k16 = 0; k16 < NW; k16++) {
          const uint32_t x = w[k16];
          sts128(dst + k16 * LBO, x & 0x03030303u, (x >> 2) & 0x03030303u, (x >> 4) & 0x03030303u, (x >> 6) & 0x03030303u);
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the tensor core
        __syncwarp();
        if (lane == 0) mbar_arrive(bar + 8 * stage);
        if (++stage == STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    // ================= two consumer warpgroups: MMAs, then the int32 sums straight from the registers =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(MMA_REGS));
    const int cw = (warp - PROD_WARPS) >> 2, wq = warp & 3;
    uint32_t d[64];
    int stage = 0;
    uint32_t phase = 0;
    consume_pass(d, sbase, bar, nsteps, cw, lane, stage, phase);
    int *out = sums + t.out;
#pragma unroll
    for (int j = 0; j < 64; j += 2) {
      const int r = 64 * cw + wg::acc_row(wq, lane, j), c = wg::acc_col(lane, j);
      *reinterpret_cast<int2 *>(out + (int64_t)r * T5N + c) = make_int2((int)d[j], (int)d[j + 1]);
    }
  }
}

}  // namespace gram5

// ===================================================================================================
// Weighted Gram on wgmma for bed_tcrossprodSelf:  K[i][j] += scale * sum_k fA(code(i,k)) * fB(code(j,k)) * d_k
// One CTA per 128 x 128 tile of the lower triangle; passes = weight slices x plane products, each pass a
// full sweep over k into the consumers' register accumulators, then K += scale * S from those registers.  The
// producers run ahead into the next pass's stages while the consumers fold the previous one into K.
//   warps 0..7   producers (as k_gram5; the B operand bytes are code * digit: ((x & 1) ? d : 0) | ((x & 2) ? 2d : 0))
//   warps 8..15  two consumer warpgroups (wgmma + epilogue, 64 tile rows each)
// ===================================================================================================
namespace wg5 {
using namespace gram5;

constexpr int W5_THREADS = THREADS;
constexpr int W5_SMEM_BYTES = STAGES * STAGE_BYTES + 256;

struct W5Tile {
  int i0, j0, mode;  // mode 0: product aa only; 1: aa, an, na, nn
};

struct W5Args {
  const uint8_t *P;
  int64_t stride;
  int nlines, nsteps, nslices;
  const gram::Tile *ctiles;  // KIND 1: correlation tiles {i0, j0, mode, out}
  int *sums;                 // KIND 1: [tile.out + prod * 128 * 128 + row * 128 + col]
  const uint8_t *dig[3];  // W1, W2', W3 digits: [nslices][nwords * 16], 16 bytes per packed word in class order [c][r]
  int64_t dig_stride;     // bytes per slice
  double scale[3][10];
  const W5Tile *tiles;
  double *K;
  int64_t ldk;
};

// plane of the A / B operand per product: 0 = genotype (missing -> 0), 1 = missing indicator
__device__ __forceinline__ void pass_info(int mode, int nslices, int pass, int &prod, int &slice, int &wsel) {
  if (mode == 0) {
    prod = 0;
    slice = nslices - 1 - pass;
  } else {
    slice = nslices - 1 - pass / 4;
    prod = pass & 3;
  }
  wsel = prod == 0 ? 0 : (prod == 3 ? 2 : 1);  // aa -> W1 ; an, na -> W2' ; nn -> W3
}

// planes of the pairwise-complete statistics (KIND 1), products in the order k_cor_from_sums reads them:
// aa (xySum), bb (nona), ab (xSum), ba (ySum), hb, bh  with a = genotype (NA -> 0), b = valid, h = [genotype == 2]
__device__ __forceinline__ uint32_t cor_plane(uint32_t x, int pl) {
  const uint32_t n = x & (x >> 1) & 0x55555555u;
  const uint32_t av = x & ~(n | (n << 1));
  return pl == 0 ? av : (pl == 1 ? (~n & 0x55555555u) : ((av >> 1) & 0x55555555u));
}

template <int KIND>
__global__ void __launch_bounds__(W5_THREADS, 1) k_wgram5(const W5Args a) {
  extern __shared__ __align__(1024) uint8_t smem[];
  W5Tile t;
  long long out_off = 0;
  if (KIND == 0) {
    t = a.tiles[blockIdx.x];
  } else {
    const gram::Tile ct = a.ctiles[blockIdx.x];
    if (ct.mode == 0) return;  // missing-free tiles are done by k_gram5
    t = W5Tile{ct.i0, ct.j0, 1};
    out_off = ct.out;
  }
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t sbase = smem_u32(smem);
  const uint32_t bar = sbase + STAGES * STAGE_BYTES;  // full[s] +8s | empty[s] +8(STAGES+s)
  const int npass = KIND == 1 ? 6 : (t.mode == 0 ? a.nslices : 4 * a.nslices);

  if (threadIdx.x == 0) {
    for (int s = 0; s < STAGES; s++) {
      mbar_init(bar + 8 * s, PROD_WARPS);            // one arrive per producer warp
      mbar_init(bar + 8 * (STAGES + s), MMA_WARPS);  // one arrive per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < PROD_WARPS) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(PROD_REGS));
    // ================= producers =================
    const int row = threadIdx.x & 127, oper = threadIdx.x >> 7;
    int line = (oper ? t.j0 : t.i0) + row;
    line = min(max(line, 0), a.nlines - 1);
    const uint8_t *src = a.P + (int64_t)line * a.stride;
    const uint32_t row_off = (uint32_t)oper * OPER_BYTES + (row >> 3) * SBO + (row & 7) * 16;
    int stage = 0;
    uint32_t phase = 0;
    for (int pass = 0; pass < npass; pass++) {
      int prod = pass, slice = 0, wsel = 0;
      if (KIND == 0) pass_info(t.mode, a.nslices, pass, prod, slice, wsel);
      // plane of this thread's operand: A uses the missing indicator for products na (2), nn (3); B for an (1), nn (3)
      const bool nplane = oper == 0 ? (prod >= 2) : (prod == 1 || prod == 3);
      const bool raw = t.mode == 0;  // no missing value in the tile: the packed word is the genotype plane
      const uint8_t *dg = KIND == 0 ? a.dig[wsel] + (int64_t)slice * a.dig_stride : nullptr;
      // KIND 1 planes per product: A = {a, b, a, b, h, b}, B = {a, b, b, a, b, h}
      const int cpl = oper == 0 ? ((0x121010 >> (4 * prod)) & 0xF) : ((0x210110 >> (4 * prod)) & 0xF);
      uint4 pf[PF][NW / 4];
#pragma unroll
      for (int u = 0; u < PF; u++) {
#pragma unroll
        for (int v = 0; v < NW / 4; v++)
          pf[u][v] = u < a.nsteps ? *reinterpret_cast<const uint4 *>(src + (int64_t)u * SBYTES + 16 * v) : make_uint4(0, 0, 0, 0);
      }
      for (int st0 = 0; st0 < a.nsteps; st0 += PF) {
#pragma unroll
        for (int u = 0; u < PF; u++) {
          const int st = st0 + u;
          if (st >= a.nsteps) break;
          uint32_t w[NW];
#pragma unroll
          for (int v = 0; v < NW / 4; v++) {
            w[4 * v] = pf[u][v].x; w[4 * v + 1] = pf[u][v].y; w[4 * v + 2] = pf[u][v].z; w[4 * v + 3] = pf[u][v].w;
          }
          if (st + PF < a.nsteps) {
#pragma unroll
            for (int v = 0; v < NW / 4; v++)
              pf[u][v] = *reinterpret_cast<const uint4 *>(src + (int64_t)(st + PF) * SBYTES + 16 * v);
          }
          mbar_wait(bar + 8 * (STAGES + stage), phase ^ 1);
          const uint32_t dst = sbase + stage * STAGE_BYTES + row_off;
#pragma unroll
          for (int k16 = 0; k16 < NW; k16++) {
            uint32_t x = w[k16];
            if (KIND == 1) {
              x = cor_plane(x, cpl);
            } else {
              const uint32_t nmask = x & (x >> 1) & 0x55555555u;
              if (nplane) x = nmask;
              else if (!raw) x &= ~(nmask | (nmask << 1));
            }
            uint32_t o[4];
            if (oper == 0 || KIND == 1) {
#pragma unroll
              for (int c = 0; c < 4; c++) o[c] = (x >> (2 * c)) & 0x03030303u;
            } else {
              const uint4 d4 = __ldg(reinterpret_cast<const uint4 *>(dg + ((int64_t)st * NW + k16) * 16));
              const uint32_t d[4] = {d4.x, d4.y, d4.z, d4.w};
#pragma unroll
              for (int c = 0; c < 4; c++) {
                const uint32_t xc = x >> (2 * c);
                const uint32_t m = (xc & 0x01010101u) * 0xFFu, hsel = ((xc >> 1) & 0x01010101u) * 0xFFu;
                o[c] = (m & d[c]) | (hsel & (d[c] << 1));
              }
            }
            sts128(dst + k16 * LBO, o[0], o[1], o[2], o[3]);
          }
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) mbar_arrive(bar + 8 * stage);
          if (++stage == STAGES) {
            stage = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ================= consumer warpgroups: one pass of MMAs, then K += scale * S (or the int32 sums) =================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(MMA_REGS));
    const int cw = (warp - PROD_WARPS) >> 2, wq = warp & 3;
    int stage = 0;
    uint32_t phase = 0;
    uint32_t d[64];
    for (int pass = 0; pass < npass; pass++) {
      int prod = pass, slice = 0, wsel = 0;
      if (KIND == 0) pass_info(t.mode, a.nslices, pass, prod, slice, wsel);
      consume_pass(d, sbase, bar, a.nsteps, cw, lane, stage, phase);
      if (KIND == 0) {
        const double sc = a.scale[wsel][slice];
#pragma unroll
        for (int j = 0; j < 64; j++) {
          const int i = t.i0 + 64 * cw + wg::acc_row(wq, lane, j), jj = t.j0 + wg::acc_col(lane, j);
          if (i < a.nlines && jj < a.nlines && i >= jj) a.K[(int64_t)jj * a.ldk + i] += sc * (double)(int)d[j];
        }
      } else {
        int *dst = a.sums + out_off + (int64_t)pass * (T5M * T5N);
#pragma unroll
        for (int j = 0; j < 64; j += 2) {
          const int r = 64 * cw + wg::acc_row(wq, lane, j), c = wg::acc_col(lane, j);
          *reinterpret_cast<int2 *>(dst + (int64_t)r * T5N + c) = make_int2((int)d[j], (int)d[j + 1]);
        }
      }
    }
  }
}

}  // namespace wg5

int wgram5_launch(const uint8_t *P, int64_t stride, int nlines, int nslices, const uint8_t *const dig[3],
                  int64_t dig_stride, const double (*scale)[10], const int *h_tiles /* i0, j0, mode triplets */,
                  int ntiles, double *K, int64_t ldk, cudaStream_t s) {
  using namespace wg5;
  if (ntiles == 0) return BSG_OK;
  W5Tile *d_tiles = nullptr;
  BSG_CUDA(cudaMalloc((void **)&d_tiles, (size_t)ntiles * sizeof(W5Tile)));
  cudaError_t e = cudaMemcpyAsync(d_tiles, h_tiles, (size_t)ntiles * sizeof(W5Tile), cudaMemcpyHostToDevice, s);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(k_wgram5<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, W5_SMEM_BYTES);
  if (e != cudaSuccess) {
    cudaFree(d_tiles);
    return cuda_fail(e, "wgram5 setup");
  }
  W5Args a;
  a.P = P;
  a.stride = stride;
  a.nlines = nlines;
  a.nsteps = (int)((stride + SBYTES - 1) / SBYTES);
  a.nslices = nslices;
  for (int w = 0; w < 3; w++) {
    a.dig[w] = dig[w];
    for (int sl = 0; sl < 10; sl++) a.scale[w][sl] = scale[w][sl];
  }
  a.dig_stride = dig_stride;
  a.tiles = d_tiles;
  a.ctiles = nullptr;
  a.sums = nullptr;
  a.K = K;
  a.ldk = ldk;
  k_wgram5<0><<<ntiles, W5_THREADS, W5_SMEM_BYTES, s>>>(a);
  count_launch();
  e = cudaGetLastError();
  cudaError_t e2 = cudaStreamSynchronize(s);
  cudaFree(d_tiles);
  if (e != cudaSuccess) return cuda_fail(e, "k_wgram5 launch");
  if (e2 != cudaSuccess) return cuda_fail(e2, "k_wgram5");
  return BSG_OK;
}

// host wrapper: sums[tile] = 128 x 128 int32 Gram of lines [i0, i0+128) x [j0, j0+128) of P
int gram5_launch(const uint8_t *P, int64_t stride, int nlines, int64_t line_bytes, const void *d_tiles, int ntiles,
                 int *d_sums, bool any_clean, bool any_na, cudaStream_t s) {
  using namespace gram5;
  if (ntiles == 0) return BSG_OK;
  BSG_CUDA(cudaFuncSetAttribute(k_gram5, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
  const int nsteps = (int)((line_bytes + SBYTES - 1) / SBYTES);
  if (any_clean) {
    k_gram5<<<ntiles, THREADS, SMEM_BYTES, s>>>(P, stride, nlines, nsteps, reinterpret_cast<const Tile5 *>(d_tiles), d_sums);
    count_launch();
  }
  if (any_na) {
    using namespace wg5;
    BSG_CUDA(cudaFuncSetAttribute(k_wgram5<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, W5_SMEM_BYTES));
    W5Args a;
    memset(&a, 0, sizeof a);
    a.P = P;
    a.stride = stride;
    a.nlines = nlines;
    a.nsteps = nsteps;
    a.nslices = 1;
    a.ctiles = reinterpret_cast<const gram::Tile *>(d_tiles);
    a.sums = d_sums;
    k_wgram5<1><<<ntiles, W5_THREADS, W5_SMEM_BYTES, s>>>(a);
    count_launch();
  }
  BSG_CUDA(cudaGetLastError());
  return BSG_OK;
}



}  // namespace bsg
