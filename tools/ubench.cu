// ubench.cu -- microbenchmarks that size the design choices of k_pmv on a real GPU:
//   (1) IMMA.16832.U8.S8 issue rate per SM (legacy mma.sync path on sm_90a)
//   (2) cp.async.bulk (UBLKCP) throughput per SM as a function of the copy size
//   (3) plain LDG.128 streaming bandwidth (for reference)
//   (4) load-only loaders of k_pmvT at the configs[4] line geometry (121,856-byte line stride, 2^17 lines >> L2):
//       (a) per-warp cp.async 64-byte strips, (b) one cp.async.bulk of 512 B per line per CTA stage, (c) a 2D TMA
//       stage of 32 lines x 4 boxes of 128 B (128-byte swizzle, L2_256B promotion), (d) = (a) with .L2::256B
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cuda.h>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

__global__ void k_imma(int iters, int *out, long long *cyc) {
  int acc[4][4] = {};
  uint32_t a = threadIdx.x * 0x01010101u, b = 0x01020304u;
  long long t0 = clock64();
  for (int i = 0; i < iters; i++) {
#pragma unroll
    for (int k = 0; k < 4; k++)
      asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
                   : "+r"(acc[k][0]), "+r"(acc[k][1]), "+r"(acc[k][2]), "+r"(acc[k][3])
                   : "r"(a), "r"(a + k), "r"(a ^ 5), "r"(a + 7), "r"(b), "r"(b + k));
  }
  long long t1 = clock64();
  int s = 0;
  for (int k = 0; k < 4; k++) for (int j = 0; j < 4; j++) s += acc[k][j];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}

// each CTA: one warp streams `total` bytes from global through a 4-stage smem ring using bulk copies of `csz` bytes
__global__ void k_bulk(const uint8_t *src, size_t per_cta, int csz, int stage_bytes, long long *cyc) {
  extern __shared__ __align__(128) uint8_t sm[];
  __shared__ uint64_t bars[4];
  uint32_t sb = (uint32_t)__cvta_generic_to_shared(sm);
  uint32_t bb = (uint32_t)__cvta_generic_to_shared(bars);
  int lane = threadIdx.x;
  if (lane == 0) {
    for (int s = 0; s < 4; s++) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(bb + 8 * s));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncwarp();
  const uint8_t *base = src + (size_t)blockIdx.x * per_cta;
  int nstage = (int)(per_cta / stage_bytes);
  int ncopy = stage_bytes / csz;
  long long t0 = clock64();
  for (int st = 0; st < nstage + 3; st++) {
    if (st >= 3) mbar_wait(bb + 8 * ((st - 3) & 3), ((st - 3) >> 2) & 1);
    if (st < nstage) {
      int s = st & 3;
      if (lane == 0) asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bb + 8 * s), "r"(stage_bytes) : "memory");
      __syncwarp();
      for (int c = lane; c < ncopy; c += 32)
        asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(sb + s * stage_bytes + c * csz),
                     "l"(base + (size_t)st * stage_bytes + (size_t)c * csz), "r"(csz), "r"(bb + 8 * s) : "memory");
    }
  }
  long long t1 = clock64();
  if (lane == 0) cyc[blockIdx.x] = t1 - t0;
}

__global__ void k_ldg(const uint4 *src, size_t n, uint4 *out) {
  uint4 acc = make_uint4(0, 0, 0, 0);
  size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x, st = (size_t)gridDim.x * blockDim.x;
  for (; i + 3 * st < n; i += 4 * st) {
    uint4 a = __ldg(src + i), b = __ldg(src + i + st), c = __ldg(src + i + 2 * st), d = __ldg(src + i + 3 * st);
    acc.x ^= a.x ^ b.x ^ c.x ^ d.x; acc.y ^= a.y ^ b.y ^ c.y ^ d.y; acc.z ^= a.z ^ b.z ^ c.z ^ d.z; acc.w ^= a.w ^ b.w ^ c.w ^ d.w;
  }
  if (acc.x == 0x12345678u) out[0] = acc;
}

// ---- (4) load-only loaders at k_pmvT's line geometry ------------------------------------------------------------------
// Grid = nblocks x ksplit CTAs, 2 per SM; CTA (blk, ks) reads bytes [512 blk, 512 blk + 512) of lines
// [ks lps, (ks + 1) lps), 32 lines per step.  Consumers touch one shared word per step so each stage is waited for.
constexpr int LD_STRIDE = 121856, LD_NBYTES = 121750, LD_SEG = 512, LD_STAGES = 6, LD_WARPS = 8;
constexpr int LD_PITCH = 544, LD_BSTAGE = 32 * LD_PITCH + 288;  // (b): padded rows + two 128-byte digit copies
constexpr int LD_TSTAGE = 4 * 4096 + 1024;                      // (c): 4 swizzled boxes + digits, 1 KB aligned

__device__ __forceinline__ uint32_t s32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ void bar_init(uint32_t b, uint32_t c) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(b), "r"(c)); }
__device__ __forceinline__ void bar_tx(uint32_t b, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(b), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bar_arrive(uint32_t b) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(b) : "memory"); }
__device__ __forceinline__ void bulk(uint32_t dst, const void *src, uint32_t bytes, uint32_t b) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(b) : "memory");
}

template <bool HINT>
__global__ void __launch_bounds__(LD_WARPS * 32, 2) k_ld_strip(const uint8_t *P, int nlines, int lps, int nblocks, uint32_t *out) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int blk = blockIdx.x % nblocks, ks = blockIdx.x / nblocks;
  const int64_t byte0 = (int64_t)blk * LD_SEG + 64 * warp;
  const int l0 = ks * lps, l1 = min(nlines, l0 + lps), nsteps = (l1 - l0) / 32;
  const uint32_t wbase = s32(sm) + warp * LD_STAGES * 2048;
  const int lrow = lane >> 2, lch = lane & 3;
  const int64_t colb = (byte0 + 16 * lch < LD_STRIDE) ? byte0 + 16 * lch : 0;
  const uint8_t *src = P + colb + (int64_t)(l0 + lrow) * LD_STRIDE;
  auto issue = [&](int step) {
    const uint32_t dst = wbase + (step % LD_STAGES) * 2048 + lane * 16;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint8_t *g = src + ((int64_t)step * 32 + 8 * i) * LD_STRIDE;
      if (HINT)
        asm volatile("cp.async.cg.shared.global.L2::256B [%0], [%1], 16;" ::"r"(dst + i * 512), "l"(g) : "memory");
      else
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst + i * 512), "l"(g) : "memory");
    }
  };
  uint32_t acc = 0;
  for (int st = 0; st < LD_STAGES - 1; st++) {
    if (st < nsteps) issue(st);
    asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int step = 0; step < nsteps; step++) {
    asm volatile("cp.async.wait_group %0;" ::"n"(LD_STAGES - 2) : "memory");
    __syncwarp();
    if (step + LD_STAGES - 1 < nsteps) issue(step + LD_STAGES - 1);
    asm volatile("cp.async.commit_group;" ::: "memory");
    acc ^= lds32(wbase + (step % LD_STAGES) * 2048 + lane * 4);
  }
  asm volatile("cp.async.wait_group 0;" ::: "memory");
  if (acc == 0x9e3779b9u) out[0] = acc;
}

// (b) and (c): one producer warp fills CTA-wide stages (full / empty mbarriers), LD_WARPS consumer warps drain them
template <bool TMA>
__global__ void __launch_bounds__((LD_WARPS + 1) * 32, 2)
    k_ld_stage(const __grid_constant__ CUtensorMap map, const uint8_t *P, const uint8_t *dig, int nlines, int lps, int nblocks,
               uint32_t *out) {
  extern __shared__ __align__(128) uint8_t sm[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int blk = blockIdx.x % nblocks, ks = blockIdx.x / nblocks;
  const int64_t byte0 = (int64_t)blk * LD_SEG;
  const int l0 = ks * lps, l1 = min(nlines, l0 + lps), nsteps = (l1 - l0) / 32;
  constexpr int STAGE = TMA ? LD_TSTAGE : LD_BSTAGE;
  const uint32_t sbase = TMA ? (s32(sm) + 1023u) & ~1023u : s32(sm), bars = sbase + LD_STAGES * STAGE;
  if (threadIdx.x == 0) {
    for (int s = 0; s < LD_STAGES; s++) {
      bar_init(bars + 8 * s, 1);
      bar_init(bars + 8 * (LD_STAGES + s), LD_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  int stage = 0;
  uint32_t ph = 0;
  if (warp == LD_WARPS) {
    const uint32_t bytes = (uint32_t)(LD_STRIDE - byte0 < LD_SEG ? LD_STRIDE - byte0 : LD_SEG);
    const int row = (lane & 16) | ((lane & 3) << 2) | ((lane >> 2) & 3);
    for (int step = 0; step < nsteps; step++) {
      const uint32_t full = bars + 8 * stage, empty = bars + 8 * (LD_STAGES + stage), dst = sbase + stage * STAGE;
      asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(empty),
                   "r"(ph ^ 1) : "memory");
      const uint8_t *dg = dig + (int64_t)(l0 / 32 + step) * 256;
      if (TMA) {
        if (lane == 0) {
          bar_tx(full, 4 * 4096 + 256);
          for (int j = 0; j < 4; j++)
            asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst + j * 4096),
                         "l"(&map), "r"(full), "r"((int)byte0 + 128 * j), "r"(l0 + 32 * step) : "memory");
          bulk(dst + 4 * 4096, dg, 256, full);
        }
      } else {
        if (lane == 0) bar_tx(full, 32 * bytes + 256);
        __syncwarp();
        bulk(dst + row * LD_PITCH, P + (int64_t)(l0 + 32 * step + lane) * LD_STRIDE + byte0, bytes, full);
        if (lane < 2) bulk(dst + 32 * LD_PITCH + 144 * lane, dg + 128 * lane, 128, full);
      }
      if (++stage == LD_STAGES) { stage = 0; ph ^= 1; }
    }
  } else {
    uint32_t acc = 0;
    for (int step = 0; step < nsteps; step++) {
      const uint32_t full = bars + 8 * stage, empty = bars + 8 * (LD_STAGES + stage);
      asm volatile("{\n\t.reg .pred p;\n\tW_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra D_%=;\n\tbra W_%=;\n\tD_%=:\n\t}" ::"r"(full),
                   "r"(ph) : "memory");
      acc ^= lds32(sbase + stage * STAGE + warp * 64 + lane * 4);
      __syncwarp();
      if (lane == 0) bar_arrive(empty);
      if (++stage == LD_STAGES) { stage = 0; ph ^= 1; }
    }
    if (acc == 0x9e3779b9u) out[0] = acc;
  }
}

typedef CUresult (*EncodeFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *, const cuuint64_t *,
                             const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave, CUtensorMapSwizzle,
                             CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int loaders(uint32_t *out) {
  const int nlines = 1 << 17, ks = 4, lps = nlines / ks, nblocks = (LD_NBYTES + LD_SEG - 1) / LD_SEG;
  const double bytes = (double)nlines * LD_NBYTES;
  uint8_t *P, *dig;
  CK(cudaMalloc(&P, (size_t)nlines * LD_STRIDE));
  CK(cudaMemset(P, 0x5a, (size_t)nlines * LD_STRIDE));
  CK(cudaMalloc(&dig, (size_t)nlines / 32 * 256));
  CK(cudaMemset(dig, 1, (size_t)nlines / 32 * 256));
  CUtensorMap map;
  {
    void *p = nullptr;
    cudaDriverEntryPointQueryResult qr;
    CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr));
    cuuint64_t gdim[2] = {(cuuint64_t)LD_STRIDE, (cuuint64_t)nlines}, gstr[1] = {(cuuint64_t)LD_STRIDE};
    cuuint32_t box[2] = {128, 32}, estr[2] = {1, 1};
    if (((EncodeFn)p)(&map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, P, gdim, gstr, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
      printf("cuTensorMapEncodeTiled failed\n");
      return 1;
    }
  }
  const int strip_smem = LD_WARPS * LD_STAGES * 2048;
  const int bulk_smem = LD_STAGES * LD_BSTAGE + 128, tma_smem = LD_STAGES * LD_TSTAGE + 1024 + 128;
  CK(cudaFuncSetAttribute(k_ld_strip<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, strip_smem));
  CK(cudaFuncSetAttribute(k_ld_strip<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, strip_smem));
  CK(cudaFuncSetAttribute(k_ld_stage<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, bulk_smem));
  CK(cudaFuncSetAttribute(k_ld_stage<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, tma_smem));
  const int grid = nblocks * ks;
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  const char *names[4] = {"(a) per-warp cp.async 64 B strips      ", "(b) cp.async.bulk 512 B per line       ",
                          "(c) TMA 2D 4 x 128 B boxes, L2_256B    ", "(d) (a) + cp.async .L2::256B           "};
  for (int v = 0; v < 4; v++) {
    float t[6];
    for (int r = 0; r < 6; r++) {  // launch 0 warms up
      cudaEventRecord(e0);
      if (v == 0) k_ld_strip<false><<<grid, LD_WARPS * 32, strip_smem>>>(P, nlines, lps, nblocks, out);
      if (v == 3) k_ld_strip<true><<<grid, LD_WARPS * 32, strip_smem>>>(P, nlines, lps, nblocks, out);
      if (v == 1) k_ld_stage<false><<<grid, (LD_WARPS + 1) * 32, bulk_smem>>>(map, P, dig, nlines, lps, nblocks, out);
      if (v == 2) k_ld_stage<true><<<grid, (LD_WARPS + 1) * 32, tma_smem>>>(map, P, dig, nlines, lps, nblocks, out);
      cudaEventRecord(e1);
      CK(cudaDeviceSynchronize());
      cudaEventElapsedTime(&t[r], e0, e1);
    }
    std::sort(t + 1, t + 6);
    printf("load-only %s %d x %d CTAs: median %.3f ms = %.1f GB/s (best %.1f GB/s) over %.2f GB\n", names[v], nblocks, ks, t[3],
           bytes / (t[3] * 1e-3) / 1e9, bytes / (t[1] * 1e-3) / 1e9, bytes / 1e9);
  }
  CK(cudaFree(P));
  CK(cudaFree(dig));
  return 0;
}

int main() {
  int nsm = 132;
  cudaDeviceGetAttribute(&nsm, cudaDevAttrMultiProcessorCount, 0);
  int clk = 0;
  cudaDeviceGetAttribute(&clk, cudaDevAttrClockRate, 0);
  printf("SMs %d, clock attr %d kHz\n", nsm, clk);
  int *out; long long *cyc;
  CK(cudaMalloc(&out, nsm * 1024 * 4)); CK(cudaMalloc(&cyc, nsm * 8));
  long long hc[1024];
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  // (1) IMMA
  for (int warps : {1, 4, 8, 16}) {
    int iters = 20000;
    k_imma<<<nsm, warps * 32>>>(100, out, cyc);
    cudaEventRecord(e0);
    k_imma<<<nsm, warps * 32>>>(iters, out, cyc);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    CK(cudaMemcpy(hc, cyc, 8 * nsm, cudaMemcpyDeviceToHost));
    double imma_per_sm = (double)iters * 4 * warps;
    printf("IMMA.16832 warps/SM=%2d: %.2f cycles per IMMA per SM (clock64), %.3f ms, %.1f TOPS dense-equivalent\n", warps,
           (double)hc[0] / imma_per_sm, ms, imma_per_sm * nsm * 16 * 8 * 32 * 2 / (ms * 1e-3) / 1e12);
  }
  // (2) bulk copies
  size_t per_cta = (size_t)64 << 20;
  uint8_t *src; CK(cudaMalloc(&src, per_cta * nsm)); CK(cudaMemset(src, 1, per_cta * nsm));
  for (int stage_bytes : {32768}) {
    for (int csz : {128, 256, 512, 1024, 2048, 4096, 16384, 32768}) {
      CK(cudaFuncSetAttribute(k_bulk, cudaFuncAttributeMaxDynamicSharedMemorySize, 4 * stage_bytes));
      k_bulk<<<nsm, 32, 4 * stage_bytes>>>(src, per_cta / 16, csz, stage_bytes, cyc);
      cudaEventRecord(e0);
      k_bulk<<<nsm, 32, 4 * stage_bytes>>>(src, per_cta, csz, stage_bytes, cyc);
      cudaEventRecord(e1);
      CK(cudaDeviceSynchronize());
      float ms; cudaEventElapsedTime(&ms, e0, e1);
      CK(cudaMemcpy(hc, cyc, 8 * nsm, cudaMemcpyDeviceToHost));
      printf("UBLKCP copy %6d B (stage %d B, 4 stages, 1 CTA/SM): %.1f GB/s total, %.1f cycles per copy per SM\n", csz, stage_bytes,
             (double)per_cta * nsm / (ms * 1e-3) / 1e9, (double)hc[0] / ((double)per_cta / csz));
    }
  }
  // (3) LDG streaming
  {
    size_t n = per_cta * nsm / 16;
    k_ldg<<<nsm * 8, 512>>>((const uint4 *)src, n, (uint4 *)out);
    cudaEventRecord(e0);
    k_ldg<<<nsm * 8, 512>>>((const uint4 *)src, n, (uint4 *)out);
    cudaEventRecord(e1);
    CK(cudaDeviceSynchronize());
    float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("LDG.128 stream: %.1f GB/s\n", (double)n * 16 / (ms * 1e-3) / 1e9);
  }
  CK(cudaFree(src));
  // (4) load-only loaders of k_pmvT
  return loaders((uint32_t *)out);
}
