// ubench.cu -- microbenchmarks that size the design choices of k_pmv on a real GPU:
//   (1) IMMA.16832.U8.S8 issue rate per SM (legacy mma.sync path on sm_90a)
//   (2) cp.async.bulk (UBLKCP) throughput per SM as a function of the copy size
//   (3) plain LDG.128 streaming bandwidth (for reference)
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/ubench tools/ubench.cu
#include <cstdint>
#include <cstdio>
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
  return 0;
}
