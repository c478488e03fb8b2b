// bsg_pmv_shared.cuh -- device-side pieces of the matvecs shared between bsg_pmv.cu (2-bit kernels, plain finish kernels),
// bsg_dosage.cu (byte-operand kernels) and bsg_comm.cu (finish fused with the all-reduce over NVLink peer memory).
#pragma once
#include <cuda.h>
#include <math.h>
#include <stdint.h>

namespace bsg {
namespace pmv {

constexpr int SUMCZ_BLOCKS = 128;

// ---- PTX wrappers and the fixed-point vector format, shared by the 2-bit kernels (bsg_pmv.cu) and the byte-operand
// kernels (bsg_dosage.cu)
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
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
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void *src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst),
               "l"(src), "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void mma_u8s8(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                         uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint4 lds128(uint32_t addr) {
  uint4 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
  return v;
}

__device__ __forceinline__ uint4 ldg_stream(const uint8_t *p) {
  uint4 v;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p));
  return v;
}

__device__ __forceinline__ uint32_t lds32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel) {
  uint32_t r;
  asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
  return r;
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}

// CTA stage of k_pmvT / k_dmvT (128-byte-swizzled TMA boxes): address bits of read i (row i, chunk ^ i) and of word column
// half sl (chunk ^ 2 sl), relative to the lane's i = sl = 0
__host__ __device__ constexpr uint32_t TRD(int i, int sl) { return (uint32_t)((i << 7) ^ (i << 4) ^ (sl << 5)); }

// e = bits - exponent(maxabs) - hb, so that |sum of <= 2^hb quantised values| < 2^bits (bits = 60: hb_bits in
// bsg_pmv.cu adds a bit where rint could round an entry up to 2^(bits - hb)).  bits = 60: one vector in 8
// signed base-256 digits; bits = 30: one of two vectors sharing a pass in 4 digits (max 127 * (2^32 - 1) / 255).
__device__ __forceinline__ int pick_e(double m, int hb, int bits) {
  int ex = 0;
  if (m > 0 && isfinite(m)) {
    frexp(m, &ex);
    return bits - ex - hb;
  }
  return 0;
}

// the next signed base-256 digit of q (its low byte as int8); q keeps the exact rest (q - d) / 256
__device__ __forceinline__ int peel(long long &q) {
  const int d = (int)(signed char)(q & 0xFF);
  q = (q - d) >> 8;
  return d;
}

struct Scal {          // device-resident scalars of one call (of one vector, when two vectors share a pass)
  double maxabs[2];    // [0] raw-plane vector, [1] NA-plane vector
  int nonfinite;
  int e[2];            // Q = rint(v * 2^e); published by the digit-layout kernel, derived from maxabs and hb
  int hb;              // headroom bits (log2 of the largest index multiplicity)
  long long sum_hi, sum_lo;
  double cpart[128];   // per-block partials of sum_k c_k z_k (X.y), added in index order by the finish kernel
};

// (raw-plane * c0 + NA-plane * c1) per digit slice s0 .. s0 + NS - 1, exact in integers, then one top-down fp64 sum of
// the NS scaled slice totals (slice s0 + s weighs 2^(8 s - e)).  NS = 8: one vector; NS = 4: one of two vectors.
template <int NS>
__device__ __forceinline__ double combine(const long long *__restrict__ part, int64_t line, int s0, int c0, int c1, int e) {
  const long long *p = part + line * 16 + s0;
  double acc = 0;
#pragma unroll
  for (int s = NS - 1; s >= 0; s--) {
    long long v = 0;
    if (c0) v += c0 * p[s];
    if (c1) v += c1 * p[8 + s];
    acc += scalbn((double)v, 8 * s - e);
  }
  return acc;
}

// X.y:  full_l = R + Nw - C   with Nw the NA-plane sum against w = (c - 3) z;  without scaling full_l = R - 3 N.
// The vector's slices are s0 .. s0 + NS - 1 of the line, its scalars *sc.
template <int NS = 8>
__device__ __forceinline__ double finish_prod_value(const long long *__restrict__ part, int64_t l, const Scal *sc,
                                                    int has_scaling, int use_na, int s0 = 0) {
  if (sc->nonfinite) return nan("");
  if (has_scaling) {
    double C = 0;
    for (int b = 0; b < SUMCZ_BLOCKS; b++) C += sc->cpart[b];
    double R = combine<NS>(part, l, s0, 1, 0, sc->e[0]);
    double Nw = use_na ? combine<NS>(part, l, s0, 0, 1, sc->e[1]) : 0.0;
    return (R + Nw) - C;
  }
  return combine<NS>(part, l, s0, 1, use_na ? -3 : 0, sc->e[0]);  // R - 3N, exact
}

}  // namespace pmv
}  // namespace bsg
