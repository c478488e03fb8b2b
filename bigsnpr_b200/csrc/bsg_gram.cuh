// bsg_gram.cuh -- integer Gram tiles between lines of a packed 2-bit matrix on the tensor pipe.
//
//   S[i][j] = sum_k  fA(code(i, k)) * fB(code(j, k))        (exact, int32)
//
// for a 128 x 64 tile of line pairs, where fA / fB select a "plane" of the staged code:
//   PL_A : the genotype with missing -> 0   (0, 1, 2)
//   PL_B : valid indicator                   (1 unless missing)
//   PL_H : [genotype == 2]                   (so that sum a^2 = sum a + 2 sum h)
// Both operands of mma.sync.m16n8k32.u8.u8 come straight from the packed words of their lines: a register of the
// A fragment and a register of the B fragment are both "4 consecutive-k bytes of one line", i.e. a class mask
// ((plane >> 2c) & 0x03030303) of the same word index -- no shared-memory staging, no per-element unpack.
// Used, with a per-k weight digit folded into the B bytes, by the Gram product of bed_tcrossprodSelf (bsg_la.cu).  The
// wgmma helpers at the end serve the 128 x 128 tile kernels, which the windowed correlations (bsg_cor.cu) run on.
#pragma once
#include <stdint.h>

namespace bsg {
namespace gram {

constexpr int TM = 128, TN = 64;    // tile of line pairs per CTA
constexpr int WARPS = 8;            // 4 (M) x 2 (N) warps, 32 x 32 outputs each
constexpr int THREADS = WARPS * 32;
constexpr int CHUNK = 64;           // bytes per line per step (one LDG.128 per lane = 4 words = 64 codes)

enum Plane { PL_A = 0, PL_B = 1, PL_H = 2 };

struct Tile {
  int i0, j0;        // first A line, first B line
  int mode;          // 0: one product (a,a), codes without missing values; 1: the six products of the NA-aware cor
  long long out;     // offset (in int32) of this tile's sums: [nprod][TM][128]
};

__device__ __forceinline__ void mma_u8u8(int (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k32.row.col.s32.u8.u8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}

__device__ __forceinline__ uint4 ldg128(const uint8_t *p) {
  uint4 v;
  asm volatile("ld.global.nc.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}

// plane word of 16 codes
template <int PL>
__device__ __forceinline__ uint32_t plane_word(uint32_t w) {
  const uint32_t n = w & (w >> 1) & 0x55555555u;  // bit 2p set iff code p is missing
  if (PL == PL_A) return w & ~(n | (n << 1));
  if (PL == PL_B) return ~n & 0x55555555u;
  return ((w & ~(n | (n << 1))) >> 1) & 0x55555555u;  // PL_H
}

}  // namespace gram

// ---- Hopper warpgroup MMA (wgmma) on u8 operands in shared memory, int32 accumulators in registers ----------------
// Used by the 128 x 128 Gram tiles (bsg_gram5.cu, bsg_gramt.cu).  Integer wgmma needs both operands K-major.
// Accumulator fragment of m64n128 (thread t of the warpgroup, w = t / 32, l = t % 32): d[j] holds
//   row 16 w + l / 4 + 8 ((j / 2) % 2),  column 8 (j / 4) + 2 (l % 4) + (j % 2).
namespace wg {

// shared-memory matrix descriptor (sm_90 GMMA): start >> 4 at [0,14), LBO >> 4 at [16,30), SBO >> 4 at [32,46),
// layout type at [62,64): 0 = no swizzle (core matrices 8 rows x 16 B), 1 = 128-byte swizzle
__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t lbo, uint32_t sbo, uint32_t layout) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo >> 4) & 0x3FFFu) << 16) |
         ((uint64_t)((sbo >> 4) & 0x3FFFu) << 32) | ((uint64_t)layout << 62);
}
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// d (64 x 128, s32) = A (64 x 32 u8) . B (128 x 32 u8)^T + (accumulate ? d : 0)
__device__ __forceinline__ void mma_u8_n128(uint32_t (&d)[64], uint64_t da, uint64_t db, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k32.s32.u8.u8 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,"
      "%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,"
      "%60,%61,%62,%63}, %64, %65, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
        "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
        "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
        "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31]), "+r"(d[32]),
        "+r"(d[33]), "+r"(d[34]), "+r"(d[35]), "+r"(d[36]), "+r"(d[37]), "+r"(d[38]), "+r"(d[39]), "+r"(d[40]),
        "+r"(d[41]), "+r"(d[42]), "+r"(d[43]), "+r"(d[44]), "+r"(d[45]), "+r"(d[46]), "+r"(d[47]), "+r"(d[48]),
        "+r"(d[49]), "+r"(d[50]), "+r"(d[51]), "+r"(d[52]), "+r"(d[53]), "+r"(d[54]), "+r"(d[55]), "+r"(d[56]),
        "+r"(d[57]), "+r"(d[58]), "+r"(d[59]), "+r"(d[60]), "+r"(d[61]), "+r"(d[62]), "+r"(d[63])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

// row / column of accumulator element j for lane l of warp w (0..3) of the warpgroup
__device__ __forceinline__ int acc_row(int w, int l, int j) { return 16 * w + (l >> 2) + 8 * ((j >> 1) & 1); }
__device__ __forceinline__ int acc_col(int l, int j) { return 8 * (j >> 2) + 2 * (l & 3) + (j & 1); }

}  // namespace wg
}  // namespace bsg
