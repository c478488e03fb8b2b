// bsg_pmv_shared.cuh -- device-side pieces of the matvec epilogue shared between bsg_pmv.cu (plain finish kernels) and
// bsg_comm.cu (finish fused with the all-reduce over NVLink peer memory).
#pragma once
#include <stdint.h>

namespace bsg {
namespace pmv {

constexpr int SUMCZ_BLOCKS = 128;

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
