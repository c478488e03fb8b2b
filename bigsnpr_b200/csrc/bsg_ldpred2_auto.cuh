/* bsg_ldpred2_auto.cuh -- the arithmetic of LDpred2-auto's sampler (src/ldpred2-auto.cpp:56-202), shared by the device
 * kernel (nvcc) and the tests' sequential CPU restatement (gcc, tests/ldpred2_auto_*.c), so both compute the same bits.
 *
 * Valid C99 and CUDA C++.  Only + - * /, sqrt (correctly rounded on both sides), integer and bit operations: on the
 * device every floating operation is an __d*_rn intrinsic, on the host the restatement is built with -ffp-contract=off, so no
 * product is contracted into an FMA on either side.  exp and log are implemented here because CUDA's and glibc's differ
 * in the last bit.
 *
 *   - MRG32k3a (L'Ecuyer 1999) on 6 uint32 words, R's L'Ecuyer-CMRG unif_rand formula and fixup into (0, 1); skip-ahead
 *     by the transition matrices A^k mod m, and the 2^127 stream jump (parallel::nextRNGStream's).
 *   - norm_rand by inversion as R's INVERSION kind: u = floor(2^27 u1) + u2, z = qnorm(u / 2^27), qnorm Wichura's AS241
 *     (PPND16); rnorm(mu, sigma) = mu + sigma z, no draw when sigma == 0 or mu is not finite.
 *   - rbeta: Cheng's (1978) algorithms BB (min(a, b) > 1) and BC (otherwise), as R's rbeta uses them.
 *   - exp / log: Cody-Waite reduction and the minimax polynomials of fdlibm's e_exp.c / e_log.c (< 1 ulp).
 *   - the coordinate update of the Gibbs sweep, the MLE objective's profile in alpha + 1 and its golden-section search;
 *   - LDpred2-grid's coordinate update (src/ldpred2.cpp:9-69, src/ldpred2-sampling.cpp:9-59) and the draw offset of a
 *     warp lane when a sparse point skips the uniform of the coordinates it zeroes.
 */
#ifndef BSG_LDPRED2_AUTO_CUH
#define BSG_LDPRED2_AUTO_CUH

#include <stdint.h>

#ifdef __CUDACC__
#define LDA_FN static __host__ __device__ inline
#else
#define LDA_FN static inline
#endif

#ifdef __CUDA_ARCH__
#define LDA_ADD(a, b) __dadd_rn((a), (b))
#define LDA_SUB(a, b) __dsub_rn((a), (b))
#define LDA_MUL(a, b) __dmul_rn((a), (b))
#define LDA_DIV(a, b) __ddiv_rn((a), (b))
#define LDA_SQRT(a) __dsqrt_rn(a)
#define LDA_BITS(d) ((uint64_t)__double_as_longlong(d))
#define LDA_DBL(u) __longlong_as_double((long long)(u))
#else
#include <math.h>
#include <string.h>
#define LDA_ADD(a, b) ((a) + (b))
#define LDA_SUB(a, b) ((a) - (b))
#define LDA_MUL(a, b) ((a) * (b))
#define LDA_DIV(a, b) ((a) / (b))
#define LDA_SQRT(a) sqrt(a)
static inline uint64_t lda_bits_(double d) {
  uint64_t u;
  memcpy(&u, &d, sizeof u);
  return u;
}
static inline double lda_dbl_(uint64_t u) {
  double d;
  memcpy(&d, &u, sizeof d);
  return d;
}
#define LDA_BITS(d) lda_bits_(d)
#define LDA_DBL(u) lda_dbl_(u)
#endif

#define LDA_INF LDA_DBL(0x7FF0000000000000ULL)
#define LDA_NAN LDA_DBL(0x7FF8000000000000ULL)
#define LDA_DBL_MAX 1.7976931348623157e308

/* ---- MRG32k3a ------------------------------------------------------------------------------------------------------- */

#define LDA_M1 4294967087ULL
#define LDA_M2 4294944443ULL
#define LDA_NORMC 2.328306549295727688e-10 /* 1 / (m1 + 1) */
#define LDA_I2_32M1 2.328306437080797e-10  /* 1 / (2^32 - 1), R's fixup */

/* A transition matrix pair: a[0..8] the first component (mod m1), a[9..17] the second (mod m2), row-major.  One step maps
 * the state (s0, s1, s2 | s3, s4, s5) to A s; its output is from the new s2 and s5. */
typedef struct {
  uint32_t a[18];
} lda_mat;

LDA_FN uint32_t lda_mulmod3(const uint32_t *row, const uint32_t *v, uint64_t m) {
  uint64_t r = ((uint64_t)row[0] * v[0]) % m;
  r = (r + ((uint64_t)row[1] * v[1]) % m) % m;
  return (uint32_t)((r + ((uint64_t)row[2] * v[2]) % m) % m);
}

LDA_FN lda_mat lda_mat_one_step(void) {
  lda_mat A;
  for (int i = 0; i < 18; i++) A.a[i] = 0;
  A.a[1] = 1, A.a[5] = 1, A.a[6] = (uint32_t)(LDA_M1 - 810728), A.a[7] = 1403580;
  A.a[10] = 1, A.a[14] = 1, A.a[15] = (uint32_t)(LDA_M2 - 1370589), A.a[17] = 527612;
  return A;
}

/* X Y (mod m1 / m2) */
LDA_FN lda_mat lda_mat_mul(const lda_mat *X, const lda_mat *Y) {
  lda_mat Z;
  for (int c = 0; c < 2; c++) {
    const uint64_t m = c ? LDA_M2 : LDA_M1;
    const uint32_t *x = X->a + 9 * c, *y = Y->a + 9 * c;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) {
        const uint32_t col[3] = {y[j], y[3 + j], y[6 + j]};
        Z.a[9 * c + 3 * i + j] = lda_mulmod3(x + 3 * i, col, m);
      }
  }
  return Z;
}

/* s = A s */
LDA_FN void lda_mat_apply(const lda_mat *A, uint32_t *s) {
  uint32_t t[6];
  for (int i = 0; i < 3; i++) t[i] = lda_mulmod3(A->a + 3 * i, s, LDA_M1);
  for (int i = 0; i < 3; i++) t[3 + i] = lda_mulmod3(A->a + 9 + 3 * i, s + 3, LDA_M2);
  for (int i = 0; i < 6; i++) s[i] = t[i];
}

/* R's unif_rand for L'Ecuyer-CMRG from the two new components; the fixup never triggers for this generator (the value
 * lies in [normc, m1 normc]) and is kept as R has it */
LDA_FN double lda_u01(uint32_t p1, uint32_t p2) {
  const int64_t d = (int64_t)p1 - (int64_t)p2;
  const double v = LDA_MUL((double)(p1 > p2 ? d : d + (int64_t)LDA_M1), LDA_NORMC);
  if (v <= 0.0) return 0.5 * LDA_I2_32M1;
  if (LDA_SUB(1.0, v) <= 0.0) return 1.0 - 0.5 * LDA_I2_32M1;
  return v;
}

/* one draw: R's recurrence (p1 = a12 s1 - a13n s0 mod m1, p2 = a21 s5 - a23n s3 mod m2) */
LDA_FN double lda_unif(uint32_t *s) {
  int64_t p1 = 1403580LL * s[1] - 810728LL * s[0];
  p1 %= (int64_t)LDA_M1;
  if (p1 < 0) p1 += (int64_t)LDA_M1;
  s[0] = s[1], s[1] = s[2], s[2] = (uint32_t)p1;
  int64_t p2 = 527612LL * s[5] - 1370589LL * s[3];
  p2 %= (int64_t)LDA_M2;
  if (p2 < 0) p2 += (int64_t)LDA_M2;
  s[3] = s[4], s[4] = s[5], s[5] = (uint32_t)p2;
  return lda_u01((uint32_t)p1, (uint32_t)p2);
}

/* pw[i] = A^(2^i), i < n */
LDA_FN void lda_pow2_table(lda_mat *pw, int n) {
  pw[0] = lda_mat_one_step();
  for (int i = 1; i < n; i++) pw[i] = lda_mat_mul(&pw[i - 1], &pw[i - 1]);
}

/* A^k from the table pw[i] = A^(2^i) (2^n > k for a table of n entries) */
LDA_FN lda_mat lda_mat_pow(const lda_mat *pw, uint64_t k) {
  lda_mat M;
  for (int i = 0; i < 18; i++) M.a[i] = (i % 9) % 4 == 0; /* identity */
  for (int i = 0; k; i++, k >>= 1)
    if (k & 1) M = lda_mat_mul(&M, &pw[i]);
  return M;
}

/* s advanced by k draws, from a table pw[i] = A^(2^i) with 2^npw > k */
LDA_FN void lda_skip(uint32_t *s, uint64_t k, const lda_mat *pw) {
  for (int i = 0; k; i++, k >>= 1)
    if (k & 1) lda_mat_apply(&pw[i], s);
}

/* s advanced by 2^127 draws: the next stream (parallel::nextRNGStream) */
LDA_FN void lda_jump127(uint32_t *s) {
  lda_mat A = lda_mat_one_step();
  for (int i = 0; i < 127; i++) A = lda_mat_mul(&A, &A);
  lda_mat_apply(&A, s);
}

/* ---- exp and log (fdlibm's e_exp.c / e_log.c algorithms) ----------------------------------------------------------- */

LDA_FN double lda_exp(double x) {
  const double ln2hi = 6.93147180369123816490e-01, ln2lo = 1.90821492927058770002e-10;
  const double invln2 = 1.44269504088896338700e+00;
  const double P1 = 1.66666666666666019037e-01, P2 = -2.77777777770155933842e-03, P3 = 6.61375632143793436117e-05,
               P4 = -1.65339022054652515390e-06, P5 = 4.13813679705723846039e-08;
  if (x != x) return x;
  if (x > 7.09782712893383973096e+02) return LDA_INF;
  if (x < -7.45133219101941108420e+02) return 0.0;
  const uint64_t ax = LDA_BITS(x) & 0x7FFFFFFFFFFFFFFFULL;
  if (ax < 0x3E30000000000000ULL) return LDA_ADD(1.0, x); /* |x| < 2^-28 */
  const int k = (int)LDA_ADD(LDA_MUL(invln2, x), x < 0 ? -0.5 : 0.5);
  const double dk = (double)k;
  const double hi = LDA_SUB(x, LDA_MUL(dk, ln2hi)), lo = LDA_MUL(dk, ln2lo);
  const double r = LDA_SUB(hi, lo);
  const double t = LDA_MUL(r, r);
  const double c =
      LDA_SUB(r, LDA_MUL(t, LDA_ADD(P1, LDA_MUL(t, LDA_ADD(P2, LDA_MUL(t, LDA_ADD(P3, LDA_MUL(t, LDA_ADD(P4, LDA_MUL(t, P5))))))))));
  const double y = LDA_SUB(1.0, LDA_SUB(LDA_SUB(lo, LDA_DIV(LDA_MUL(r, c), LDA_SUB(2.0, c))), hi));
  if (k >= -1021) {
    if (k == 1024) return LDA_MUL(LDA_MUL(y, 2.0), LDA_DBL(0x7FE0000000000000ULL));
    return LDA_DBL(LDA_BITS(y) + ((uint64_t)(int64_t)k << 52));
  }
  /* a subnormal result: one rounding, in the last product */
  return LDA_MUL(LDA_DBL(LDA_BITS(y) + ((uint64_t)(int64_t)(k + 1000) << 52)), LDA_DBL(0x0170000000000000ULL));
}

LDA_FN double lda_log(double x) {
  const double ln2_hi = 6.93147180369123816490e-01, ln2_lo = 1.90821492927058770002e-10;
  const double Lg1 = 6.666666666666735130e-01, Lg2 = 3.999999999940941908e-01, Lg3 = 2.857142874366239149e-01,
               Lg4 = 2.222219843214978396e-01, Lg5 = 1.818357216161805012e-01, Lg6 = 1.531383769920937332e-01,
               Lg7 = 1.479819860511658591e-01;
  uint64_t u = LDA_BITS(x);
  int32_t hx = (int32_t)(u >> 32);
  const uint32_t lx = (uint32_t)u;
  int k = 0;
  if (hx < 0x00100000) { /* x < 2^-1022 */
    if (((hx & 0x7fffffff) | lx) == 0) return -LDA_INF;
    if (hx < 0) return LDA_NAN;
    k -= 54;
    x = LDA_MUL(x, 1.80143985094819840000e+16); /* 2^54 */
    u = LDA_BITS(x);
    hx = (int32_t)(u >> 32);
  }
  if (hx >= 0x7ff00000) return LDA_ADD(x, x);
  k += (hx >> 20) - 1023;
  hx &= 0x000fffff;
  const int32_t i0 = (hx + 0x95f64) & 0x100000;
  x = LDA_DBL(((uint64_t)(uint32_t)(hx | (i0 ^ 0x3ff00000)) << 32) | (u & 0xffffffffULL)); /* x or x / 2 in [sqrt2/2, sqrt2) */
  k += (i0 >> 20);
  const double f = LDA_SUB(x, 1.0);
  const double dk = (double)k;
  if ((0x000fffff & (2 + hx)) < 3) { /* |f| < 2^-20 */
    if (f == 0.0) return k == 0 ? 0.0 : LDA_ADD(LDA_MUL(dk, ln2_hi), LDA_MUL(dk, ln2_lo));
    const double R = LDA_MUL(LDA_MUL(f, f), LDA_SUB(0.5, LDA_MUL(0.33333333333333333, f)));
    if (k == 0) return LDA_SUB(f, R);
    return LDA_SUB(LDA_MUL(dk, ln2_hi), LDA_SUB(LDA_SUB(R, LDA_MUL(dk, ln2_lo)), f));
  }
  const double s = LDA_DIV(f, LDA_ADD(2.0, f));
  const double z = LDA_MUL(s, s), w = LDA_MUL(z, z);
  const int32_t i = (hx - 0x6147a) | (0x6b851 - hx);
  const double t1 = LDA_MUL(w, LDA_ADD(Lg2, LDA_MUL(w, LDA_ADD(Lg4, LDA_MUL(w, Lg6)))));
  const double t2 = LDA_MUL(z, LDA_ADD(Lg1, LDA_MUL(w, LDA_ADD(Lg3, LDA_MUL(w, LDA_ADD(Lg5, LDA_MUL(w, Lg7)))))));
  const double R = LDA_ADD(t2, t1);
  if (i > 0) {
    const double hfsq = LDA_MUL(LDA_MUL(0.5, f), f);
    if (k == 0) return LDA_SUB(f, LDA_SUB(hfsq, LDA_MUL(s, LDA_ADD(hfsq, R))));
    return LDA_SUB(LDA_MUL(dk, ln2_hi),
                   LDA_SUB(LDA_SUB(hfsq, LDA_ADD(LDA_MUL(s, LDA_ADD(hfsq, R)), LDA_MUL(dk, ln2_lo))), f));
  }
  if (k == 0) return LDA_SUB(f, LDA_MUL(s, LDA_SUB(f, R)));
  return LDA_SUB(LDA_MUL(dk, ln2_hi), LDA_SUB(LDA_SUB(LDA_MUL(s, LDA_SUB(f, R)), LDA_MUL(dk, ln2_lo)), f));
}

/* ---- normal and beta draws ----------------------------------------------------------------------------------------- */

#define LDA_HORNER8(r, c0, c1, c2, c3, c4, c5, c6, c7)                                                                   \
  LDA_ADD(LDA_MUL(LDA_ADD(LDA_MUL(LDA_ADD(LDA_MUL(LDA_ADD(LDA_MUL(LDA_ADD(LDA_MUL(LDA_ADD(LDA_MUL(LDA_ADD(LDA_MUL(c7, r), \
  c6), r), c5), r), c4), r), c3), r), c2), r), c1), r), c0)

/* Wichura's AS241 (PPND16): the standard normal quantile of p in (0, 1), relative accuracy about 1e-16 */
LDA_FN double lda_qnorm(double p) {
  if (!(p > 0.0 && p < 1.0)) return p == 0.0 ? -LDA_INF : p == 1.0 ? LDA_INF : LDA_NAN;
  const double q = LDA_SUB(p, 0.5);
  if ((q < 0 ? -q : q) <= 0.425) {
    const double r = LDA_SUB(0.180625, LDA_MUL(q, q));
    return LDA_DIV(LDA_MUL(q, LDA_HORNER8(r, 3.387132872796366608, 133.14166789178437745, 1971.5909503065514427,
                                          13731.693765509461125, 45921.953931549871457, 67265.770927008700853,
                                          33430.575583588128105, 2509.0809287301226727)),
                   LDA_HORNER8(r, 1.0, 42.313330701600911252, 687.1870074920579083, 5394.1960214247511077,
                               21213.794301586595867, 39307.89580009271061, 28729.085735721942674,
                               5226.495278852854561));
  }
  double r = q < 0 ? p : LDA_SUB(1.0, p);
  r = LDA_SQRT(-lda_log(r));
  double val;
  if (r <= 5.0) {
    r = LDA_SUB(r, 1.6);
    val = LDA_DIV(LDA_HORNER8(r, 1.42343711074968357734, 4.6303378461565452959, 5.7694972214606914055,
                              3.64784832476320460504, 1.27045825245236838258, 0.24178072517745061177,
                              0.0227238449892691845833, 7.7454501427834140764e-4),
                  LDA_HORNER8(r, 1.0, 2.05319162663775882187, 1.6763848301838038494, 0.68976733498510000455,
                              0.14810397642748007459, 0.0151986665636164571966, 5.475938084995344946e-4,
                              1.05075007164441684324e-9));
  } else {
    r = LDA_SUB(r, 5.0);
    val = LDA_DIV(LDA_HORNER8(r, 6.6579046435011037772, 5.4637849111641143699, 1.7848265399172913358,
                              0.29656057182850489123, 0.026532189526576123093, 0.0012426609473880784386,
                              2.71155556874348757815e-5, 2.01033439929228813265e-7),
                  LDA_HORNER8(r, 1.0, 0.59983220655588793769, 0.13692988092273580531, 0.0148753612908506148525,
                              7.868691311456132591e-4, 1.8463183175100546818e-5, 1.4215117583164458887e-7,
                              2.04426310338993978564e-15));
  }
  return q < 0 ? -val : val;
}

/* R's norm_rand, INVERSION kind: two draws */
LDA_FN double lda_norm_rand(uint32_t *s) {
  const double big = 134217728.0; /* 2^27 */
  const double u1 = lda_unif(s);
  const double u = LDA_ADD((double)(int)LDA_MUL(big, u1), lda_unif(s));
  return lda_qnorm(LDA_DIV(u, big));
}

/* R's rnorm(mu, sigma) */
LDA_FN double lda_rnorm(double mu, double sigma, uint32_t *s) {
  if (mu != mu || !(sigma >= 0.0) || sigma == LDA_INF) return LDA_NAN;
  if (sigma == 0.0 || mu == LDA_INF || mu == -LDA_INF) return mu;
  return LDA_ADD(mu, LDA_MUL(sigma, lda_norm_rand(s)));
}

/* v = beta log(u1 / (1 - u1)), w = c exp(v) (DBL_MAX past overflow), as R's rbeta forms them */
LDA_FN void lda_beta_vw(double beta, double u1, double c, double *v, double *w) {
  *v = LDA_MUL(beta, lda_log(LDA_DIV(u1, LDA_SUB(1.0, u1))));
  if (*v <= 7.09782712893383973096e+02) {
    *w = LDA_MUL(c, lda_exp(*v));
    if (*w == LDA_INF) *w = LDA_DBL_MAX;
  } else {
    *w = LDA_DBL_MAX;
  }
}

/* rbeta(a0, b0) for finite a0, b0 > 0 (the sampler's 1 + nb / mean_ld, 1 + (m - nb) / mean_ld): Cheng's BB when
 * min(a0, b0) > 1, else BC.  Two draws per trial. */
LDA_FN double lda_rbeta(double a0, double b0, uint32_t *s) {
  const double alpha = LDA_ADD(a0, b0);
  double v, w;
  if ((a0 < b0 ? a0 : b0) > 1.0) { /* BB: a = min, b = max */
    const double a = a0 < b0 ? a0 : b0, b = a0 < b0 ? b0 : a0;
    const double beta = LDA_SQRT(LDA_DIV(LDA_SUB(alpha, 2.0), LDA_SUB(LDA_MUL(LDA_MUL(2.0, a), b), alpha)));
    const double gamma = LDA_ADD(a, LDA_DIV(1.0, beta));
    for (;;) {
      const double u1 = lda_unif(s), u2 = lda_unif(s);
      lda_beta_vw(beta, u1, a, &v, &w);
      const double z = LDA_MUL(LDA_MUL(u1, u1), u2);
      const double r = LDA_SUB(LDA_MUL(gamma, v), 1.3862944);
      const double ss = LDA_SUB(LDA_ADD(a, r), w);
      if (LDA_ADD(ss, 2.609438) >= LDA_MUL(5.0, z)) break;
      const double t = lda_log(z);
      if (ss > t) break;
      if (!(LDA_ADD(r, LDA_MUL(alpha, lda_log(LDA_DIV(alpha, LDA_ADD(b, w))))) < t)) break;
    }
    return a0 == a ? LDA_DIV(w, LDA_ADD(b, w)) : LDA_DIV(b, LDA_ADD(b, w));
  }
  /* BC: a = max, b = min <= 1 */
  const double a = a0 < b0 ? b0 : a0, b = a0 < b0 ? a0 : b0;
  const double beta = LDA_DIV(1.0, b);
  const double delta = LDA_SUB(LDA_ADD(1.0, a), b);
  const double k1 =
      LDA_DIV(LDA_MUL(delta, LDA_ADD(0.0138889, LDA_MUL(0.0416667, b))), LDA_SUB(LDA_MUL(a, beta), 0.777778));
  const double k2 = LDA_ADD(0.25, LDA_MUL(LDA_ADD(0.5, LDA_DIV(0.25, delta)), b));
  for (;;) {
    const double u1 = lda_unif(s), u2 = lda_unif(s);
    double z;
    if (u1 < 0.5) {
      const double y = LDA_MUL(u1, u2);
      z = LDA_MUL(u1, y);
      if (LDA_SUB(LDA_ADD(LDA_MUL(0.25, u2), z), y) >= k1) continue;
    } else {
      z = LDA_MUL(LDA_MUL(u1, u1), u2);
      if (z <= 0.25) {
        lda_beta_vw(beta, u1, a, &v, &w);
        break;
      }
      if (z >= k2) continue;
    }
    lda_beta_vw(beta, u1, a, &v, &w);
    if (LDA_SUB(LDA_MUL(alpha, LDA_ADD(lda_log(LDA_DIV(alpha, LDA_ADD(b, w))), v)), 1.3862944) >= lda_log(z)) break;
  }
  return a0 == a ? LDA_DIV(w, LDA_ADD(b, w)) : LDA_DIV(b, LDA_ADD(b, w));
}

/* ---- the sampler's arithmetic --------------------------------------------------------------------------------------- */

/* One coordinate of the sweep (src/ldpred2-auto.cpp:111-125), in the reference's operation order */
typedef struct {
  double postp, C3, C4, dps;
} lda_coord_t;

LDA_FN lda_coord_t lda_coord(double beta_hat, double dotprod, double cur, double n, double log_var, double shrink,
                             int use_mle, double alpha_plus_one, double sigma2, double inv_odd_p) {
  lda_coord_t o;
  const double res = LDA_SUB(beta_hat, LDA_MUL(shrink, LDA_SUB(dotprod, cur)));
  const double scale_freq = use_mle ? lda_exp(LDA_MUL(alpha_plus_one, log_var)) : 1.0;
  const double C1 = LDA_MUL(LDA_MUL(scale_freq, sigma2), n);
  const double C2 = LDA_DIV(1.0, LDA_ADD(1.0, LDA_DIV(1.0, C1)));
  o.C3 = LDA_MUL(C2, res);
  o.C4 = LDA_DIV(C2, n);
  const double e = lda_exp(LDA_DIV(LDA_DIV(LDA_MUL(-o.C3, o.C3), o.C4), 2.0));
  o.postp = LDA_DIV(1.0, LDA_ADD(1.0, LDA_MUL(LDA_MUL(inv_odd_p, LDA_SQRT(LDA_ADD(1.0, C1))), e)));
  o.dps = LDA_ADD(LDA_MUL(shrink, dotprod), LDA_MUL(LDA_SUB(1.0, shrink), cur));
  return o;
}

/* One coordinate of LDpred2-grid's sweep (src/ldpred2.cpp:39-47, src/ldpred2-sampling.cpp:36-44) from its residual, in
 * the reference's operation order.  The residual is formed by lda_grid_res: ldpred2_gibbs_one takes beta_hat - (dotprod -
 * cur), ldpred2_gibbs_one_sampling (beta_hat + cur) - dotprod, two roundings of the same value. */
typedef struct {
  double postp, C3, C4;
} lda_gcoord_t;

LDA_FN double lda_grid_res(double beta_hat, double dotprod, double cur, int sampling) {
  return sampling ? LDA_SUB(LDA_ADD(beta_hat, cur), dotprod) : LDA_SUB(beta_hat, LDA_SUB(dotprod, cur));
}

LDA_FN lda_gcoord_t lda_grid_coord(double res, double h2_per_var, double n, double inv_odd_p) {
  lda_gcoord_t o;
  const double C1 = LDA_MUL(h2_per_var, n);
  const double C2 = LDA_DIV(1.0, LDA_ADD(1.0, LDA_DIV(1.0, C1)));
  o.C3 = LDA_MUL(C2, res);
  o.C4 = LDA_DIV(C2, n);
  const double e = lda_exp(LDA_DIV(LDA_DIV(LDA_MUL(-o.C3, o.C3), o.C4), 2.0));
  o.postp = LDA_DIV(1.0, LDA_ADD(1.0, LDA_MUL(LDA_MUL(inv_odd_p, LDA_SQRT(LDA_ADD(1.0, C1))), e)));
  return o;
}

/* Whether the coordinate draws its uniform: a sparse point sets beta to 0 without a draw when postp < p */
LDA_FN int lda_grid_draws(int sparse, double postp, double p) { return !(sparse && postp < p); }

/* The draw offset of lane `lane` in a warp whose drawing lanes are the bits of `draws`: the number of uniforms the lanes
 * below it take first.  Its uniform is the (offset + 1)-th from the warp's state, row 2 of A^(offset + 1). */
LDA_FN int lda_grid_offset(uint32_t draws, int lane) {
  const uint32_t below = draws & ((1u << lane) - 1u); /* lane < 32 */
#ifdef __CUDA_ARCH__
  return __popc(below);
#else
  return __builtin_popcount(below);
#endif
}

/* p after a sweep with nb causal variants out of m (src/ldpred2-auto.cpp:166-168) */
LDA_FN double lda_draw_p(int nb, int m, double mean_ld, double p_lo, double p_hi, uint32_t *s) {
  double p = lda_rbeta(LDA_ADD(1.0, LDA_DIV((double)nb, mean_ld)), LDA_ADD(1.0, LDA_DIV((double)(m - nb), mean_ld)), s);
  p = p_lo < p ? p : p_lo; /* std::max(p_lo, p) */
  return p_hi < p ? p_hi : p; /* std::min(., p_hi) */
}

/* MLE_alpha's objective at alpha + 1 = t, profiled over sigma2 in [s2_lo, s2_hi]: with sum_a = sum a_k and
 * C = sum b_k exp(-t a_k), the minimising sigma2 is clamp(C / nb, s2_lo, s2_hi) and f = t sum_a + nb log sigma2 +
 * C / sigma2 (src/optim-MLE-alpha.h:38-48).  f(t, log sigma2) is jointly convex, so this profile is convex in t. */
LDA_FN double lda_mle_profile(double t, double sum_a, double C, int nb, double s2_lo, double s2_hi, double *sigma2) {
  double s2 = LDA_DIV(C, (double)nb);
  if (s2 < s2_lo) s2 = s2_lo;
  if (s2 > s2_hi) s2 = s2_hi;
  *sigma2 = s2;
  return LDA_ADD(LDA_ADD(LDA_MUL(t, sum_a), LDA_MUL((double)nb, lda_log(s2))), LDA_DIV(C, s2));
}

/* Golden-section search for the minimum of a convex function of t on [lo, hi], LDA_GOLDEN_STEPS steps after the four
 * first evaluations (lo, hi and the two inner points), keeping the first of the smallest values seen.  Driven as a
 * state machine so that the device and the CPU restatement share it while evaluating f their own way:
 *   t = lda_golden_start(&g, lo, hi); while (lda_golden_next(&g, f(t), &t)) {}  -> g.best_t */
#define LDA_GOLDEN_STEPS 64
typedef struct {
  double a, b, c, d, fc, fd, best_t, best_f;
  int n;    /* evaluations fed so far */
  int to_d; /* the point asked for last is the new d (else the new c) */
} lda_golden;

LDA_FN double lda_golden_start(lda_golden *g, double lo, double hi) {
  g->a = lo, g->b = hi, g->n = 0, g->to_d = 0;
  g->best_t = lo, g->best_f = LDA_INF;
  return lo;
}

LDA_FN int lda_golden_next(lda_golden *g, double f, double *t) {
  const double invphi = 0.6180339887498949;
  if (g->n == 0 || f < g->best_f) g->best_f = f, g->best_t = *t;
  const int n = g->n++;
  if (n == 0) {
    if (!(g->a < g->b)) return 0;
    *t = g->b;
    return 1;
  }
  if (n == 1) {
    g->c = LDA_SUB(g->b, LDA_MUL(invphi, LDA_SUB(g->b, g->a)));
    *t = g->c;
    return 1;
  }
  if (n == 2) {
    g->fc = f;
    g->d = LDA_ADD(g->a, LDA_MUL(invphi, LDA_SUB(g->b, g->a)));
    *t = g->d;
    g->to_d = 1;
    return 1;
  }
  if (g->to_d)
    g->fd = f;
  else
    g->fc = f;
  if (n - 3 >= LDA_GOLDEN_STEPS) return 0;
  if (g->fc <= g->fd) { /* the minimum lies in [a, d] */
    g->b = g->d, g->d = g->c, g->fd = g->fc;
    g->c = LDA_SUB(g->b, LDA_MUL(invphi, LDA_SUB(g->b, g->a)));
    g->to_d = 0;
    *t = g->c;
  } else { /* in [c, b] */
    g->a = g->c, g->c = g->d, g->fc = g->fd;
    g->d = LDA_ADD(g->a, LDA_MUL(invphi, LDA_SUB(g->b, g->a)));
    g->to_d = 1;
    *t = g->d;
  }
  return 1;
}

#endif /* BSG_LDPRED2_AUTO_CUH */
