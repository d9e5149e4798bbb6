// em_math.h -- the VBEM per-transcript transform  theta = exp(digamma(x) - logNorm)  as ONE branch-light function
// (reference call sites: src/inference/CollapsedEMOptimizer.cpp:119-131,256-272: expTheta[i] =
// exp(digamma(alpha_i + prior_i) - logNorm), 0 when alpha_i + prior_i <= digammaMin).
//
// A Boost-style digamma (log + divisions, a `while (x > 2) result += 1/x` recurrence) followed by exp() lets the
// lanes of a warp take different paths, so a warp executes their union.
// Here:  x' = x (x >= 10)  or  x + 10 (x < 10), and
//     digamma(x) = ln x' - 1/(2x') - sum_{k=1..8} B_2k / (2k x'^2k) - [ 1/x + sum_{k=1..9} 1/(x+k) ]        (x < 10)
// (recurrence digamma(x) = digamma(x+n) - sum_{k<n} 1/(x+k) and the asymptotic series, Abramowitz & Stegun 6.3.5,
// 6.3.18; truncation error at x' >= 10 below 3.1e-18), so that
//     theta = x' * exp(-(1/(2x') + series + 1/x + R(x) + logNorm))
// needs no logarithm; the nine-term sum R(x) is one rational Q'(x)/Q(x), Q = prod_{k=1..9}(x+k), its division and
// 1/x' share one reciprocal.  Absolute error of the exponent ~1e-14 at worst (x ~ 0.01, where digamma ~ -100), i.e. the
// same few-ulp level as the reference's own evaluation; checked against the oracle's digamma in
// tests/test_em_math.py.  Compiles for the host too (the test harness), where the reciprocal is a plain division.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define SB_HD __host__ __device__ __forceinline__
#else
#define SB_HD static inline
#endif

namespace sb {

// 1/a for a normal positive a: hardware seed (about 20 bits) + two Newton steps, error ~1 ulp
SB_HD double fast_rcp(double a) {
#if defined(__CUDA_ARCH__)
  double r;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(a));
  double e = fma(-a, r, 1.0);
  r = fma(r, e, r);
  e = fma(-a, r, 1.0);
  r = fma(r, e, r);
  return r;
#else
  return 1.0 / a;
#endif
}

// exp(digamma(x) - logNorm), x > 0 (callers guard with digammaMin = 1e-10)
SB_HD double exp_digamma_shifted(double x, double logNorm) {
  const bool small = x < 10.0;
  const double xp = small ? x + 10.0 : x;
  double q = 1.0, dq = 0.0;                 // Q(x) = prod (x+k), dq = Q'(x)
  if (small) {
#pragma unroll
    for (int k = 1; k <= 9; ++k) {
      const double f = x + (double)k;
      dq = fma(dq, f, q);
      q *= f;
    }
  }
  const double r = fast_rcp(xp * q);        // 1 / (x' Q)
  const double inv_xp = r * q;              // 1 / x'
  const double rest = dq * (r * xp);        // Q'/Q  (0 when x >= 10)
  const double inv_x = small ? fast_rcp(x) : 0.0;
  const double z = inv_xp * inv_xp;
  // sum_{k=1..8} B_2k / (2k) z^k, two interleaved Horner chains (even / odd powers) for instruction-level parallelism
  const double z2 = z * z;
  double pe = -3617.0 / 8160.0;             // z^8
  pe = fma(pe, z2, -691.0 / 32760.0);       // z^6
  pe = fma(pe, z2, -1.0 / 240.0);           // z^4
  pe = fma(pe, z2, -1.0 / 120.0);           // z^2
  double po = 1.0 / 12.0;                   // z^7
  po = fma(po, z2, 1.0 / 132.0);            // z^5
  po = fma(po, z2, 1.0 / 252.0);            // z^3
  po = fma(po, z2, 1.0 / 12.0);             // z^1
  const double series = z * fma(pe, z, po); // z*(po + z*pe)
  const double e = (fma(0.5, inv_xp, series) + rest) + (inv_x + logNorm);
  return xp * exp(-e);
}

}  // namespace sb
