// float sine / cosine with the SAME results as glibc's sinf / cosf / sincosf (sysdeps/ieee754/flt-32/s_sincosf.h,
// glibc >= 2.28; this image: 2.39), for |x| < 120 — every angle a SLAM pose can hold.  The reference's Hector code
// takes std::sin / std::cos of a float pose angle (Eigen::Rotation2Df, GridMapBase.h:238-242, OccGridMapUtil.h:437-440)
// and truncates the transformed coordinates to cell indices, so a last-ulp difference moves Bresenham cells; CUDA's
// sinf/cosf are different (equally valid) roundings.  glibc evaluates a double-precision polynomial after a
// one-multiply range reduction and rounds once to float; the steps below restate that published algorithm.
// x86-64 glibc selects an FMA build of the same source when the CPU has FMA (ifunc): every `a + b * c` of the source
// is then one fused operation.  `FMA` picks the variant; the host probes which one its libm uses
// (glibc_sincosf_variant_of_host) so the device follows the machine's own reference arithmetic.
// Host + device code: tests/glibc_math_check.cpp runs the same functions on the CPU against the C library.
#pragma once

#include <math.h>
#include <stdint.h>
#include <string.h>

#if defined(__CUDACC__)
#define B2S_HD __host__ __device__ __forceinline__
#else
#define B2S_HD static inline
#endif

namespace b2s {

B2S_HD double gm_madd(double a, double b, double c, bool use_fma) {  // a * b + c as the selected glibc build rounds it
#if defined(__CUDA_ARCH__)
  return use_fma ? fma(a, b, c) : __dadd_rn(__dmul_rn(a, b), c);
#else
  if (use_fma) return fma(a, b, c);
  volatile double p = a * b;  // keep the product's rounding even if the host compiler would contract
  return p + c;
#endif
}

B2S_HD uint32_t gm_asuint(float x) {
#if defined(__CUDA_ARCH__)
  return __float_as_uint(x);
#else
  uint32_t u;
  memcpy(&u, &x, 4);
  return u;
#endif
}

// polynomial of quadrant n (odd: cosine polynomial) on the reduced argument; `neg` = the negated coefficient set that
// glibc uses for quadrants 2, 3
B2S_HD float gm_sinf_poly(double x, double x2, bool neg, int n, bool use_fma) {
  const double sg = neg ? -1.0 : 1.0;
  const double c0 = sg * 0x1p0, c1 = sg * -0x1.ffffffd0c621cp-2, c2 = sg * 0x1.55553e1068f19p-5,
               c3 = sg * -0x1.6c087e89a359dp-10, c4 = sg * 0x1.99343027bf8c3p-16;
  const double s1 = -0x1.555545995a603p-3, s2 = 0x1.1107605230bc4p-7, s3 = -0x1.994eb3774cf24p-13;
  if ((n & 1) == 0) {
    const double x3 = x * x2;
    const double t1 = gm_madd(x2, s3, s2, use_fma);
    const double x7 = x3 * x2;
    const double s = gm_madd(x3, s1, x, use_fma);
    return (float)gm_madd(x7, t1, s, use_fma);
  }
  const double x4 = x2 * x2;
  const double t2 = gm_madd(x2, c4, c3, use_fma);
  const double t1 = gm_madd(x2, c1, c0, use_fma);
  const double x6 = x4 * x2;
  const double c = gm_madd(x4, c2, t1, use_fma);
  return (float)gm_madd(x6, t2, c, use_fma);
}

// which: 0 = sine, 1 = cosine.  Returns false (result untouched) outside the supported range (|y| >= 120, inf, NaN).
B2S_HD bool gm_sincosf_one(float y, int which, bool use_fma, float *out) {
  const uint32_t top = (gm_asuint(y) >> 20) & 0x7ffu;
  double x = (double)y;
  if (top < 0x3f4u) {  // |y| < pi/4 (abstop12(0x1.921FB6p-1f))
    if (top < 0x398u) {  // |y| < 2^-12
      *out = which ? 1.0f : y;
      return true;
    }
    *out = gm_sinf_poly(x, x * x, false, which, use_fma);
    return true;
  }
  if (top < 0x42fu) {  // |y| < 120
    const double hpi_inv = 0x1.45F306DC9C883p+23, hpi = 0x1.921FB54442D18p0;
    const double r = x * hpi_inv;
    const int n = (int)(((int32_t)r + 0x800000) >> 24);
    x = gm_madd(-(double)n, hpi, x, use_fma);
    const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;  // { 1, -1, -1, 1 }
    *out = gm_sinf_poly(x * sign, x * x, (n & 2) != 0, n ^ which, use_fma);
    return true;
  }
  return false;
}

// sincosf(y): both values from one range reduction (glibc's sincosf shares it too and returns the same floats as
// sinf / cosf — the host check compares all three)
B2S_HD void glibc_sincosf(float y, bool use_fma, float *sp, float *cp) {
  const uint32_t top = (gm_asuint(y) >> 20) & 0x7ffu;
  double x = (double)y;
  if (top < 0x3f4u) {
    if (top < 0x398u) { *sp = y; *cp = 1.0f; return; }
    const double x2 = x * x;
    *sp = gm_sinf_poly(x, x2, false, 0, use_fma);
    *cp = gm_sinf_poly(x, x2, false, 1, use_fma);
    return;
  }
  if (top < 0x42fu) {
    const double hpi_inv = 0x1.45F306DC9C883p+23, hpi = 0x1.921FB54442D18p0;
    const double r = x * hpi_inv;
    const int n = (int)(((int32_t)r + 0x800000) >> 24);
    x = gm_madd(-(double)n, hpi, x, use_fma);
    const double sign = ((n & 3) == 1 || (n & 3) == 2) ? -1.0 : 1.0;
    const double xs = x * sign, x2 = x * x;
    *sp = gm_sinf_poly(xs, x2, (n & 2) != 0, n, use_fma);
    *cp = gm_sinf_poly(xs, x2, (n & 2) != 0, n ^ 1, use_fma);
    return;
  }
  *sp = sinf(y);
  *cp = cosf(y);
}

B2S_HD float glibc_sinf(float y, bool use_fma) {
  float r;
  if (gm_sincosf_one(y, 0, use_fma, &r)) return r;
  return sinf(y);  // |y| >= 120: outside the restated range (never a pose angle); library sine
}
B2S_HD float glibc_cosf(float y, bool use_fma) {
  float r;
  if (gm_sincosf_one(y, 1, use_fma, &r)) return r;
  return cosf(y);
}

// The reference's unqualified sin / cos of a float (OccGridMapUtil.h:87-88): the C library's DOUBLE functions, rounded to
// float.  The device takes its own double sincos (within 2 double ulps of the exact value), so the two floats could only
// differ where the exact value lies within a few double ulps of a float rounding boundary; tests/device_math_check.cu
// compares every float with |a| <= 16 against the C library and finds none that differ.
B2S_HD void libm_sincos_to_float(float a, float *s, float *c) {
#if defined(__CUDA_ARCH__)
  double ds, dc;
  sincos((double)a, &ds, &dc);
#else
  const double ds = sin((double)a), dc = cos((double)a);
#endif
  *s = (float)ds;
  *c = (float)dc;
}

// (host function)
// Which build of s_sincosf does THIS host's libm run?  1 = FMA, 0 = separate multiply / add, -1 = neither restatement
// reproduces it on the probe inputs (an unknown libm: callers fall back to 1 and report it).  The two builds differ on
// exactly 34 of the 2 246 049 792 floats with |x| < 120 (all with |x| > 17.2, next to multiples of pi/2 where the
// reduction cancels); the probes are those inputs, so for pose angles (|x| < 2 pi + 14 * 0.2) the variant is immaterial.
inline int glibc_sincosf_variant_of_host() {
  static const uint32_t probes[17] = {0x418a3adbu, 0x418a3adcu, 0x418a3addu, 0x418a3adeu, 0x41bc76d9u, 0x4202eb4bu,
                                      0x4255b0a9u, 0x42687a55u, 0x4280ce28u, 0x42870e40u, 0x42a35c07u, 0x42a35d44u,
                                      0x42a97360u, 0x42c55faau, 0x42cf5854u, 0x42d8d23eu, 0x42e87a55u};
  int ok[2] = {1, 1};
  for (int i = 0; i < 17; i++)
    for (int sg = 0; sg < 2; sg++) {
      const uint32_t bits = probes[i] | (sg ? 0x80000000u : 0u);
      float y;
      memcpy(&y, &bits, 4);
      volatile float vy = y;
      const float hs = sinf(vy), hc = cosf(vy);
      for (int v = 0; v < 2; v++)
        if (glibc_sinf(y, v != 0) != hs || glibc_cosf(y, v != 0) != hc) ok[v] = 0;
    }
  if (ok[1]) return 1;
  if (ok[0]) return 0;
  return -1;
}

}  // namespace b2s
