// ccd_detmath.h -- device flavour (sm_90a) of the canonical elementary functions.
// The oracle holds its own copy of the same operation sequence (oracle/detmath.h, plain C);
// tests/test_detmath.py::test_detmath_device_equals_oracle compares the two bit for bit.
#pragma once
#include <cuda_runtime.h>
#define CCDM_FN static __device__ __forceinline__
#define CCDM_MUL(a, b) __dmul_rn((a), (b))
#define CCDM_ADD(a, b) __dadd_rn((a), (b))
#define CCDM_FMA(a, b, c) __fma_rn((a), (b), (c))
#define CCDM_DIV(a, b) __ddiv_rn((a), (b))
#define CCDM_RINT(a) rint(a)
#define CCDM_D2LL(a) __double_as_longlong(a)
#define CCDM_LL2D(a) __longlong_as_double(a)
/* Canonical double-precision sin / cos / log used where the path needs an elementary function
 * (windowed-sinc warp coefficients, warp.py:226-268; Box-Muller common randomness, noise.py:28-34).
 * The reference evaluates these with its platform's libm (glibc / SLEEF), which no other platform
 * reproduces bit for bit; the CPU oracle and the CUDA kernels therefore share THIS algorithm, built
 * only from IEEE-754 operations that are exactly specified (+, *, fma, /, rint, bit moves), in a fixed
 * order: same input -> same 64 bits on x86-64 and on sm_90a.  Accuracy, in ulp of the exact double, over every
 * argument of the decoder's domain (tools/detmath_scan.c; DESIGN.md, "Canonical elementary functions"):
 *   sin <= 1.46 ulp at every float 0 < |x| <= fl(7 pi)       (the sinc taps, N <= 14)
 *   cos <= 1.41 ulp at every float |x| <= fl(pi / 2)         (the sinc window)
 *   cos <= 1.45 ulp, log <= 2.68 ulp at the Box-Muller arguments fl(2 pi_ref) s / m and s / m, s in [1, m - 1]
 * No bound holds outside that domain: near k pi / 2 the two-term reduction loses relative accuracy where the
 * result is tiny (cos is 451 ulp off at the double nearest 29 pi / 2).
 *   sin / cos: Cody-Waite reduction by pi/2 (two terms), Taylor kernels on [-pi/4, pi/4]
 *   log      : x = m 2^e, m in [sqrt(1/2), sqrt(2)); log m = 2 atanh((m-1)/(m+1)), series to s^23   */
CCDM_FN double ccdm_sin_k(double r) {
    const double z = CCDM_MUL(r, r);
    double p = 0x1.952c77030ad4ap-49;
    p = CCDM_FMA(p, z, -0x1.ae7f3e733b81fp-41);
    p = CCDM_FMA(p, z, 0x1.6124613a86d09p-33);
    p = CCDM_FMA(p, z, -0x1.ae64567f544e4p-26);
    p = CCDM_FMA(p, z, 0x1.71de3a556c734p-19);
    p = CCDM_FMA(p, z, -0x1.a01a01a01a01ap-13);
    p = CCDM_FMA(p, z, 0x1.1111111111111p-7);
    p = CCDM_FMA(p, z, -0x1.5555555555555p-3);
    return CCDM_FMA(CCDM_MUL(r, z), p, r);
}
CCDM_FN double ccdm_cos_k(double r) {
    const double z = CCDM_MUL(r, r);
    double p = 0x1.ae7f3e733b81fp-45;
    p = CCDM_FMA(p, z, -0x1.93974a8c07c9dp-37);
    p = CCDM_FMA(p, z, 0x1.1eed8eff8d898p-29);
    p = CCDM_FMA(p, z, -0x1.27e4fb7789f5cp-22);
    p = CCDM_FMA(p, z, 0x1.a01a01a01a01ap-16);
    p = CCDM_FMA(p, z, -0x1.6c16c16c16c17p-10);
    p = CCDM_FMA(p, z, 0x1.5555555555555p-5);
    p = CCDM_FMA(p, z, -0x1.0000000000000p-1);
    return CCDM_FMA(z, p, 1.0);
}
/* x -> (r, quadrant): x = j pi/2 + r, |r| <= pi/4 (+ rounding) */
CCDM_FN double ccdm_reduce(double x, int *q) {
    const double j = CCDM_RINT(CCDM_MUL(x, 0x1.45f306dc9c883p-1));
    double r = CCDM_FMA(-j, 0x1.921fb54442d18p+0, x);
    r = CCDM_FMA(-j, 0x1.1a62633145c07p-54, r);
    *q = (int)j & 3;
    return r;
}
CCDM_FN double ccdm_sin(double x) {
    int q;
    const double r = ccdm_reduce(x, &q);
    const double v = (q & 1) ? ccdm_cos_k(r) : ccdm_sin_k(r);
    return (q & 2) ? -v : v;
}
CCDM_FN double ccdm_cos(double x) {
    int q;
    const double r = ccdm_reduce(x, &q);
    const double v = (q & 1) ? ccdm_sin_k(r) : ccdm_cos_k(r);
    return ((q + 1) & 2) ? -v : v;
}
/* natural logarithm of a positive normal double */
CCDM_FN double ccdm_log(double x) {
    long long b = CCDM_D2LL(x);
    int e = (int)((b >> 52) & 0x7ff) - 1022;
    b = (b & 0x000fffffffffffffLL) | 0x3fe0000000000000LL; /* m in [0.5, 1) */
    double m = CCDM_LL2D(b);
    if (m < 0x1.6a09e667f3bcdp-1) { /* sqrt(1/2) */
        m = CCDM_MUL(m, 2.0);
        e -= 1;
    }
    const double f = CCDM_ADD(m, -1.0);
    const double s = CCDM_DIV(f, CCDM_ADD(m, 1.0));
    const double z = CCDM_MUL(s, s);
    double p = 0x1.642c8590b2164p-4;
    p = CCDM_FMA(p, z, 0x1.8618618618618p-4);
    p = CCDM_FMA(p, z, 0x1.af286bca1af28p-4);
    p = CCDM_FMA(p, z, 0x1.e1e1e1e1e1e1ep-4);
    p = CCDM_FMA(p, z, 0x1.1111111111111p-3);
    p = CCDM_FMA(p, z, 0x1.3b13b13b13b14p-3);
    p = CCDM_FMA(p, z, 0x1.745d1745d1746p-3);
    p = CCDM_FMA(p, z, 0x1.c71c71c71c71cp-3);
    p = CCDM_FMA(p, z, 0x1.2492492492492p-2);
    p = CCDM_FMA(p, z, 0x1.999999999999ap-2);
    p = CCDM_FMA(p, z, 0x1.5555555555555p-1);
    p = CCDM_FMA(p, z, 0x1.0000000000000p+1);
    const double lm = CCDM_MUL(s, p); /* log(m) */
    return CCDM_FMA((double)e, 0x1.62e42fefa39efp-1, CCDM_FMA((double)e, 0x1.abc9e3b39803fp-56, lm));
}
