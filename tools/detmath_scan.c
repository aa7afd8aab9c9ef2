/* detmath_scan.c -- development tool: the accuracy of the canonical functions (oracle/detmath.h) over every argument
 * the decoder passes them, against long double libm (64-bit significand: ~2^-11 ulp of a double).
 *   sin: every float 0 < |x| <= fl(7 pi)   (pa of the sinc taps, N <= 14)
 *   cos: every float |x| <= fl(pi / 2)      (pa / N of the sinc window)
 *   cos: fl(2 pi_ref) * (s / m), log: s / m, every s in [1, m - 1]   (Box-Muller, noise.py)
 * Prints the largest error of each in ulp of the exact value, and where it is reached; tests/test_detmath.py
 * holds these as its bounds and confirms each worst argument with mpmath.  Then the fp32 noise samples of the
 * generator's whole period with the canonical log / cos against the same formula with this platform's libm log / cos
 * (what noise.py's math.log / math.cos call on glibc): every sample where they differ.
 *
 *     gcc -O2 -ffp-contract=off -fopenmp -o /tmp/detmath_scan tools/detmath_scan.c -lm && /tmp/detmath_scan
 * (about 15 CPU-minutes) */
#include <math.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../oracle/detmath.h"

static double ulperr(double y, long double r) {
    if (r == 0) return y == 0 ? 0 : INFINITY;
    int e;
    frexpl(r, &e);
    return (double)(fabsl((long double)y - r) / ldexpl(1.0L, e - 53));
}
static float f_of(uint32_t b) { float f; memcpy(&f, &b, 4); return f; }
static uint32_t b_of(float f) { uint32_t b; memcpy(&b, &f, 4); return b; }

int main(void) {
    const uint32_t smax = b_of(7.0f * (float)M_PI), cmax = b_of((float)(M_PI / 2));
    double ms = 0, mc = 0;
    float as = 0, ac = 0;
#pragma omp parallel
    {
        double ts = 0, tc = 0;
        float tas = 0, tac = 0;
#pragma omp for schedule(dynamic, 1 << 20)
        for (uint64_t i = 1; i <= 2ull * smax; i++) {
            const uint32_t b = (uint32_t)((i + 1) / 2) | (i & 1 ? 0x80000000u : 0u);
            const float x = f_of(b);
            const double es = ulperr(ccdm_sin((double)x), sinl((long double)x));
            if (es > ts) { ts = es; tas = x; }
            if ((b & 0x7fffffffu) <= cmax) {
                const double ec = ulperr(ccdm_cos((double)x), cosl((long double)x));
                if (ec > tc) { tc = ec; tac = x; }
            }
        }
#pragma omp critical
        {
            if (ts > ms) { ms = ts; as = tas; }
            if (tc > mc) { mc = tc; ac = tac; }
        }
    }
    printf("sin, every float 0 < |x| <= %.9g: max %.4f ulp at x = %.9g\n", f_of(smax), ms, as);
    printf("cos, every float |x| <= %.9g: max %.4f ulp at x = %.9g\n", f_of(cmax), mc, ac);

    const uint64_t m = 2147483647ULL;
    const double pi2 = 2 * 3.14159265359;
    double ml = 0, mb = 0;
    uint64_t sl = 0, sb = 0;
#pragma omp parallel
    {
        double tl = 0, tb = 0;
        uint64_t tsl = 0, tsb = 0;
#pragma omp for schedule(static)
        for (uint64_t s = 1; s < m; s++) {
            const double u = (double)s / (double)m, x = pi2 * u;
            const double el = ulperr(ccdm_log(u), logl((long double)u));
            const double eb = ulperr(ccdm_cos(x), cosl((long double)x));
            if (el > tl) { tl = el; tsl = s; }
            if (eb > tb) { tb = eb; tsb = s; }
        }
#pragma omp critical
        {
            if (tl > ml) { ml = tl; sl = tsl; }
            if (tb > mb) { mb = tb; sb = tsb; }
        }
    }
    printf("log(s / m), every s in [1, m - 1]: max %.4f ulp at s = %llu\n", ml, (unsigned long long)sl);
    printf("cos(2 pi_ref s / m), every s in [1, m - 1]: max %.4f ulp at s = %llu\n", mb, (unsigned long long)sb);

    /* noise samples k in [0, (m - 1) / 2), in blocks that each jump ahead to their first state */
    const uint64_t period = (m - 1) / 2, blk = 1 << 20;
    uint64_t n_diff = 0;
#pragma omp parallel for schedule(dynamic, 1) reduction(+ : n_diff)
    for (uint64_t k0 = 0; k0 < period; k0 += blk) {
        uint64_t seed = 18101995ULL, b = 16807ULL;
        for (uint64_t e = 2 * k0; e; e >>= 1) {
            if (e & 1) seed = (seed * b) % m;
            b = (b * b) % m;
        }
        for (uint64_t k = k0; k < k0 + blk && k < period; k++) {
            seed = (16807ULL * seed) % m;
            const double u1 = (double)seed / (double)m;
            seed = (16807ULL * seed) % m;
            const double u2 = (double)seed / (double)m;
            const float c = (float)(sqrt(-2 * ccdm_log(u1)) * ccdm_cos(pi2 * u2));
            const float l = (float)(sqrt(-2 * log(u1)) * cos(pi2 * u2));
            if (c != l) {
                n_diff++;
#pragma omp critical
                printf("noise sample %llu: canonical %.9g, libm %.9g\n", (unsigned long long)k, c, l);
            }
        }
    }
    printf("noise, every sample of the period [0, %llu): %llu differ from libm\n", (unsigned long long)period,
           (unsigned long long)n_diff);
    return 0;
}
