"""The canonical elementary functions (oracle/detmath.h, csrc/ccd_detmath.h) and what is built from them.

The windowed-sinc warp taps and the common-randomness (CR) noise are evaluated with one sin / cos / log
algorithm, built from exactly specified IEEE-754 operations in a fixed order, so that the CPU oracle and
the kernels return the same 64 bits.  This module proves that, and how far that algorithm is from the
libm calls the reference makes:

- CPU: accuracy against a high-precision reference (long double, checked by mpmath at 200 bits) on
  every argument the sinc taps form and on the Box-Muller arguments; a third implementation (a Python
  restatement of detmath.h with exactly rounded fma) equal to the oracle bit for bit; negative controls
  that a plausible wrong variant of that restatement fails; the taps against the reference's own fp32
  formula; the noise against the reference's generator over a 3840x2160 frame with 8 grids.
- GPU: ccd_debug_detmath / ccd_debug_sinc_coeffs / ccd_debug_cr_noise against the oracle bit for bit,
  and a full-size CR decode against the oracle.

tools/gpu_detmath.py extends the device / oracle comparison to every Box-Muller argument and to the
generator's whole period.
"""
import math
import struct
from fractions import Fraction

import numpy as np
import pytest

M = 2**31 - 1                      # Park-Miller modulus (noise.py)
A = 16807
SEED0 = 18101995
PI_REF = 3.14159265359             # the reference's pi in Box-Muller (noise.py)
TAPS = (6, 8, 10, 12, 14)          # every windowed-sinc size the header can carry
PI_F = np.float32(math.pi)
CR_4K = 11059110                   # noise samples of a 3840x2160 frame with 8 grids
SQRT_HALF_S = int(math.sqrt(0.5) * M)

# Bounds, in ulp of the double result, and the arguments where they are reached.  tools/detmath_scan.c evaluates
# every argument of the decoder's domain against long double: sin at every float 0 < |x| <= fl(7 pi) (every pa the
# sinc taps form), cos at every float |x| <= fl(pi / 2) (every pa / N) and at fl(2 pi_ref) s / m for every
# s in [1, m - 1] (Box-Muller), log at s / m for every s.  The worst arguments are in the sets below, where mpmath
# confirms them.  Outside that domain the two-term Cody-Waite reduction loses relative accuracy where the result is
# tiny: see test_adversarial_arguments_recorded.
SIN_ULP, COS_ULP, LOG_ULP = 1.46, 1.45, 2.68
SIN_WORST, COS_WORST_SINC = float(np.float32(-15.2038345)), float(np.float32(-1.06369293))
LOG_WORST_S, COS_WORST_S = 1515289142, 1599930950
# Measured maximum distance of a canonical sinc tap from the reference's fp32 formula, in fp32 ulp
TAP_REF_ULP = 3


# ----------------------------------------------------------------------------------------------
# argument sets
def sinc_offsets(n=2**16, seed=3):
    """About 2^16 fractional offsets in [0, 1) and the edges: 0, the smallest subnormal, the smallest normal,
    0.5 and its two neighbours, the largest float below 1."""
    rng = np.random.default_rng(seed)
    s = rng.random(n, dtype=np.float32)
    f32 = np.float32
    edges = [f32(0), np.nextafter(f32(0), f32(1)), np.finfo(np.float32).tiny, f32(0.5),
             np.nextafter(f32(0.5), f32(0)), np.nextafter(f32(0.5), f32(1)), np.nextafter(f32(1), f32(0))]
    return np.concatenate([np.asarray(edges, np.float32), s])


def sinc_arguments(offsets):
    """Every double the N-tap sinc forms, for every N: pa = fp32(pi_f * (s - j)) (sin, where s - j != 0) and
    fp32(pa / N) (cos), and the worst float of the scan for each.  Returns (sin arguments, cos arguments), unique."""
    sin_x, cos_x = [], []
    for n in TAPS:
        for k in range(n):
            arg = offsets - np.float32(-(n // 2) + 1 + k)
            pa = PI_F * arg
            sin_x.append(pa[arg != 0])
            cos_x.append(pa / np.float32(n))
    sin_x.append(np.float32([SIN_WORST]))
    cos_x.append(np.float32([COS_WORST_SINC]))
    return np.unique(np.concatenate(sin_x).astype(np.float64)), np.unique(np.concatenate(cos_x).astype(np.float64))


def box_muller_s(n=2**18, seed=5):
    """LCG states s: a random sample of [1, m - 1], s = 1, 2, m - 1, m - 2, the s around sqrt(1/2) m and
    around every power of two, and the worst s of the scan for log and for cos."""
    rng = np.random.default_rng(seed)
    s = [rng.integers(1, M, n, dtype=np.int64)]
    s.append(np.array([1, 2, M - 1, M - 2, LOG_WORST_S, COS_WORST_S], np.int64))
    s.append(np.arange(SQRT_HALF_S - 2048, SQRT_HALF_S + 2048, dtype=np.int64))
    # u = s / m just below and above 2^-k (s near m 2^-k) and s near 2^k
    for k in range(1, 31):
        for c in (M >> k, 1 << k):
            s.append(np.arange(max(c - 4, 1), min(c + 5, M), dtype=np.int64))
    return np.unique(np.concatenate(s))


def box_muller_arguments(s):
    """(log arguments u1 = s / m, cos arguments fl(2 pi_ref) * (s / m)) as noise.py forms them."""
    u = s.astype(np.float64) / float(M)
    return u, (2 * PI_REF) * u


def adversarial_arguments():
    """The doubles nearest k pi / 2, k = 1 ... 40, and 1.0."""
    import mpmath

    mpmath.mp.prec = 200
    return np.array([float(k * mpmath.pi / 2) for k in range(1, 41)] + [1.0])


# ----------------------------------------------------------------------------------------------
# high-precision reference
def _ld_ref(fn, x):
    assert np.finfo(np.longdouble).nmant >= 63, "the long double reference needs at least a 64-bit significand"
    xl = x.astype(np.longdouble)
    return {"sin": np.sin, "cos": np.cos, "log": np.log}[fn](xl)


def ulp_error(y, ref):
    """|y - ref| in ulp of the exact value ref (ulp(r) = 2^(e - 53) for r = f 2^e, f in [0.5, 1))."""
    ref = np.asarray(ref, dtype=np.longdouble)
    _, e = np.frexp(ref)
    u = np.ldexp(np.ones_like(ref), e - 53)
    return np.asarray(np.abs(y.astype(np.longdouble) - ref) / u, dtype=np.float64)


def mp_ulp_error(fn, x, y):
    """The same error with the exact value from mpmath at 200 bits."""
    import mpmath

    mpmath.mp.prec = 200
    f = {"sin": mpmath.sin, "cos": mpmath.cos, "log": mpmath.log}[fn]
    out = []
    for xi, yi in zip(x.tolist(), y.tolist()):
        r = f(mpmath.mpf(xi))
        _, e = mpmath.frexp(r)
        out.append(float(abs(mpmath.mpf(yi) - r) / mpmath.ldexp(1, e - 53)))
    return np.array(out)


def checked_max_error(fn, x, y, n_check=300):
    """Max ulp error of y = fn(x) by the long double reference, confirmed by mpmath on the n_check worst
    arguments and on n_check others: the two references agree to 0.01 ulp there.  Returns (max, argmax x)."""
    err = ulp_error(y, _ld_ref(fn, x))
    worst = np.argsort(err)[-n_check:]
    other = np.random.default_rng(7).choice(x.size, min(n_check, x.size), replace=False)
    idx = np.unique(np.concatenate([worst, other]))
    mp = mp_ulp_error(fn, x[idx], y[idx])
    assert np.abs(mp - err[idx]).max() < 0.01
    i = int(idx[np.argmax(mp)])
    return float(mp.max()), float(x[i])


# ----------------------------------------------------------------------------------------------
# third implementation: detmath.h restated in Python, fma exactly rounded through Fraction
def fma(a, b, c):
    r = Fraction(a) * Fraction(b) + Fraction(c)
    if r == 0:  # IEEE-754 sign of an exact zero sum in round-to-nearest
        neg_prod = (math.copysign(1.0, a) * math.copysign(1.0, b)) < 0
        return -0.0 if (a * b == 0 and c == 0 and neg_prod and math.copysign(1.0, c) < 0) else 0.0
    return float(r)  # int / int true division: correctly rounded


SIN_C = [float.fromhex(h) for h in ("0x1.952c77030ad4ap-49", "-0x1.ae7f3e733b81fp-41", "0x1.6124613a86d09p-33",
                                    "-0x1.ae64567f544e4p-26", "0x1.71de3a556c734p-19", "-0x1.a01a01a01a01ap-13",
                                    "0x1.1111111111111p-7", "-0x1.5555555555555p-3")]
COS_C = [float.fromhex(h) for h in ("0x1.ae7f3e733b81fp-45", "-0x1.93974a8c07c9dp-37", "0x1.1eed8eff8d898p-29",
                                    "-0x1.27e4fb7789f5cp-22", "0x1.a01a01a01a01ap-16", "-0x1.6c16c16c16c17p-10",
                                    "0x1.5555555555555p-5", "-0x1.0000000000000p-1")]
LOG_C = [float.fromhex(h) for h in ("0x1.642c8590b2164p-4", "0x1.8618618618618p-4", "0x1.af286bca1af28p-4",
                                    "0x1.e1e1e1e1e1e1ep-4", "0x1.1111111111111p-3", "0x1.3b13b13b13b14p-3",
                                    "0x1.745d1745d1746p-3", "0x1.c71c71c71c71cp-3", "0x1.2492492492492p-2",
                                    "0x1.999999999999ap-2", "0x1.5555555555555p-1", "0x1.0000000000000p+1")]
TWO_OVER_PI = float.fromhex("0x1.45f306dc9c883p-1")
PIO2_HI, PIO2_LO = float.fromhex("0x1.921fb54442d18p+0"), float.fromhex("0x1.1a62633145c07p-54")
SQRT_HALF = float.fromhex("0x1.6a09e667f3bcdp-1")
LN2_HI, LN2_LO = float.fromhex("0x1.62e42fefa39efp-1"), float.fromhex("0x1.abc9e3b39803fp-56")


class Restated:
    """detmath.h, operation by operation.  The keyword arguments make the plausible wrong variants the
    negative controls need: cw2=False drops the second Cody-Waite term, log_terms=11 ends the atanh series
    one term short."""

    def __init__(self, cw2=True, log_terms=12):
        self.cw2, self.log_terms = cw2, log_terms

    @staticmethod
    def _poly(c, z):
        p = c[0]
        for ci in c[1:]:
            p = fma(p, z, ci)
        return p

    def sin_k(self, r):
        z = r * r
        return fma(r * z, self._poly(SIN_C, z), r)

    def cos_k(self, r):
        z = r * r
        return fma(z, self._poly(COS_C, z), 1.0)

    def reduce(self, x):
        j = float(round(x * TWO_OVER_PI))  # rint: round half to even
        r = fma(-j, PIO2_HI, x)
        if self.cw2:
            r = fma(-j, PIO2_LO, r)
        return r, int(j) & 3

    def sin(self, x):
        r, q = self.reduce(x)
        v = self.cos_k(r) if q & 1 else self.sin_k(r)
        return -v if q & 2 else v

    def cos(self, x):
        r, q = self.reduce(x)
        v = self.sin_k(r) if q & 1 else self.cos_k(r)
        return -v if (q + 1) & 2 else v

    def log(self, x):
        b = struct.unpack("<q", struct.pack("<d", x))[0]
        e = ((b >> 52) & 0x7FF) - 1022
        m = struct.unpack("<d", struct.pack("<q", (b & 0x000FFFFFFFFFFFFF) | 0x3FE0000000000000))[0]
        if m < SQRT_HALF:
            m, e = m * 2.0, e - 1
        f = m + -1.0
        s = f / (m + 1.0)
        z = s * s
        lm = s * self._poly(LOG_C[12 - self.log_terms:], z)
        return fma(float(e), LN2_HI, fma(float(e), LN2_LO, lm))

    def __call__(self, fn, x):
        f = getattr(self, fn)
        return np.array([f(v) for v in np.asarray(x, np.float64).tolist()])


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


# ----------------------------------------------------------------------------------------------
# the reference's own formulas
def reference_taps(n, s):
    """warp.py get_coeffs for the N-tap sinc, in CPU torch fp32 as the reference evaluates it: [len(s), N]."""
    import torch

    k = torch.arange(-(n // 2) + 1, n // 2 + 1, dtype=torch.float32)
    d = torch.from_numpy(np.asarray(s, np.float32))[:, None] - k[None, :]
    return (torch.cos(torch.pi * d / n) * torch.sinc(d)).numpy()


def lcg_states(first_state, count):
    """LCG states first_state ... first_state + count - 1 (state 0 = the seed), vectorised by jumps of 2^16."""
    B = 1 << 16
    s = np.empty(count + B, dtype=np.uint64)
    x = SEED0 * pow(A, first_state, M) % M
    blk = [x]
    for _ in range(B - 1):
        x = A * x % M
        blk.append(x)
    s[:B] = blk
    aB = np.uint64(pow(A, B, M))
    for o in range(B, count, B):
        s[o:o + B] = s[o - B:o] * aB % np.uint64(M)
    return s[:count]


def noise_uniforms(first, n):
    """(u1, u2) of noise samples [first, first + n): sample k draws LCG states 2k + 1 and 2k + 2."""
    st = lcg_states(2 * first + 1, 2 * n).astype(np.float64) / float(M)
    return st[0::2], st[1::2]


def libm_noise(u1, u2):
    """noise.py grand() with the calls the reference makes (math.log, math.cos, math.sqrt), in float64."""
    lg = np.fromiter(map(math.log, u1.tolist()), np.float64, u1.size)
    cs = np.fromiter(map(math.cos, ((2 * PI_REF) * u2).tolist()), np.float64, u2.size)
    return np.sqrt(-2 * lg) * cs


def canonical_noise(oracle, u1, u2, pi=PI_REF):
    """The same with the canonical log / cos of the oracle, in float64 (before the rounding to fp32)."""
    return np.sqrt(-2 * oracle.detmath("log", u1)) * oracle.detmath("cos", (2 * pi) * u2)


def tie_distance(v):
    """Distance of each float64 v from the nearest fp32 rounding tie, in float64 ulp of v."""
    r = v.astype(np.float32)
    up = r.astype(np.float64) <= v
    lo = np.where(up, r, np.nextafter(r, np.float32(-np.inf)))
    hi = np.where(up, np.nextafter(r, np.float32(np.inf)), r)
    mid = (lo.astype(np.float64) + hi.astype(np.float64)) / 2  # exact: 25 significant bits
    return np.abs(v - mid) / np.spacing(np.abs(v))


# Window around an fp32 tie inside which the canonical and the libm noise may round differently, in float64 ulp of
# the value: relative errors, in units of 2^-52, of sqrt(-2 log u1) * cos(x) -- canonical: LOG_ULP / 2 (the sqrt
# halves it) + 0.5 (sqrt) + COS_ULP + 0.5 (product); glibc: at most 1 ulp for log and cos -- and a relative error
# of 2^-52 is at most 2 ulp of the value.
TIE_WINDOW = 2 * ((LOG_ULP / 2 + 0.5 + COS_ULP + 0.5) + (0.5 + 0.5 + 1.0 + 0.5))


def mp_noise(u1, u2):
    """The exact sqrt(-2 ln u1) cos(fl(2 pi_ref) u2) of the two doubles, as an mpmath number at 200 bits."""
    import mpmath

    mpmath.mp.prec = 200
    return mpmath.sqrt(-2 * mpmath.log(mpmath.mpf(float(u1)))) * mpmath.cos(mpmath.mpf(float((2 * PI_REF) * u2)))


def mp_correct_fp32(u1, u2):
    """The fp32 value nearest the exact noise sample (decided at 200 bits)."""
    import mpmath

    v = mp_noise(u1, u2)
    f = np.float32(float(v))
    lo, hi = (f, np.nextafter(f, np.float32(np.inf))) if mpmath.mpf(float(f)) <= v else \
        (np.nextafter(f, np.float32(-np.inf)), f)
    mid = (mpmath.mpf(float(lo)) + mpmath.mpf(float(hi))) / 2
    assert v != mid
    return lo if v < mid else hi


# ----------------------------------------------------------------------------------------------
# CPU tests
@pytest.fixture(scope="module")
def sinc_set():
    return sinc_arguments(sinc_offsets())


@pytest.fixture(scope="module")
def bm_set():
    return box_muller_arguments(box_muller_s())


def test_argument_sets(sinc_set, bm_set):
    """The sets reach what they are meant to: the sinc arguments up to |pa| = 7 pi (N = 14, s -> 1 - 2^-24) and
    subnormal and tiny offsets; the Box-Muller ones the whole (0, 2 pi_ref) and u on both sides of sqrt(1/2)."""
    sx, cx = sinc_set
    assert 20.0 < np.abs(sx).max() < 7 * math.pi + 1e-5 and np.abs(cx).max() < math.pi / 2 + 1e-6
    assert np.abs(sx).min() < 1e-6 and sx.size > 900_000 and cx.size > 2_500_000
    assert cx.min() < 0 < cx.max()
    u, x = bm_set
    assert u.min() == 1 / M and u.max() == (M - 1) / M and x.max() < 2 * PI_REF
    assert ((u < SQRT_HALF) & (u > SQRT_HALF - 1e-6)).sum() > 1000 and ((u >= SQRT_HALF) & (u < SQRT_HALF + 1e-6)).sum() > 1000


@pytest.mark.parametrize("fn", ["sin", "cos", "log"])
def test_accuracy_against_mpmath(oracle, sinc_set, bm_set, fn):
    """The canonical functions of the oracle within the stated bound of the exact value, on every argument the
    sinc taps form (sin, cos) and on the Box-Muller arguments (log, cos)."""
    sets = {"sin": [("sinc", sinc_set[0])], "cos": [("sinc", sinc_set[1]), ("box-muller", bm_set[1])],
            "log": [("box-muller", bm_set[0])]}[fn]
    bound = {"sin": SIN_ULP, "cos": COS_ULP, "log": LOG_ULP}[fn]
    for name, x in sets:
        worst, at = checked_max_error(fn, x, oracle.detmath(fn, x))
        print(f"{fn} on the {name} arguments ({x.size}): max {worst:.3f} ulp at x = {at!r}")
        assert worst <= bound, (fn, name, worst, at)
        # the worst argument of the scan is the worst of the set
        assert at == {("sin", "sinc"): SIN_WORST, ("cos", "sinc"): COS_WORST_SINC,
                      ("cos", "box-muller"): (2 * PI_REF) * (COS_WORST_S / M), ("log", "box-muller"): LOG_WORST_S / M}[fn, name]


def test_adversarial_arguments_recorded(oracle):
    """Outside the decoder's domain the bounds do not hold: near k pi / 2 the result is tiny and the two-term
    Cody-Waite reduction's absolute error j 2^-106 (and the rounding of x - j pi/2) is not small against it.
    Recorded here so that the documented domain is the one where the bounds were measured."""
    x = adversarial_arguments()
    worst = {}
    for fn in ("sin", "cos"):
        err = mp_ulp_error(fn, x, oracle.detmath(fn, x))
        worst[fn] = (float(err.max()), int(np.argmax(err)) + 1)
        print(f"{fn} near k pi / 2, k <= 40: max {err.max():.1f} ulp at k = {np.argmax(err) + 1}; "
              f"k <= 16 (|x| < 8 pi): max {err[:16].max():.2f} ulp")
        # inside |x| < 8 pi the bound holds even at these arguments
        assert err[:16].max() <= {"sin": SIN_ULP, "cos": COS_ULP}[fn]
    # 29 pi / 2 ~ 45.55: cos is 451 ulp off; no decoder path passes such an argument
    assert worst["cos"][1] == 29 and 400 < worst["cos"][0] < 500
    assert mp_ulp_error("log", x[-1:], oracle.detmath("log", x[-1:]))[0] == 0.0  # log 1 = 0 exactly


def _restatement_sample(sinc_set, bm_set, n=1500, seed=11):
    rng = np.random.default_rng(seed)
    sx, cx = sinc_set
    u, x = bm_set
    pick = lambda a: a[rng.choice(a.size, n, replace=False)]  # noqa: E731
    adv = adversarial_arguments()
    return {"sin": np.concatenate([pick(sx), sx[:20], sx[-20:], adv]),
            "cos": np.concatenate([pick(cx), pick(x), cx[:20], cx[-20:], adv]),
            "log": np.concatenate([pick(u), u[:50], u[-50:], [LOG_WORST_S / M, 1.0, 2.0, 0.5, 1e-300, 1e300]])}


def test_restatement_equals_oracle(oracle, sinc_set, bm_set):
    """A third implementation: detmath.h restated in Python with exactly rounded fma equals the oracle bit for bit,
    on a few thousand arguments of every set (and on the adversarial ones)."""
    R = Restated()
    for fn, x in _restatement_sample(sinc_set, bm_set).items():
        got, want = R(fn, x), oracle.detmath(fn, x)
        assert np.array_equal(bits(got), bits(want)), (fn, x[bits(got) != bits(want)][:5])


def test_negative_controls(oracle, sinc_set, bm_set):
    """Every bound above fails for a plausible wrong variant of the computation it checks."""
    sample = _restatement_sample(sinc_set, bm_set, n=400)
    fired = {}

    # Cody-Waite reduction without its second term: sin / cos off by far more than the bound on the sinc set, and
    # no longer the oracle's bits
    R = Restated(cw2=False)
    for fn, bound in (("sin", SIN_ULP), ("cos", COS_ULP)):
        x = sample[fn]
        y = R(fn, x)
        e = ulp_error(y, _ld_ref(fn, x))
        assert e.max() > 10 * bound and not np.array_equal(bits(y), bits(oracle.detmath(fn, x)))
        fired[f"cw1 {fn}"] = f"max {e.max():.3g} ulp"

    # the log series one term short: the truncation (< 0.01 ulp) hides inside the accuracy bound, but the bits differ
    # from the oracle's -- the bit-for-bit comparison is the bound that catches it
    x = sample["log"]
    y = Restated(log_terms=11)("log", x)
    diff = int((bits(y) != bits(oracle.detmath("log", x))).sum())
    assert diff > 0
    fired["log short"] = f"{diff} of {x.size} results differ from the oracle"

    # pi instead of 3.14159265359 in Box-Muller: the noise is no longer the reference's outside the tie window
    # (pi - pi_ref is 2e-13: a few samples in 10^5 round the other way)
    u1, u2 = noise_uniforms(0, 1 << 20)
    ref = libm_noise(u1, u2).astype(np.float32)
    wrong = canonical_noise(oracle, u1, u2, pi=math.pi)
    bad = (wrong.astype(np.float32) != ref) & (tie_distance(wrong) > TIE_WINDOW)
    assert bad.sum() > 10
    fired["pi"] = f"{int(bad.sum())} of {1 << 20} samples differ outside the tie window"

    # the sinc window divided by N - 1: taps further from the reference's than the bound
    s = sinc_offsets(4096)
    worst = 0
    for n in TAPS:
        t = restated_taps(oracle, n, s, window_div=n - 1)
        worst = max(worst, int(fp32_ulp_distance(t, reference_taps(n, s)).max()))
    assert worst > TAP_REF_ULP
    fired["window / (N - 1)"] = f"{worst} fp32 ulp from the reference"
    print("negative controls fired:", fired)


def restated_taps(oracle, n, s, window_div=None):
    """sinc_coeffs with the oracle's canonical sin / cos and numpy fp32 operations: [len(s), N]."""
    s = np.asarray(s, np.float32)
    out = np.empty((s.size, n), np.float32)
    for k in range(n):
        arg = s - np.float32(-(n // 2) + 1 + k)
        pa = PI_F * arg
        win = oracle.detmath("cos", (pa / np.float32(window_div or n)).astype(np.float64))
        nz = arg != 0
        sc = np.ones(s.size)
        sc[nz] = oracle.detmath("sin", pa[nz].astype(np.float64)) / pa[nz].astype(np.float64)
        out[:, k] = win.astype(np.float32) * sc.astype(np.float32)
    return out


def fp32_ulp_distance(a, b):
    """Number of fp32 values between a and b (the ulp distance on the ordered fp32 line)."""
    def key(x):
        i = np.asarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(key(a) - key(b))


def test_sinc_taps(oracle):
    """The canonical taps: equal to their restatement; within 3 x 2^-24 (relative) of the exact windowed sinc at the
    same fp32 arguments pa and pa / N -- the three fp32 roundings of window, sinc and product, nothing else; at the
    integer taps of offsets that round to an integer (s = 0 and below 2^-24), whose ideal value is 0, within 2^-24
    of 0 (absolute); and at most TAP_REF_ULP fp32 ulp from the reference's own fp32 formula (CPU torch)."""
    import mpmath

    s = sinc_offsets()
    for n in TAPS:
        c = oracle.sinc_coeffs(n, s)
        assert np.array_equal(c, restated_taps(oracle, n, s)), n
        # exact cos(w) sin(pa) / pa at the fp32 pa and w = fp32(pa / N), in long double (checked by mpmath below)
        k = np.arange(-(n // 2) + 1, n // 2 + 1, dtype=np.float32)
        arg = s[:, None] - k[None, :]
        pa32 = PI_F * arg
        w = (pa32 / np.float32(n)).astype(np.longdouble)
        pa = pa32.astype(np.longdouble)
        safe = np.where(pa == 0, 1, pa)
        exact = np.cos(w) * np.where(pa == 0, 1, np.sin(safe) / safe)
        rel = np.asarray(np.abs(c.astype(np.longdouble) - exact) / np.abs(exact), np.float64)
        assert rel.max() < 3 * 2.0**-24, n
        integer = (arg == np.round(arg)) & (arg != 0)
        assert integer[0].sum() == n - 1 and np.abs(c[integer]).max() < 2.0**-24, n
        i, j = np.unravel_index(np.argmax(rel), rel.shape)
        mpmath.mp.prec = 200
        p, wm = mpmath.mpf(float(pa32[i, j])), mpmath.mpf(float(pa32[i, j] / np.float32(n)))
        e = mpmath.cos(wm) * (mpmath.sin(p) / p if p != 0 else 1)
        assert abs(float(abs((mpmath.mpf(float(c[i, j])) - e) / e)) - rel[i, j]) < 1e-15
        # the reference's fp32 formula
        d = fp32_ulp_distance(c, reference_taps(n, s))
        frac = float((d > 1).any(axis=1).mean())
        print(f"N = {n}: max rel error {rel.max() / 2**-24:.2f} x 2^-24; vs reference fp32: "
              f"max {int(d.max())} ulp, > 1 ulp at {frac:.1%} of the offsets")
        assert d.max() <= TAP_REF_ULP, n


def test_noise_against_reference_generator(oracle):
    """cco_noise_samples over a 3840x2160 frame with 8 grids against noise.py's grand() with the libm calls the
    reference makes: equal in fp32 except within TIE_WINDOW float64 ulp of an fp32 tie, each such sample decided
    at 200 bits.  Also a window deep in the period, and the one sample of the whole period where they differ."""
    got = oracle.noise_samples(0, CR_4K)
    u1, u2 = noise_uniforms(0, CR_4K)
    canon = canonical_noise(oracle, u1, u2)
    assert np.array_equal(canon.astype(np.float32), got)  # the float64 path above is the oracle's
    ref = libm_noise(u1, u2).astype(np.float32)
    near = tie_distance(canon) <= TIE_WINDOW
    differ = got != ref
    assert not (differ & ~near).any(), np.flatnonzero(differ & ~near)[:5]
    print(f"noise [0, {CR_4K}): {int(near.sum())} samples within {TIE_WINDOW} ulp of an fp32 tie, "
          f"{int(differ.sum())} differ from libm")
    for k in np.flatnonzero(near).tolist():
        right = mp_correct_fp32(u1[k], u2[k])
        print(f"  k = {k}: canonical {got[k]!r}, libm {ref[k]!r}, exact rounds to {right!r}")
        assert right in (got[k], ref[k])
    assert differ.sum() == 0  # no libm / canonical difference before sample 12 000 000

    # sample 302 383 943: the only difference over the whole period; the exact value is 6.7e-17 below a tie, the
    # canonical double lands on the tie and rounds (to even) up: the canonical fp32 is 1 ulp off there
    k = 302_383_943
    w = oracle.noise_samples(k - 2, 5)
    a1, a2 = noise_uniforms(k - 2, 5)
    lib = libm_noise(a1, a2).astype(np.float32)
    assert np.array_equal(np.delete(w, 2), np.delete(lib, 2))
    assert w[2] == np.float32(0.9548049) and lib[2] == np.float32(0.95480484) and w[2] == np.nextafter(lib[2], np.float32(1))
    assert mp_correct_fp32(a1[2], a2[2]) == lib[2]
    assert tie_distance(canonical_noise(oracle, a1[2:3], a2[2:3]))[0] == 0.0


def test_noise_samples_is_the_cr_generator(oracle, kodim14):
    """cco_cr_noise draws its grids from cco_noise_samples, finest first, one sample after the other."""
    from coolchic_b200._desc import CcdCoolChicDesc

    d = CcdCoolChicDesc.from_buffer_copy(kodim14["desc"])
    d.latent_res_lo, d.latent_res_hi, d.img_h, d.img_w = 0, 0, 37, 53  # one grid: the cascade is the identity
    assert np.array_equal(oracle.cr_noise(d)[0].reshape(-1), oracle.noise_samples(0, 37 * 53))
    a = oracle.noise_samples(0, 5000)
    assert np.array_equal(oracle.noise_samples(1234, 3766), a[1234:])


# ----------------------------------------------------------------------------------------------
# GPU: device against oracle
def _random_domain(fn, n, seed):
    rng = np.random.default_rng(seed)
    if fn == "log":  # positive normal doubles, every exponent, and (0, 1]
        b = rng.integers(0x0010000000000000, 0x7FF0000000000000, n // 2, dtype=np.uint64).view(np.float64)
        return np.concatenate([b, 1.0 - rng.random(n - n // 2)])
    x = rng.uniform(-64, 64, n // 2)
    mag = np.exp2(rng.uniform(-40, 20, n - n // 2)) * rng.choice([-1.0, 1.0], n - n // 2)
    return np.concatenate([x, mag])


@pytest.mark.gpu
def test_detmath_device_equals_oracle(ctx, oracle, sinc_set, bm_set):
    """ccd_debug_detmath (the kernels' ccd_detmath.h) equals the oracle's detmath.h bit for bit on every argument
    set and on 4 million random doubles of each function's domain."""
    sets = {"sin": [sinc_set[0], adversarial_arguments(), bm_set[1]],
            "cos": [sinc_set[1], adversarial_arguments(), bm_set[1]],
            "log": [bm_set[0], adversarial_arguments()[-1:]]}
    for fn, xs in sets.items():
        for x in xs + [_random_domain(fn, 4 << 20, {"sin": 1, "cos": 2, "log": 3}[fn])]:
            got, want = ctx.detmath(fn, x), oracle.detmath(fn, x)
            bad = np.flatnonzero(bits(got) != bits(want))
            assert bad.size == 0, (fn, x[bad[:5]], got[bad[:5]], want[bad[:5]])


@pytest.mark.gpu
def test_sinc_coeffs_device_equals_oracle(ctx, oracle):
    """ccd_debug_sinc_coeffs (the warp's sinc_coeffs<N>) equals the oracle's taps for every N on 2^20 offsets,
    subnormal ones included (a flush-to-zero build would differ there); any other N is refused."""
    from coolchic_b200 import _native

    rng = np.random.default_rng(13)
    s = np.concatenate([sinc_offsets(1 << 19),
                        rng.integers(1, 1 << 23, 1 << 16, dtype=np.uint32).view(np.float32),   # subnormal
                        np.exp2(rng.uniform(-126, -1, (1 << 20) - (1 << 19) - (1 << 16) - 7)).astype(np.float32)])
    assert s.size == 1 << 20 and (s < np.finfo(np.float32).tiny).sum() > 65536
    for n in TAPS:
        got, want = ctx.sinc_coeffs(n, s), oracle.sinc_coeffs(n, s)
        bad = np.flatnonzero((got.view(np.uint32) != want.view(np.uint32)).any(axis=1))
        assert bad.size == 0, (n, s[bad[:5]])
    for n in (0, 2, 4, 7, 16):
        with pytest.raises(_native.CcdError) as e:
            ctx.sinc_coeffs(n, s[:8])
        assert e.value.code == -1


@pytest.mark.gpu
def test_cr_noise_device_equals_oracle(ctx, oracle):
    """ccd_debug_cr_noise (k_cr_noise: jump-ahead with lcg_pow, Box-Muller) equals the oracle over a 3840x2160 frame
    with 8 grids, and in windows deep in the period where lcg_pow takes large exponents; one launch per call."""
    n0 = ctx.launch_count()
    assert np.array_equal(ctx.cr_noise(0, CR_4K), oracle.noise_samples(0, CR_4K))
    assert ctx.launch_count() - n0 == 1
    for first, n in ((1 << 28, 1 << 16), ((1 << 30) - 4096, 4096), (302_383_943 - 1000, 2001), (M - 1, 3)):
        assert np.array_equal(ctx.cr_noise(first, n), oracle.noise_samples(first, n)), first


@pytest.mark.gpu
def test_common_randomness_1080p_equals_oracle(ctx, oracle, seed_stream):
    """A full-size CR decode: 1080p rgb, 7 grids, 2 764 710 noise samples.  The raw synthesis output and the
    finished 8-bit frame equal the oracle's bit for bit."""
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    data = synth.make_image_stream(ctx, seed_stream, 1080, 1920, "rgb", 8, (0, 6), None, seed=1,
                                   overrides={"flag_common_randomness": 1})
    _, f, c, nn_bytes, payload = synth.parse_single_image(data)
    d = desc_from_header(c)
    assert d.common_randomness == 1 and d.latent_res_hi - d.latent_res_lo + 1 == 7
    assert sum((-(-1080 // 2**i)) * (-(-1920 // 2**i)) for i in range(7)) == 2_764_710
    nn = oracle.decode_nn(d, nn_bytes)
    lat, _ = oracle.decode_latents(d, nn, payload)
    want = oracle.synthesize(d, nn, lat)
    raw = ctx.decode_coolchic(d, nn_bytes, payload).cpu().numpy()[0]
    assert np.array_equal(raw, want)
    out, _ = ctx.decode_many([d], [nn_bytes], [payload], finish=[(8, "rgb")])
    assert np.array_equal(out[0][0].cpu().numpy(), oracle.finish_frame(want, 8, "rgb"))
