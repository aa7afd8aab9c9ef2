"""PSNR-HVS-M and PSNR-HVS (ccd_frame_hvs, coolchic_b200.bitstream.quality with psnr_hvs=True, cc_eval.py
--psnr_hvs) against a float64 numpy restatement of their definition (DESIGN §4.13): samples in 8-bit units, the
non-overlapping 8 x 8 blocks wholly inside each plane, the orthonormal 2-D DCT-II, the masking of the larger of the two
blocks' masks and the CSF-weighted squared coefficient errors.  Two restatements are kept, one vectorised over all
blocks with scipy's DCT and one literal per-block loop with an explicitly built DCT matrix, and they check each other.
Nothing here is shared with the kernel or with the host combiner."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from scipy.fft import dctn

from test_ssim import _frame, _ints, _noisy, _source
from test_vif import _distort, _golden_planes, _pair, gop420  # noqa: F401  (gop420: a fixture)

# Ponomarenko et al. (2007): rows k = 0..7, columns l = 0..7
CSF = np.array([
    [1.608443, 2.339554, 2.573509, 1.608443, 1.072295, 0.643377, 0.504610, 0.421887],
    [2.144591, 2.144591, 1.838221, 1.354478, 0.989811, 0.443708, 0.428918, 0.467911],
    [1.838221, 1.979622, 1.608443, 1.072295, 0.643377, 0.451493, 0.372972, 0.459555],
    [1.838221, 1.513829, 1.169777, 0.887417, 0.504610, 0.295806, 0.321689, 0.415082],
    [1.429727, 1.169777, 0.695543, 0.459555, 0.378457, 0.236102, 0.249855, 0.334222],
    [1.072295, 0.735288, 0.467911, 0.402111, 0.317717, 0.247453, 0.227744, 0.279729],
    [0.525206, 0.402111, 0.329937, 0.295806, 0.249855, 0.212687, 0.214459, 0.254803],
    [0.357432, 0.279729, 0.270896, 0.262603, 0.229778, 0.257351, 0.249855, 0.259950]])
MASK = np.array([
    [0.390625, 0.826446, 1.000000, 0.390625, 0.173611, 0.062500, 0.038447, 0.026874],
    [0.694444, 0.694444, 0.510204, 0.277008, 0.147929, 0.029727, 0.027778, 0.033058],
    [0.510204, 0.591716, 0.390625, 0.173611, 0.062500, 0.030779, 0.021004, 0.031888],
    [0.510204, 0.346021, 0.206612, 0.118906, 0.038447, 0.013212, 0.015625, 0.026015],
    [0.308642, 0.206612, 0.073046, 0.031888, 0.021626, 0.008417, 0.009426, 0.016866],
    [0.173611, 0.081633, 0.033058, 0.024414, 0.015242, 0.009246, 0.007831, 0.011815],
    [0.041649, 0.024414, 0.016437, 0.013212, 0.009426, 0.006830, 0.006944, 0.009803],
    [0.019290, 0.011815, 0.011080, 0.010412, 0.007972, 0.010000, 0.009426, 0.010203]])
# the JPEG luminance quantisation table (ITU-T T.81, Annex K)
Q_JPEG = np.array([
    [16, 11, 10, 16, 24, 40, 51, 61], [12, 12, 14, 19, 26, 58, 60, 55], [14, 13, 16, 24, 40, 57, 69, 56],
    [14, 17, 22, 29, 51, 87, 80, 62], [18, 22, 37, 56, 68, 109, 103, 77], [24, 35, 55, 64, 81, 104, 113, 92],
    [49, 64, 78, 87, 103, 121, 120, 101], [72, 92, 95, 98, 112, 100, 103, 99]])


# ---- the restatements ------------------------------------------------------------------------------------------
def _blocks(k):
    """[nby, nbx, 8, 8] int64 blocks of a plane: the 8 x 8 blocks wholly inside it."""
    k = np.asarray(k, dtype=np.int64)
    nby, nbx = k.shape[0] // 8, k.shape[1] // 8
    return k[:8 * nby, :8 * nbx].reshape(nby, 8, nbx, 8).transpose(0, 2, 1, 3)


def _vari(z, s2):
    """n sum z^2 - (sum z)^2 over n - 1 from exact int64 sums over the last two axes, times s2."""
    n = z.shape[-1] * z.shape[-2]
    s, q = z.sum(axis=(-2, -1)), (z * z).sum(axis=(-2, -1))
    return (n * q - s * s).astype(np.float64) / (n - 1) * s2


def _mask(z, zd, s2):
    ac = MASK.copy()
    ac[0, 0] = 0.0
    m = (zd * zd * ac).sum(axis=(-2, -1))
    full = _vari(z, s2)
    quads = _vari(z[..., :4, :4], s2) + _vari(z[..., :4, 4:], s2) + _vari(z[..., 4:, 4:], s2) + _vari(z[..., 4:, :4], s2)
    pop = np.where(full != 0, quads / np.where(full != 0, full, 1.0), 0.0)
    return np.sqrt(m * pop) / 32


def check_blocks(ks, kd, M):
    """Vectorised restatement: per block (S_hvs_m, S_hvs) of the source ks against the decode kd, [nby, nbx] each."""
    A, B = _blocks(ks), _blocks(kd)
    s2 = (255 / M) ** 2
    ad = dctn(A * 255 / M, axes=(-2, -1), norm="ortho")
    bd = dctn(B * 255 / M, axes=(-2, -1), norm="ortho")
    T = np.maximum(_mask(A, ad, s2), _mask(B, bd, s2))[..., None, None]
    u = np.abs(ad - bd)
    um = np.maximum(u - T / MASK, 0.0)
    um[..., 0, 0] = u[..., 0, 0]
    return ((um * CSF) ** 2).sum(axis=(-2, -1)), ((u * CSF) ** 2).sum(axis=(-2, -1))


def check_sums(ks, kd, M):
    """(S_hvs_m, S_hvs, N_c) of one plane."""
    m, s = check_blocks(ks, kd, M)
    return float(m.sum()), float(s.sum()), 64 * m.size


def _dct_matrix():
    c = np.zeros((8, 8))
    for k in range(8):
        for n in range(8):
            c[k, n] = math.sqrt((1 if k == 0 else 2) / 8) * math.cos(math.pi * (2 * n + 1) * k / 16)
    return c


def literal_sums(ks, kd, M):
    """Literal restatement of the original per-block loops: the DCT as C Z C^T, vari as np.var(ddof=1) * n."""
    C = _dct_matrix()
    ks, kd = np.asarray(ks, dtype=np.float64) * 255 / M, np.asarray(kd, dtype=np.float64) * 255 / M

    def vari(z):
        return np.var(z, ddof=1) * z.size

    def maskeff(z, zdct):
        m = 0.0
        for k in range(8):
            for l in range(8):
                if k != 0 or l != 0:
                    m += zdct[k, l] ** 2 * MASK[k, l]
        pop = vari(z)
        if pop != 0:
            pop = (vari(z[:4, :4]) + vari(z[:4, 4:]) + vari(z[4:, 4:]) + vari(z[4:, :4])) / pop
        return math.sqrt(m * pop) / 32

    s_hvs_m = s_hvs = 0.0
    n = 0
    for y in range(0, ks.shape[0] - 7, 8):
        for x in range(0, ks.shape[1] - 7, 8):
            a, b = ks[y:y + 8, x:x + 8], kd[y:y + 8, x:x + 8]
            ad, bd = C @ a @ C.T, C @ b @ C.T
            t = max(maskeff(a, ad), maskeff(b, bd))
            for k in range(8):
                for l in range(8):
                    u = abs(ad[k, l] - bd[k, l])
                    s_hvs += (u * CSF[k, l]) ** 2
                    if k != 0 or l != 0:
                        u = max(u - t / MASK[k, l], 0.0)
                    s_hvs_m += (u * CSF[k, l]) ** 2
                    n += 1
    return s_hvs_m, s_hvs, n


def dist_to_db(dist):
    return -10 * math.log10(max(dist, 10 ** (-100 / 10)))


def check_db(sums):
    """Per frame: dist_to_db(sum S / sum N / 255^2) of (S, N) pairs."""
    return dist_to_db(sum(s for s, _ in sums) / sum(n for _, n in sums) / 255**2)


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_tables_follow_jpeg_table():
    """Mask = round((10 / Q)^2, 6) everywhere.  CSF = round(25.735088 / Q, 6) everywhere but at (0, 1), where the
    published 2.339554 is one unit above round(25.735088 / 11, 6) = 2.339553: the published CSF rounds 25.73509 / Q
    (any constant in [25.7350885, 25.7350915] gives all 64 entries).  The published values are used as they are."""
    assert np.all(np.abs(MASK - np.round((10 / Q_JPEG) ** 2, 6)) < 1e-12)
    off = np.abs(CSF - np.round(25.735088 / Q_JPEG, 6)) > 1e-12
    assert np.argwhere(off).tolist() == [[0, 1]] and abs(CSF[0, 1] - 2.339553 - 1e-6) < 1e-12
    assert np.all(np.abs(CSF - np.round(25.73509 / Q_JPEG, 6)) < 1e-12)


def test_restatements_agree():
    rng = np.random.default_rng(17)
    pairs = []
    for name, planes, M in _golden_planes():
        pairs += [(name, p, _distort(p, M, rng), M) for p in planes]
    for b, shape in ((8, (43, 61)), (10, (37, 90)), (16, (64, 29))):  # odd sizes: rows and columns left over
        M = 2**b - 1
        k = rng.integers(0, M + 1, size=shape)
        k = (k + np.roll(k, 1, 0) + np.roll(k, 1, 1)) // 3
        pairs.append((f"noise{b}", k, _distort(k, M, rng), M))
    assert len(pairs) >= 18
    worst = 0.0
    for name, ks, kd, M in pairs:
        a, b = check_sums(ks, kd, M), literal_sums(ks, kd, M)
        assert a[2] == b[2] == 64 * (ks.shape[0] // 8) * (ks.shape[1] // 8)
        for x, y in zip(a[:2], b[:2]):
            worst = max(worst, abs(x - y) / max(abs(x), abs(y)))
            assert abs(x - y) <= 1e-10 * max(abs(x), abs(y)), (name, a, b)
        assert 0 < a[0] < a[1], name  # the masking removes some error, never all of it here
    assert worst > 0  # the two restatements are independent


def test_known_properties():
    rng = np.random.default_rng(18)
    k = rng.integers(20, 236, size=(64, 80))
    k = (k + np.roll(k, 1, 0) + np.roll(k, 1, 1)) // 3
    assert check_sums(k, k, 255)[:2] == (0.0, 0.0)
    assert check_db([check_sums(k, k, 255)[::2]]) == 100.0
    d = _distort(k, 255, rng)
    m, s, n = check_sums(k, d, 255)
    assert dist_to_db(m / n / 255**2) >= dist_to_db(s / n / 255**2)
    assert check_sums(d, k, 255) == (m, s, n)  # the source and the decode play symmetric roles
    for b, off in ((8, 3), (10, 7), (16, 1000)):
        M = 2**b - 1
        base = rng.integers(0, M - off, size=(40, 48))
        m, s, n = check_sums(base, base + off, M)
        want = 10 * math.log10(255**2 / (1.608443 * off * 255 / M) ** 2)
        assert abs(dist_to_db(s / n / 255**2) - want) < 1e-9, (b, off)
        assert abs(dist_to_db(m / n / 255**2) - want) < 1e-9, (b, off)  # only the DC term moves: never masked
    big, bigd = k * 257, d * 257  # the same 8-bit samples at 16 bits
    for x, y in zip(check_sums(k, d, 255), check_sums(big, bigd, 65535)):
        assert abs(x - y) <= 1e-12 * abs(x)
    k2, d2 = k[:61, :77].copy(), d[:61, :77].copy()  # 7 x 9 blocks; then change what lies outside them
    want = check_sums(k2, d2, 255)
    k2[56:, :], d2[:, 72:] = 0, 255
    assert check_sums(k2, d2, 255) == want


def test_size_rule():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import HVS_MIN_SIDE, hvs_applies

    assert HVS_MIN_SIDE == 8
    k = np.random.default_rng(3).integers(0, 256, size=(8, 9))
    assert check_sums(k, k[::-1], 255)[2] == 64 and check_sums(k[:7], k[:7], 255)[2] == 0
    assert not hvs_applies((7, 400), "rgb") and not hvs_applies((400, 7), "yuv444")
    assert hvs_applies((8, 400), "rgb") and hvs_applies((400, 8), "yuv444")
    assert not hvs_applies((15, 400), "yuv420") and not hvs_applies((400, 14), "yuv420")
    assert hvs_applies((16, 16), "yuv420")


def test_host_combiner():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import FrameQuality, hvs_from_sums

    assert hvs_from_sums([65025.0 * 64], [64]) == 0.0
    assert abs(hvs_from_sums([1.0, 3.0], [64, 192]) - 10 * math.log10(256 * 65025 / 4)) < 1e-12
    assert hvs_from_sums([0.0], [64]) == 100.0
    kw = dict(display_idx=0, frame_type="I", img_size=(16, 24), bitdepth=8, n_bytes=30, sse=[1, 2, 3], max_abs=[1, 1, 1])
    planes = [(2.0, 5.0, 384), (1.0, 1.5, 64), (0.5, 0.5, 64)]
    q = FrameQuality(frame_data_type="yuv420", n_samples=[384, 96, 96], hvs_planes=planes, **kw)
    assert q.psnr_hvs_m_db == -10 * math.log10(3.5 / 512 / 65025)
    assert q.psnr_hvs_db == -10 * math.log10(7.0 / 512 / 65025)
    assert (q.psnr_hvs_m_y_db, q.psnr_hvs_m_u_db, q.psnr_hvs_m_v_db) == tuple(
        -10 * math.log10(s / n / 65025) for s, _, n in planes)
    q = FrameQuality(frame_data_type="rgb", n_samples=[384] * 3, **kw)
    assert q.psnr_hvs_m_db is None and q.psnr_hvs_db is None and q.psnr_hvs_m_y_db is None


def test_export_declared():
    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    assert "ccd_frame_hvs" in _native.EXPORTS
    assert "int ccd_frame_hvs(CcdContext *ctx, CcdHvsJob *jobs" in open(os.path.join(ROOT, "include", "ccdec.h")).read()
    assert hasattr(_native.load_library(), "ccd_frame_hvs")


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _check_job(r, dec, src, M, tol=1e-9):
    for c in range(3):
        m, s, n = check_sums(src[c], dec[c], M)
        assert r["n_coeffs"][c] == n
        for got, want in ((r["s_hvs_m"][c], m), (r["s_hvs"][c], s)):
            assert abs(got - want) <= tol * max(abs(want), 1e-300), (c, got, want)
        if "maps" in r:
            got = r["maps"][c].cpu().numpy()
            want = check_blocks(src[c], dec[c], M)[0] / 64 / 255**2
            assert got.shape == want.shape and np.all(np.abs(got - want) <= 1e-6 * np.abs(want) + 1e-12), c


@pytest.mark.gpu
def test_frame_hvs_against_checker(ctx, seed_stream):
    """One call with maps: the golden sources against seeded distortions, the bench's 1080p frame against a perturbed
    source, 12- and 16-bit frames, rgb / yuv444 / yuv420, planar and HWC, odd sizes and a plane of exactly 8."""
    import torch

    from coolchic_b200 import synth
    from coolchic_b200.bitstream.decode import decode_video_bytes

    rng = np.random.default_rng(22)
    cases = []
    for name, planes, M in _golden_planes():
        fmt = "yuv420" if planes[1].shape != planes[0].shape else ("rgb" if name.endswith(".png") else "yuv444")
        b = 10 if M == 1023 else 8
        dist = [_distort(p, M, rng) for p in planes]
        cases.append((_pair(ctx, dist, planes, fmt, b, "planar"), M))
        if fmt != "yuv420":
            cases.append((_pair(ctx, dist, planes, fmt, b, "hwc"), M))
    data = synth.make_image_stream(ctx, seed_stream, 1080, 1920, "rgb", 8, (0, 6), None, seed=0)
    dec = _ints(decode_video_bytes(data, output_device="cuda")["0"])
    cases.append((_pair(ctx, dec, [_noisy(p, 8, rng, amp=6) for p in dec], "rgb", 8, "hwc"), 255))
    for h, w, fmt, b, lay in [(8, 53, "rgb", 16, "planar"), (46, 70, "yuv420", 16, "planar"), (97, 300, "yuv444", 12, "hwc"),
                              (35, 21, "rgb", 12, "planar"), (16, 18, "yuv420", 12, "planar")]:
        M = 2**b - 1
        shapes = [(h, w)] + [(h // 2, w // 2) if fmt == "yuv420" else (h, w)] * 2
        src = [rng.integers(0, M + 1, size=s) for s in shapes]
        cases.append((_pair(ctx, [_distort(p, M, rng) for p in src], src, fmt, b, lay), M))
    frames, srcs, lays = [c[0][0] for c in cases], [c[0][1] for c in cases], [c[0][2] for c in cases]
    n0 = ctx.launch_count()
    res = ctx.frame_hvs(frames, srcs, lays, want_maps=True)
    assert ctx.launch_count() == n0 + 1
    for (case, M), r in zip(cases, res):
        _check_job(r, case[3], case[4], M)
    again = ctx.frame_hvs(frames, srcs, lays)
    assert [(a["s_hvs_m"], a["s_hvs"]) for a in res] == [(b["s_hvs_m"], b["s_hvs"]) for b in again]
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_frame_hvs_launches_and_refusals(ctx):
    import torch

    from coolchic_b200._native import CcdError

    rng = np.random.default_rng(25)
    h, w = 96, 128
    src = [rng.integers(0, 256, size=(h, w)) for _ in range(3)]
    pair = _pair(ctx, [_distort(p, 255, rng) for p in src], src, "rgb", 8, "planar")
    for n in (1, 64):
        n0 = ctx.launch_count()
        res = ctx.frame_hvs([pair[0]] * n, [pair[1]] * n, ["planar"] * n)
        assert ctx.launch_count() - n0 <= 1
        assert all(r == res[0] for r in res)
    same = ctx.frame_hvs([_frame(ctx, src, "rgb", 8)], [pair[1]], ["planar"])[0]
    assert same["s_hvs_m"] == same["s_hvs"] == [0.0] * 3

    # an off-grid sample in the rows below the last full block still refuses the frame, as in frame_distortion
    ints = [rng.integers(0, 1024, size=s) for s in [(84, 96), (42, 48), (42, 48)]]
    good = _frame(ctx, ints, "yuv420", 10)
    s420 = _source(ctx, ints, 10, "planar")
    off = _frame(ctx, ints, "yuv420", 10)
    off.data["u"][0, 0, 41, 9] += 0.3 / 1023
    off.data["v"][0, 0, 30, 3] = 1.5
    with pytest.raises(CcdError) as e_dist:
        ctx.frame_distortion([good, off], [s420, s420], ["planar"] * 2)
    with pytest.raises(CcdError) as e_hvs:
        ctx.frame_hvs([good, off], [s420, s420], ["planar"] * 2)
    assert e_hvs.value.code == e_dist.value.code == -1
    assert e_hvs.value.bad_index == e_dist.value.bad_index == [-1, 84 * 96 + 41 * 48 + 9]
    for shapes, fmt in [([(14, 96), (7, 48), (7, 48)], "yuv420"), ([(40, 7)] * 3, "rgb")]:
        small = [rng.integers(0, 256, size=s) for s in shapes]
        n0 = ctx.launch_count()
        with pytest.raises(CcdError) as e:
            ctx.frame_hvs([good, _frame(ctx, small, fmt, 8)], [s420, _source(ctx, small, 8, "planar")], ["planar"] * 2)
        assert e.value.code == -1 and ctx.launch_count() == n0
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_video_quality_gop420(ctx, gop420):
    import torch

    from coolchic_b200.bitstream.quality import video_quality

    g = gop420
    video_quality(g["data"], g["yuv"], psnr_hvs=True)  # warm
    n0 = ctx.launch_count()
    plain = video_quality(g["data"], g["yuv"])
    n1 = ctx.launch_count()
    again = video_quality(g["data"], g["yuv"], psnr_hvs=False)
    assert ctx.launch_count() - n1 == n1 - n0
    n2 = ctx.launch_count()
    q = video_quality(g["data"], g["yuv"], psnr_hvs=True, want_maps=True)
    assert ctx.launch_count() - n2 == n1 - n0 + 1
    assert sorted(fq.frame_type for fq in q.values()) == ["B", "I", "P"]
    for k, fq in q.items():
        i = int(k)
        assert plain[k].hvs_planes is None and plain[k].psnr_hvs_m_db is None and plain[k].hvs_maps is None
        assert fq.sse == plain[k].sse == again[k].sse and fq.psnr_db == plain[k].psnr_db
        want = [check_sums(s, d, 255) for d, s in zip(g["dec"][i], g["src"][i])]
        for got, w in zip(fq.hvs_planes, want):
            assert got[2] == w[2] and abs(got[0] - w[0]) <= 1e-9 * w[0] and abs(got[1] - w[1]) <= 1e-9 * w[1]
        assert abs(fq.psnr_hvs_m_db - check_db([(w[0], w[2]) for w in want])) < 1e-9
        assert abs(fq.psnr_hvs_db - check_db([(w[1], w[2]) for w in want])) < 1e-9
        assert [m.shape for m in fq.hvs_maps] == [(12, 16), (6, 8), (6, 8)]
        # the same values from one call per frame
        fd = _frame(ctx, g["dec"][i], "yuv420", 8)
        one = ctx.frame_hvs([fd], [_source(ctx, g["src"][i], 8, "planar")], ["planar"])[0]
        assert list(zip(one["s_hvs_m"], one["s_hvs"], one["n_coeffs"])) == fq.hvs_planes
    torch.cuda.synchronize()


def _cc_eval(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), *args], capture_output=True, text=True,
                          check=True).stdout.splitlines()


@pytest.mark.gpu
def test_cc_eval_psnr_hvs(ctx, gop420, tmp_path):
    from PIL import Image

    g = gop420
    lines = _cc_eval("-i", g["cool"], "--original", g["yuv"], "--psnr_hvs")
    base = _cc_eval("-i", g["cool"], "--original", g["yuv"])
    cols = ["psnr_hvs_db", "psnr_hvs_m_db", "psnr_hvs_m_y_db", "psnr_hvs_m_u_db", "psnr_hvs_m_v_db"]
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    assert lines[i].split()[-5:] == cols and lines[i].split()[:-5] == base[i].split()
    rows = [ln.split() for ln in lines[i + 1:i + 4]]
    assert all(len(r) == 16 and float(r[12]) >= float(r[11]) > 0 for r in rows)
    assert [r[:11] for r in rows] == [ln.split() for ln in base[i + 1:i + 4]]  # the other columns do not move
    assert any(ln.startswith("mean psnr_hvs_db ") and "(3 of 3 frames)" in ln for ln in lines)
    assert not any("hvs" in ln for ln in base)

    # a 129 x 7 rgb image is below the size rule: n/a everywhere
    name = "arch_129x7"
    planes = np.load(os.path.join(GOLDEN, name + ".npz"))["0"]
    path = str(tmp_path / "src.png")
    Image.fromarray(np.stack(list(planes), -1).astype(np.uint8), mode="RGB").save(path)
    lines = _cc_eval("-i", os.path.join(GOLDEN, name + ".cool"), "--original", path, "--psnr_hvs")
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    assert lines[i + 1].split()[-5:] == ["n/a"] * 5
    assert any(ln.startswith("mean psnr_hvs_db n/a  psnr_hvs_m_db n/a  (0 of 1 frames)") for ln in lines)
