"""VIF (ccd_frame_vif, coolchic_b200.bitstream.quality with vif=True, cc_eval.py --vif) against a float64 numpy
restatement of its definition (DESIGN §4.12): samples in 8-bit units, four scales of N_s = 2^(4 - s) + 1 tap Gaussian
windows (sigma N_s / 5) applied "valid", the filter-then-decimate pyramid, the per-pixel clamps and the log10 terms.
Two restatements are kept, a separable one and a naive one with the full 2-D window, and they check each other.
Nothing here is shared with the kernel or with the host combiner."""
import os
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from numpy.lib.stride_tricks import sliding_window_view
from scipy.signal import correlate2d

from test_ssim import _frame, _ints, _noisy, _source


# ---- the restatements ------------------------------------------------------------------------------------------
def taps(s):
    n = 2 ** (4 - s) + 1
    x = np.arange(n, dtype=np.float64) - (n - 1) / 2
    g = np.exp(-(x**2) / (2 * (n / 5) ** 2))
    return g / g.sum()


def filt(a, g):
    n = len(g)
    a = np.tensordot(sliding_window_view(a, n, axis=1), g, axes=([2], [0]))
    return np.tensordot(sliding_window_view(a, n, axis=0), g, axes=([2], [0]))


def window2d(s):
    """The 2-D window of scale s straight from its definition (fspecial('gaussian', N, N / 5))."""
    n = 2 ** (4 - s) + 1
    y, x = np.mgrid[0:n, 0:n] - (n - 1) / 2
    w = np.exp(-(x * x + y * y) / (2 * (n / 5) ** 2))
    return w / w.sum()


def units(k, M):
    return np.asarray(k, dtype=np.float64) * 255 / M


def terms(mu1, mu2, e11, e22, e12):
    """Per-pixel num and den terms from the local moments (1: reference, 2: distorted)."""
    s1 = np.maximum(e11 - mu1 * mu1, 0.0)
    s2 = np.maximum(e22 - mu2 * mu2, 0.0)
    s12 = e12 - mu1 * mu2
    g = s12 / (s1 + 1e-10)
    sv = s2 - g * s12
    z = s1 < 1e-10
    g, sv, s1 = np.where(z, 0.0, g), np.where(z, s2, sv), np.where(z, 0.0, s1)
    z = s2 < 1e-10
    g, sv = np.where(z, 0.0, g), np.where(z, 0.0, sv)
    z = g < 0
    sv, g = np.where(z, s2, sv), np.where(z, 0.0, g)
    sv = np.maximum(sv, 1e-10)
    return np.log10(1 + g * g * s1 / (sv + 2)), np.log10(1 + s1 / 2)


def check_scales(ks, kd, M):
    """Separable restatement: per scale (num, den) of the source ks (reference) and the decode kd (distorted)."""
    ref, dist = units(ks, M), units(kd, M)
    num, den = [], []
    for s in range(4):
        g = taps(s)
        if s > 0:
            ref, dist = filt(ref, g)[::2, ::2], filt(dist, g)[::2, ::2]
        mu1, mu2 = filt(ref, g), filt(dist, g)
        n, d = terms(mu1, mu2, filt(ref * ref, g), filt(dist * dist, g), filt(ref * dist, g))
        num.append(float(n.sum()))
        den.append(float(d.sum()))
    return num, den


def naive_scales(ks, kd, M):
    """Naive restatement: the full 2-D window, correlate2d "valid", decimation and clamps in plain numpy."""
    ref, dist = units(ks, M), units(kd, M)
    num, den = [], []
    for s in range(4):
        w = window2d(s)
        f = lambda a: correlate2d(a, w, mode="valid")  # noqa: E731
        if s > 0:
            ref, dist = f(ref)[0::2, 0::2], f(dist)[0::2, 0::2]
        mu1, mu2 = f(ref), f(dist)
        s1 = f(ref * ref) - mu1 * mu1
        s2 = f(dist * dist) - mu2 * mu2
        s12 = f(ref * dist) - mu1 * mu2
        s1[s1 < 0] = 0
        s2[s2 < 0] = 0
        g = s12 / (s1 + 1e-10)
        sv = s2 - g * s12
        i = s1 < 1e-10
        g[i], sv[i], s1[i] = 0, s2[i], 0
        i = s2 < 1e-10
        g[i], sv[i] = 0, 0
        i = g < 0
        sv[i], g[i] = s2[i], 0
        sv[sv <= 1e-10] = 1e-10
        num.append(float(np.sum(np.log10(1 + g**2 * s1 / (sv + 2)))))
        den.append(float(np.sum(np.log10(1 + s1 / 2))))
    return num, den


def check_vif(ks, kd, M):
    num, den = check_scales(ks, kd, M)
    return None if sum(den) == 0 else sum(num) / sum(den)


def _distort(k, M, rng):
    """A seeded stand-in for a decode: a 3-tap blur plus noise, on the k / M grid."""
    k = np.asarray(k, dtype=np.int64)
    b = (np.roll(k, 1, 0) + 2 * k + np.roll(k, -1, 1)) // 4
    return np.clip(b + rng.integers(-M // 64 - 1, M // 64 + 2, size=k.shape), 0, M)


def _golden_planes():
    """(name, frame, planes, M) of the golden source fixtures, integer samples."""
    z = np.load(os.path.join(GOLDEN, "originals_frames.npz"))
    out = []
    for key in sorted(k for k in z.files if k.endswith("/meta")):
        base = key[:-5]
        planes = [z[f"{base}/{c}"].astype(np.int64) for c in ("yuv" if f"{base}/y" in z.files else "012")]
        bitdepth = 10 if "10b" in base else 8
        out.append((base, planes, 2**bitdepth - 1))
    return out


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_restatements_agree():
    rng = np.random.default_rng(7)
    pairs = []
    for name, planes, M in _golden_planes():
        pairs += [(name, p, _distort(p, M, rng), M) for p in planes]
    for b in (8, 10, 16):
        M = 2**b - 1
        k = rng.integers(0, M + 1, size=(83, 97))
        pairs.append((f"noise{b}", k, _noisy(k, b, rng, amp=M // 20), M))
    assert len(pairs) >= 18
    # Scales 1..3 read filtered values, whose last bits depend on the summation order, and sigma^2 = E[v^2] - mu^2
    # cancels them up to about 1e-10 where the source is flat: the size of the model's clamps.  1e-9 relative bounds
    # what the two orders move on the golden sources.
    worst = 0.0
    for name, ks, kd, M in pairs:
        a, b = check_scales(ks, kd, M), naive_scales(ks, kd, M)
        for x, y in zip(a[0] + a[1], b[0] + b[1]):
            worst = max(worst, abs(x - y) / max(abs(x), abs(y)))
            assert abs(x - y) <= 1e-9 * max(abs(x), abs(y)), (name, a, b)
        assert all(d > 0 for d in a[1]), name
    assert worst > 0  # the two restatements are independent


def test_known_properties():
    rng = np.random.default_rng(8)
    k = rng.integers(20, 236, size=(96, 112))
    k = (k + np.roll(k, 1, 0) + np.roll(k, 1, 1)) // 3  # some local structure
    assert abs(check_vif(k, k, 255) - 1) < 1e-9
    gain = 1.2 * (k - k.mean()) + k.mean()  # a contrast gain, not on the integer grid: v units directly
    num, den = check_scales(k, gain, 255)
    assert sum(num) / sum(den) > 1
    prev = 1.0 + 1e-9
    for sigma in (1, 2, 4, 8, 16, 32):
        noisy = k + np.random.default_rng(9).normal(0, sigma, size=k.shape)
        v = check_vif(k, noisy, 255)
        assert v < prev, (sigma, v, prev)
        prev = v
    assert check_vif(np.full((64, 64), 77), k[:64, :64], 255) is None
    big = k * 257
    for a, b in zip(check_scales(k, k[::-1], 255), check_scales(big, big[::-1], 65535)):
        assert max(abs(x - y) / abs(x) for x, y in zip(a, b)) < 1e-12


def test_size_rule():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import VIF_MIN_SIDE, vif_applies

    def last_side(n):  # the sides of the definition: filter "valid" with N_s taps, keep the even samples
        for s in range(1, 4):
            n = (n - (2 ** (4 - s) + 1) + 1 + 1) // 2
        return n - 3 + 1  # valid outputs at scale 3

    assert last_side(40) == 0 and last_side(41) == 1 and VIF_MIN_SIDE == 41
    rng = np.random.default_rng(2)
    k = rng.integers(0, 256, size=(41, 41))
    assert check_scales(k, _noisy(k, 8, rng), 255)[1][3] > 0
    with pytest.raises(ValueError):  # nothing left to filter at scale 3
        check_scales(k[:40, :], k[:40, :], 255)
    assert not vif_applies((40, 400), "rgb") and not vif_applies((400, 40), "yuv444")
    assert vif_applies((41, 400), "rgb") and vif_applies((400, 41), "yuv444")
    assert not vif_applies((81, 400), "yuv420") and not vif_applies((400, 80), "yuv420")
    assert vif_applies((82, 82), "yuv420")


def test_host_combiner():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import FrameQuality, vif_from_scales

    assert vif_from_scales([1.0, 2.0, 0.5, 0.5], [2.0, 2.0, 1.0, 1.0]) == 4.0 / 6.0
    assert vif_from_scales([0.0] * 4, [0.0] * 4) is None
    kw = dict(display_idx=0, frame_type="I", img_size=(4, 6), bitdepth=8, n_bytes=30, sse=[1, 2, 3], max_abs=[1, 1, 1])
    q = FrameQuality(frame_data_type="yuv420", n_samples=[24, 6, 6], vif_planes=[0.9, 0.6, 0.3], **kw)
    assert abs(q.vif - (24 * 0.9 + 6 * 0.6 + 6 * 0.3) / 36) < 1e-15
    assert (q.vif_y, q.vif_u, q.vif_v) == (0.9, 0.6, 0.3)
    q = FrameQuality(frame_data_type="rgb", n_samples=[24] * 3, vif_planes=[0.9, None, 0.3], **kw)
    assert q.vif is None and q.vif_u is None and q.vif_y == 0.9
    q = FrameQuality(frame_data_type="rgb", n_samples=[24] * 3, **kw)
    assert q.vif is None and q.vif_y is None


def test_export_declared():
    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    assert "ccd_frame_vif" in _native.EXPORTS
    assert "int ccd_frame_vif(CcdContext *ctx, CcdVifJob *jobs" in open(os.path.join(ROOT, "include", "ccdec.h")).read()
    assert hasattr(_native.load_library(), "ccd_frame_vif")


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _check_job(r, dec, src, M, tol=1e-9):
    for c in range(3):
        num, den = check_scales(src[c], dec[c], M)
        for got, want in ((r["num"][c], num), (r["den"][c], den)):
            for x, y in zip(got, want):
                assert abs(x - y) <= tol * max(abs(y), 1e-300), (c, got, want)


def _pair(ctx, dec, src, fmt, bitdepth, layout):
    return _frame(ctx, dec, fmt, bitdepth), _source(ctx, src, bitdepth, layout), layout, dec, src


@pytest.mark.gpu
def test_frame_vif_against_checker(ctx, seed_stream):
    """One call: the golden sources against seeded distortions, the bench's 1080p frame against a perturbed source,
    a 16-bit frame, rgb / yuv444 / yuv420, planar and HWC, a plane at exactly 41 and an odd size."""
    import torch

    from coolchic_b200 import synth
    from coolchic_b200.bitstream.decode import decode_video_bytes

    rng = np.random.default_rng(12)
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
    for h, w, fmt, b, lay in [(41, 53, "rgb", 16, "planar"), (82, 90, "yuv420", 16, "planar"), (97, 41, "yuv444", 12, "hwc")]:
        M = 2**b - 1
        shapes = [(h, w)] + [(h // 2, w // 2) if fmt == "yuv420" else (h, w)] * 2
        src = [rng.integers(0, M + 1, size=s) for s in shapes]
        cases.append((_pair(ctx, [_distort(p, M, rng) for p in src], src, fmt, b, lay), M))
    frames, srcs, lays = [c[0][0] for c in cases], [c[0][1] for c in cases], [c[0][2] for c in cases]
    n0 = ctx.launch_count()
    res = ctx.frame_vif(frames, srcs, lays)
    assert ctx.launch_count() == n0 + 4
    for (case, M), r in zip(cases, res):
        _check_job(r, case[3], case[4], M)
    again = ctx.frame_vif(frames, srcs, lays)
    assert [(a["num"], a["den"]) for a in res] == [(b["num"], b["den"]) for b in again]
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_frame_vif_launches_and_refusals(ctx):
    import torch

    from coolchic_b200._native import CcdError

    rng = np.random.default_rng(5)
    h, w = 96, 128
    src = [rng.integers(0, 256, size=(h, w)) for _ in range(3)]
    pair = _pair(ctx, [_distort(p, 255, rng) for p in src], src, "rgb", 8, "planar")
    for n in (1, 64):
        n0 = ctx.launch_count()
        res = ctx.frame_vif([pair[0]] * n, [pair[1]] * n, ["planar"] * n)
        assert ctx.launch_count() - n0 <= 4
        assert all(r == res[0] for r in res)
    same = ctx.frame_vif([_frame(ctx, src, "rgb", 8)], [pair[1]], ["planar"])[0]
    for c in range(3):
        assert abs(sum(same["num"][c]) / sum(same["den"][c]) - 1) < 1e-9

    ints = [rng.integers(0, 1024, size=s) for s in [(88, 96), (44, 48), (44, 48)]]
    good = _frame(ctx, ints, "yuv420", 10)
    s420 = _source(ctx, ints, 10, "planar")
    off = _frame(ctx, ints, "yuv420", 10)
    off.data["u"][0, 0, 7, 9] += 0.3 / 1023
    off.data["v"][0, 0, 30, 3] = 1.5
    with pytest.raises(CcdError) as e_dist:
        ctx.frame_distortion([good, off], [s420, s420], ["planar"] * 2)
    with pytest.raises(CcdError) as e_vif:
        ctx.frame_vif([good, off], [s420, s420], ["planar"] * 2)
    assert e_vif.value.code == e_dist.value.code == -1
    assert e_vif.value.bad_index == e_dist.value.bad_index == [-1, 88 * 96 + 7 * 48 + 9]
    for shapes, fmt in [([(80, 96), (40, 48), (40, 48)], "yuv420"), ([(40, 64)] * 3, "rgb")]:
        small = [rng.integers(0, 256, size=s) for s in shapes]
        n0 = ctx.launch_count()
        with pytest.raises(CcdError) as e:
            ctx.frame_vif([good, _frame(ctx, small, fmt, 8)], [s420, _source(ctx, small, 8, "planar")], ["planar"] * 2)
        assert e.value.code == -1 and ctx.launch_count() == n0
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def gop420(ctx, seed_stream, tmp_path_factory):
    """A synthetic 96 x 128 4:2:0 I-B-P GOP and a source: its decoded frames plus noise."""
    from coolchic_b200 import synth
    from coolchic_b200.bitstream.decode import decode_video_bytes

    h, w = 96, 128
    data = synth.make_video_stream(ctx, seed_stream, h, w, 3, "yuv420", 8, 8, seed=6)
    dec = decode_video_bytes(data, output_device="cuda")
    rng = np.random.default_rng(96)
    ints = [_ints(dec[str(i)]) for i in range(len(dec))]
    src = [[_noisy(p, 8, rng) for p in fr] for fr in ints]
    d = tmp_path_factory.mktemp("gop420vif")
    cool, yuv = str(d / "gop.cool"), str(d / f"src_{w}x{h}_30p_yuv420_8b.yuv")
    open(cool, "wb").write(data)
    np.concatenate([np.concatenate([p.reshape(-1) for p in fr]) for fr in src]).astype(np.uint8).tofile(yuv)
    return {"data": data, "cool": cool, "yuv": yuv, "dec": ints, "src": src, "h": h, "w": w}


@pytest.mark.gpu
def test_video_quality_gop420(ctx, gop420):
    import torch

    from coolchic_b200.bitstream.quality import video_quality

    g = gop420
    video_quality(g["data"], g["yuv"], vif=True)  # warm
    n0 = ctx.launch_count()
    plain = video_quality(g["data"], g["yuv"])
    n1 = ctx.launch_count()
    again = video_quality(g["data"], g["yuv"], vif=False)
    assert ctx.launch_count() - n1 == n1 - n0
    n2 = ctx.launch_count()
    q = video_quality(g["data"], g["yuv"], vif=True)
    assert ctx.launch_count() - n2 == n1 - n0 + 4
    assert sorted(fq.frame_type for fq in q.values()) == ["B", "I", "P"]
    for k, fq in q.items():
        i = int(k)
        assert plain[k].vif_planes is None and plain[k].vif is None
        assert fq.sse == plain[k].sse == again[k].sse and fq.psnr_db == plain[k].psnr_db
        want = [check_vif(s, d, 255) for d, s in zip(g["dec"][i], g["src"][i])]
        assert max(abs(a - b) for a, b in zip(fq.vif_planes, want)) < 1e-9, (k, fq.vif_planes, want)
        assert abs(fq.vif - (4 * want[0] + want[1] + want[2]) / 6) < 1e-9
        # the same values from one call per frame
        fd = _frame(ctx, g["dec"][i], "yuv420", 8)
        one = ctx.frame_vif([fd], [_source(ctx, g["src"][i], 8, "planar")], ["planar"])[0]
        assert [n / d for n, d in zip(map(sum, one["num"]), map(sum, one["den"]))] == fq.vif_planes
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_cc_eval_vif(ctx, gop420, tmp_path, monkeypatch):
    g = gop420
    out = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", g["cool"], "--original", g["yuv"],
                          "--vif"], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    assert lines[i].split()[-4:] == ["vif", "vif_y", "vif_u", "vif_v"]
    rows = [ln.split() for ln in lines[i + 1:i + 4]]
    assert all(len(r) == 15 and 0 < float(r[11]) < 1 for r in rows)
    assert any(ln.startswith("mean vif ") and "(3 of 3 frames)" in ln for ln in lines)

    # the golden 64 x 96 4:2:0 GOP is below the size rule (chroma 32 x 48): n/a everywhere
    name = "gop5_64x96_yuv420"
    gold = np.load(os.path.join(GOLDEN, name + "_frames.npz"))
    n = len({k.split("_")[0] for k in gold.files})
    frames = [[gold[f"{j}_{c}"] for c in "yuv"] for j in range(n)]
    h, w = frames[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"g_{w}x{h}_yuv420_8b.yuv"
    np.concatenate([np.concatenate([p.reshape(-1) for p in fr]) for fr in frames]).astype(np.uint8).tofile(path)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", os.path.join(GOLDEN, name + ".cool"),
                          "--original", path, "--vif"], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    assert all(ln.split()[-4:] == ["n/a"] * 4 for ln in lines[i + 1:i + 1 + n])
    assert any(ln.startswith("mean vif n/a") for ln in lines)
