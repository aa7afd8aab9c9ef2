"""MS-SSIM (ccd_frame_ssim, coolchic_b200.bitstream.quality with ms_ssim=True, cc_eval.py --ms_ssim) against a float64
numpy restatement of its definition (DESIGN §4.6): the integer pyramid, the 11-tap Gaussian window applied "valid" in
two tensordot passes, the per-pixel cs and l * cs, their per-scale means and the weighted product.  Nothing here is
shared with the kernel or with the host combiner."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from numpy.lib.stride_tricks import sliding_window_view

WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)


# ---- the restatement -------------------------------------------------------------------------------------------
def taps():
    i = np.arange(11, dtype=np.float64)
    g = np.exp(-((i - 5) ** 2) / (2 * 1.5**2))
    return g / g.sum()


def pyramid(k):
    """Five levels of exact integer sums: level j + 1 sums 2 x 2 samples of level j, floor sizes."""
    levels = [np.asarray(k, dtype=np.int64)]
    for _ in range(4):
        a = levels[-1]
        a = a[: a.shape[0] // 2 * 2, : a.shape[1] // 2 * 2]
        levels.append(a[0::2, 0::2] + a[1::2, 0::2] + a[0::2, 1::2] + a[1::2, 1::2])
    return levels


def filt(a, g):
    a = np.tensordot(sliding_window_view(a, 11, axis=1), g, axes=([2], [0]))
    return np.tensordot(sliding_window_view(a, 11, axis=0), g, axes=([2], [0]))


def check_scales(kx, ky, M):
    """Per scale, the mean of cs and of l * cs of two integer planes; and the scale-0 SSIM map."""
    g, C1, C2 = taps(), (0.01 * M) ** 2, (0.03 * M) ** 2
    cs_j, ssim_j, map0 = [], [], None
    for j, (sx, sy) in enumerate(zip(pyramid(kx), pyramid(ky))):
        x, y = sx / 4.0**j, sy / 4.0**j
        mx, my = filt(x, g), filt(y, g)
        vx, vy, cxy = filt(x * x, g) - mx * mx, filt(y * y, g) - my * my, filt(x * y, g) - mx * my
        cs = (2 * cxy + C2) / (vx + vy + C2)
        lum = (2 * mx * my + C1) / (mx * mx + my * my + C1)
        cs_j.append(float(cs.mean()))
        ssim_j.append(float((lum * cs).mean()))
        if j == 0:
            map0 = lum * cs
    return cs_j, ssim_j, map0


def check_ms_ssim(cs, ssim):
    v = 1.0
    for j in range(4):
        v *= max(cs[j], 0.0) ** WEIGHTS[j]
    return v * max(ssim[4], 0.0) ** WEIGHTS[4]


def dist_to_db(dist):
    return -10 * math.log10(max(dist, 10 ** (-100 / 10)))


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_restatement_identity_and_offset():
    rng = np.random.default_rng(0)
    k = rng.integers(0, 256, size=(190, 213))
    cs, ssim, m = check_scales(k, k, 255)
    assert cs == [1.0] * 5 and ssim == [1.0] * 5 and np.all(m == 1.0)
    assert check_ms_ssim(cs, ssim) == 1.0
    k = rng.integers(0, 200, size=(181, 177))
    cs, ssim, _ = check_scales(k, k + 17, 255)  # the same structure, another mean: only the luminance term moves
    assert all(abs(c - 1.0) < 1e-12 for c in cs)
    assert all(s < 1.0 for s in ssim)


def test_restatement_pyramid_is_avg_pool():
    import torch
    import torch.nn.functional as F

    k = np.random.default_rng(1).integers(0, 1024, size=(389, 517))
    x = torch.from_numpy(k.astype(np.float64))[None, None]
    for j, level in enumerate(pyramid(k)):
        assert level.shape == tuple(x.shape[-2:])
        assert np.array_equal(level / 4.0**j, x[0, 0].numpy())
        x = F.avg_pool2d(x, 2)


def test_host_combiner():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import FrameQuality, ms_ssim_from_scales

    cs, ssim = [0.9, 0.8, 0.7, 0.6, 0.55], [0.85, 0.75, 0.65, 0.5, 0.4]
    want = 0.9**0.0448 * 0.8**0.2856 * 0.7**0.3001 * 0.6**0.2363 * 0.4**0.1333
    assert abs(ms_ssim_from_scales(cs, ssim) - want) < 1e-15
    assert ms_ssim_from_scales([0.9, -0.1, 0.7, 0.6, 0.5], ssim) == 0.0
    assert ms_ssim_from_scales(cs, [0.9, 0.8, 0.7, 0.6, -0.2]) == 0.0
    assert ms_ssim_from_scales([1.0] * 5, [1.0] * 5) == 1.0
    kw = dict(display_idx=0, frame_type="I", img_size=(4, 6), bitdepth=8, n_bytes=30, sse=[1, 2, 3], max_abs=[1, 1, 1])
    q = FrameQuality(frame_data_type="yuv420", n_samples=[24, 6, 6], ms_ssim_planes=[0.9, 0.6, 0.3], **kw)
    assert abs(q.ms_ssim - (24 * 0.9 + 6 * 0.6 + 6 * 0.3) / 36) < 1e-15  # (4 D_Y + D_U + D_V) / 6
    assert abs(q.ms_ssim_db - -10 * math.log10(1 - q.ms_ssim)) < 1e-12
    assert (q.ms_ssim_y, q.ms_ssim_u, q.ms_ssim_v) == (0.9, 0.6, 0.3)
    q = FrameQuality(frame_data_type="rgb", n_samples=[24] * 3, ms_ssim_planes=[1.0] * 3, **kw)
    assert q.ms_ssim == 1.0 and q.ms_ssim_db == 100.0
    q = FrameQuality(frame_data_type="rgb", n_samples=[24] * 3, **kw)
    assert q.ms_ssim is None and q.ms_ssim_db is None and q.ms_ssim_y is None and q.ssim_maps is None


def test_size_rule():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import ms_ssim_applies

    assert not ms_ssim_applies((175, 400), "rgb") and not ms_ssim_applies((400, 175), "yuv444")
    assert ms_ssim_applies((176, 400), "rgb") and ms_ssim_applies((400, 176), "yuv444")
    assert not ms_ssim_applies((350, 400), "yuv420") and not ms_ssim_applies((400, 350), "yuv420")
    assert ms_ssim_applies((352, 352), "yuv420")
    assert 176 // 16 == 11 and 175 // 16 == 10  # five scales: 11 samples at the fifth


def test_export_declared():
    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    assert "ccd_frame_ssim" in _native.EXPORTS
    assert "int ccd_frame_ssim(CcdContext *ctx, CcdSsimJob *jobs" in open(os.path.join(ROOT, "include", "ccdec.h")).read()
    assert hasattr(_native.load_library(), "ccd_frame_ssim")


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _ints(fd):
    """Integer planes (int64) of a FrameData on any device."""
    M = 2**fd.bitdepth - 1
    ts = [fd.data[c][0, 0] for c in "yuv"] if fd.frame_data_type == "yuv420" else [fd.data[0, c] for c in range(3)]
    return [np.rint(t.cpu().numpy().astype(np.float32) * np.float32(M)).astype(np.int64) for t in ts]


def _check_job(r, dec, src, bitdepth, maps=None):
    for c in range(3):
        cs, ssim, m0 = check_scales(dec[c], src[c], 2**bitdepth - 1)
        assert max(abs(a - b) for a, b in zip(r["cs"][c], cs)) < 1e-10, (c, r["cs"][c], cs)
        assert max(abs(a - b) for a, b in zip(r["ssim"][c], ssim)) < 1e-10, (c, r["ssim"][c], ssim)
        if maps is not None:
            got = maps[c].cpu().numpy()
            assert got.shape == m0.shape and np.abs(got - m0).max() < 1e-6


def _frame(ctx, k, fmt, bitdepth):
    """FrameData of integer planes k (int64 numpy, FrameData shapes) on the device."""
    import torch

    from coolchic_b200.io.framedata import FrameData

    M = 2**bitdepth - 1
    t = [torch.from_numpy(p.astype(np.float32) / np.float32(M)).to(ctx.torch_device) for p in k]
    if fmt == "yuv420":
        return FrameData(bitdepth, fmt, {c: x[None, None] for c, x in zip("yuv", t)})
    return FrameData(bitdepth, fmt, torch.stack(t)[None])


def _source(ctx, planes, bitdepth, layout):
    import torch

    flat = np.stack(planes, -1).reshape(-1) if layout == "hwc" else np.concatenate([p.reshape(-1) for p in planes])
    return torch.from_numpy(flat.astype(np.uint8 if bitdepth <= 8 else np.int16)).to(ctx.torch_device)


def _case(ctx, rng, h, w, fmt, bitdepth, layout, amp=3):
    M = 2**bitdepth - 1
    shapes = [(h, w)] + [(h // 2, w // 2) if fmt == "yuv420" else (h, w)] * 2
    # a smooth ramp plus texture, and the source a few steps away from it
    dec = []
    for s in shapes:
        yy, xx = np.mgrid[0:s[0], 0:s[1]]
        base = (M * (0.3 + 0.2 * np.sin(yy / 17.0) + 0.2 * np.cos(xx / 23.0))).astype(np.int64)
        dec.append(np.clip(base + rng.integers(-M // 8, M // 8 + 1, size=s), 0, M))
    src = [np.clip(d + rng.integers(-amp, amp + 1, size=d.shape), 0, M) for d in dec]
    return _frame(ctx, dec, fmt, bitdepth), _source(ctx, src, bitdepth, layout), layout, dec, src


@pytest.mark.gpu
def test_frame_ssim_mixed_call(ctx):
    """One call: rgb / yuv444 / yuv420, 8 and 10 bits, planar and HWC, odd sizes and 2 x SM + 5 Kodak-size frames."""
    import torch

    rng = np.random.default_rng(11)
    cases = [(389, 517, "rgb", 8, "hwc"), (517, 389, "yuv444", 10, "planar"), (389, 517, "rgb", 10, "planar"),
             (354, 706, "yuv420", 8, "planar"), (386, 362, "yuv420", 10, "planar"), (176, 176, "yuv444", 8, "hwc")]
    n_kodak = 2 * torch.cuda.get_device_properties(ctx.device).multi_processor_count + 5
    for i in range(n_kodak):
        cases.append((512, 768, "rgb" if i % 2 == 0 else "yuv444", 10 if i % 3 == 1 else 8, "hwc" if i % 2 == 0 else "planar"))
    jobs = [_case(ctx, rng, *c) for c in cases]
    frames, srcs, lays = [j[0] for j in jobs], [j[1] for j in jobs], [j[2] for j in jobs]
    n0 = ctx.launch_count()
    res = ctx.frame_ssim(frames, srcs, lays, want_maps=True)
    assert ctx.launch_count() == n0 + 5
    checked = list(range(6)) + [6, 7, 6 + n_kodak // 2, len(cases) - 1]
    for i in checked:
        _check_job(res[i], jobs[i][3], jobs[i][4], cases[i][3], res[i]["maps"])
    again = ctx.frame_ssim(frames, srcs, lays, want_maps=True)
    for a, b in zip(res, again):
        assert a["cs"] == b["cs"] and a["ssim"] == b["ssim"]
        assert all(torch.equal(x, y) for x, y in zip(a["maps"], b["maps"]))


@pytest.mark.gpu
def test_frame_ssim_identical_and_off_grid(ctx):
    import torch

    from coolchic_b200._native import CcdError

    rng = np.random.default_rng(3)
    frames, srcs, lays = [], [], []
    for h, w, fmt, b, lay in [(400, 353, "rgb", 8, "hwc"), (352, 384, "yuv420", 10, "planar")]:
        fd, _, _, dec, _ = _case(ctx, rng, h, w, fmt, b, lay)
        frames.append(fd)
        srcs.append(_source(ctx, dec, b, lay))
        lays.append(lay)
    for r in ctx.frame_ssim(frames, srcs, lays):
        assert r["cs"] == [[1.0] * 5] * 3 and r["ssim"] == [[1.0] * 5] * 3

    off = _frame(ctx, _ints(frames[1]), "yuv420", 10)
    off.data["u"][0, 0, 7, 9] += 0.3 / 1023
    off.data["v"][0, 0, 100, 3] = 1.5
    with pytest.raises(CcdError) as e_dist:
        ctx.frame_distortion([frames[1], off], [srcs[1], srcs[1]], ["planar"] * 2)
    with pytest.raises(CcdError) as e_ssim:
        ctx.frame_ssim([frames[1], off], [srcs[1], srcs[1]], ["planar"] * 2)
    assert e_ssim.value.code == e_dist.value.code == -1
    assert e_ssim.value.bad_index == e_dist.value.bad_index == [-1, 352 * 384 + 7 * 192 + 9]
    small = _case(ctx, rng, 350, 384, "yuv420", 8, "planar")
    n0 = ctx.launch_count()
    with pytest.raises(CcdError) as e:
        ctx.frame_ssim([small[0]], [small[1]], ["planar"])
    assert e.value.code == -1 and ctx.launch_count() == n0
    torch.cuda.synchronize()


def _noisy(k, bitdepth, rng, amp=4):
    return np.clip(k + rng.integers(-amp, amp + 1, size=k.shape), 0, 2**bitdepth - 1)


@pytest.mark.gpu
def test_video_quality_kodim14(ctx, kodim14, tmp_path):
    from PIL import Image

    from coolchic_b200.bitstream.decode import decode_video_bytes
    from coolchic_b200.bitstream.quality import video_quality

    dec = _ints(decode_video_bytes(kodim14["data"], output_device="cuda")["0"])
    src = [_noisy(x, 8, np.random.default_rng(14)) for x in dec]
    path = str(tmp_path / "kodim14.png")
    Image.fromarray(np.stack(src, -1).astype(np.uint8), mode="RGB").save(path)
    video_quality(kodim14["data"], path, ms_ssim=True)  # warm
    n0 = ctx.launch_count()
    plain = video_quality(kodim14["data"], path)["0"]
    n1 = ctx.launch_count()
    fq = video_quality(kodim14["data"], path, ms_ssim=True, want_maps=True)["0"]
    assert ctx.launch_count() - n1 == n1 - n0 + 5
    assert plain.ms_ssim is None and plain.ssim_maps is None and plain.sse == fq.sse
    want = []
    for c in range(3):
        cs, ssim, m0 = check_scales(dec[c], src[c], 255)
        want.append(check_ms_ssim(cs, ssim))
        assert np.abs(fq.ssim_maps[c].cpu().numpy() - m0).max() < 1e-6
    assert max(abs(a - b) for a, b in zip(fq.ms_ssim_planes, want)) < 1e-9
    assert abs(fq.ms_ssim - sum(want) / 3) < 1e-9 and 0.5 < fq.ms_ssim < 1
    assert abs(fq.ms_ssim_db - dist_to_db(1 - sum(want) / 3)) < 1e-6


@pytest.fixture(scope="module")
def gop420(ctx, seed_stream, tmp_path_factory):
    """A synthetic 384 x 352 4:2:0 I-B-P GOP, its decoded frames and a source: the decoded frames plus noise."""
    from coolchic_b200 import synth
    from coolchic_b200.bitstream.decode import decode_video_bytes

    h, w = 352, 384
    data = synth.make_video_stream(ctx, seed_stream, h, w, 3, "yuv420", 8, 8, seed=5)
    dec = decode_video_bytes(data, output_device="cuda")
    rng = np.random.default_rng(420)
    ints = [_ints(dec[str(i)]) for i in range(len(dec))]
    src = [[_noisy(p, 8, rng) for p in fr] for fr in ints]
    d = tmp_path_factory.mktemp("gop420")
    cool, yuv = str(d / "gop.cool"), str(d / f"src_{w}x{h}_30p_yuv420_8b.yuv")
    open(cool, "wb").write(data)
    np.concatenate([np.concatenate([p.reshape(-1) for p in fr]) for fr in src]).astype(np.uint8).tofile(yuv)
    return {"data": data, "cool": cool, "yuv": yuv, "dec": ints, "src": src, "h": h, "w": w}


@pytest.mark.gpu
def test_video_quality_gop420(ctx, gop420):
    from coolchic_b200.bitstream.quality import video_quality

    g = gop420
    video_quality(g["data"], g["yuv"], ms_ssim=True)  # warm
    n0 = ctx.launch_count()
    plain = video_quality(g["data"], g["yuv"])
    n1 = ctx.launch_count()
    q = video_quality(g["data"], g["yuv"], ms_ssim=True)
    assert ctx.launch_count() - n1 == n1 - n0 + 5
    assert sorted(fq.frame_type for fq in q.values()) == ["B", "I", "P"]
    for k, fq in q.items():
        i = int(k)
        assert fq.sse == plain[k].sse and plain[k].ms_ssim is None
        want = [check_ms_ssim(*check_scales(d, s, 255)[:2]) for d, s in zip(g["dec"][i], g["src"][i])]
        assert max(abs(a - b) for a, b in zip(fq.ms_ssim_planes, want)) < 1e-9, (k, fq.ms_ssim_planes, want)
        assert abs(fq.ms_ssim - (4 * want[0] + want[1] + want[2]) / 6) < 1e-9


@pytest.mark.gpu
def test_cc_eval_ms_ssim(ctx, gop420, tmp_path):
    g = gop420
    maps = str(tmp_path / "m.npz")
    out = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", g["cool"], "--original", g["yuv"],
                          "--ms_ssim", "--maps", maps], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    assert lines[i].split()[-5:] == ["ms_ssim", "ms_ssim_db", "ms_ssim_y", "ms_ssim_u", "ms_ssim_v"]
    rows = [ln.split() for ln in lines[i + 1:i + 4]]
    assert all(len(r) == 16 and 0 < float(r[11]) <= 1 for r in rows)
    assert any(ln.startswith("mean ms_ssim ") for ln in lines)
    z = np.load(maps)
    h, w = g["h"], g["w"]
    assert z["frame0_ssim_y"].shape == (h - 10, w - 10) and z["frame2_ssim_v"].shape == (h // 2 - 10, w // 2 - 10)
    assert "frame1_pred" in z and "frame0_error" in z


@pytest.mark.gpu
def test_small_frames_na(ctx, tmp_path, monkeypatch):
    """The golden 64 x 96 GOP is below the size rule: n/a everywhere, and no MS-SSIM launch."""
    from coolchic_b200.bitstream.quality import video_quality

    name = "gop5_64x96_yuv420"
    gold = np.load(os.path.join(GOLDEN, name + "_frames.npz"))
    n = len({k.split("_")[0] for k in gold.files})
    frames = [[gold[f"{i}_{c}"] for c in "yuv"] for i in range(n)]
    h, w = frames[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"g_{w}x{h}_yuv420_8b.yuv"
    np.concatenate([np.concatenate([p.reshape(-1) for p in fr]) for fr in frames]).astype(np.uint8).tofile(path)
    cool = os.path.join(GOLDEN, name + ".cool")
    data = open(cool, "rb").read()
    video_quality(data, path)  # warm
    n0 = ctx.launch_count()
    video_quality(data, path)
    n1 = ctx.launch_count()
    q = video_quality(data, path, ms_ssim=True, want_maps=True)
    assert ctx.launch_count() - n1 == n1 - n0
    assert all(fq.ms_ssim is None and fq.ssim_maps is None for fq in q.values())
    out = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", cool, "--original", path, "--ms_ssim"],
                         capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    assert all(ln.split()[-5:] == ["n/a"] * 5 for ln in lines[i + 1:i + 1 + n])
    assert any(ln.startswith("mean ms_ssim n/a") for ln in lines)
