"""Every bit depth the header allows (8 to 16): the decode path and the analyses above 10 bits.

Above 8 bits samples travel as int16 holding uint16 values, and the frame tails round on grids of up to 65535 levels.
The reference fixtures above 10 bits (oracle/gen_golden_bitdepths.py: 9-bit rgb, 12-bit 4:2:0, 16-bit 4:4:4 and rgb,
16-bit 4:2:0 and 13-bit rgb GOPs, each frame with samples at 0, at M = 2^b - 1 and, at 16 bits, far above 32768) pin
the decode and the writers' bytes to the unmodified reference.  The frame tails and the packing run at every bit depth
against the oracle bit for bit and against the float64 restatement of test_reference64.  The analyses (distortion,
MS-SSIM, prediction statistics, motion and grid analysis) run at 12 and 16 bits on sources with samples at 0, at M and
at 32768 or more, against numpy int64 / float64 restatements on the same integers.  The negative controls show that a
checker which sign-extends the int16 container, or a tail that rounds at M - 1, would be caught."""
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch
from conftest import GOLDEN, ROOT
from test_motion import _frame_sse, flow_stats
from test_quality import _check_dist, check_psnr
from test_reference64 import T, _stream, assert_within, check_levels, inter, intra, recon_inputs, to444
from test_ssim import _frame, _source, check_scales

BITDEPTHS = list(range(8, 17))
FORMATS = ["rgb", "yuv444", "yuv420"]
# name -> (format, bitdepth): oracle/gen_golden_bitdepths.py
FIXTURES = {"img_40x56_rgb_9bit": ("rgb", 9), "img_44x60_yuv420_12bit": ("yuv420", 12),
            "img_40x56_yuv444_16bit": ("yuv444", 16), "img_37x53_rgb_16bit": ("rgb", 16),
            "gop3_40x56_yuv420_16bit": ("yuv420", 16), "gop3_39x57_rgb_13bit": ("rgb", 13)}


# ---- helpers -------------------------------------------------------------------------------------------------------
def fixture_frames(name):
    """{display index: [three int64 planes]} of the reference's decode."""
    fmt, _ = FIXTURES[name]
    if name.startswith("img"):
        g = np.load(os.path.join(GOLDEN, name + ".npz"))
        return {0: [g[k].astype(np.int64) for k in "yuv"] if fmt == "yuv420" else list(g["rgb"].astype(np.int64))}
    g = np.load(os.path.join(GOLDEN, name + "_frames.npz"))
    n = len({k.split("_")[0] for k in g.files})
    return {i: [g[f"{i}_{k}"].astype(np.int64) for k in "yuv"] if fmt == "yuv420" else list(g[str(i)].astype(np.int64))
            for i in range(n)}


def int_planes(x, bitdepth):
    """Integer planes (int64) of a finished frame: numpy [3, H, W] or y / u / v dict, torch FrameData.data."""
    M = np.float32(2**bitdepth - 1)
    if isinstance(x, dict):
        ps = [x[k] for k in "yuv"]
    else:
        ps = [x.reshape(-1, *x.shape[-2:])[c] for c in range(3)]
    ps = [p.cpu().numpy() if hasattr(p, "cpu") else np.asarray(p) for p in ps]
    return [np.rint(p.reshape(p.shape[-2:]).astype(np.float32) * M).astype(np.int64) for p in ps]


def high_count(planes, bitdepth, what):
    """Samples >= 32768, printed; a 16-bit case must have at least 1 % of them."""
    n_hi = sum(int((p >= 32768).sum()) for p in planes)
    n = sum(p.size for p in planes)
    print(f"{what}: {n_hi} of {n} samples >= 32768")
    if bitdepth == 16:
        assert n_hi >= n // 100, f"{what}: only {n_hi} of {n} samples >= 32768"
    return n_hi


def sse_sign_extended(dec, src):
    """The wrong checker: the uint16 samples widened through the int16 container."""
    return [int(((d - s.astype(np.int16).astype(np.int64)) ** 2).sum()) for d, s in zip(dec, src)]


def analysis_planes(rng, shapes, bitdepth):
    """(decoded, source) integer planes: a ramp over the whole range plus texture, so that 0, M and (at 16 bits)
    values >= 32768 all occur; the source a few steps away, and at distance M from the decoded sample at a few
    pixels of every plane (decoded 0 / source M and the reverse)."""
    M = 2**bitdepth - 1
    dec, src = [], []
    for s in shapes:
        yy, xx = np.mgrid[0:s[0], 0:s[1]]
        base = (M * (0.5 + 0.7 * np.sin(yy / 13.0) * np.cos(xx / 17.0))).astype(np.int64)
        d = np.clip(base + rng.integers(-M // 16, M // 16 + 1, size=s), 0, M)
        e = np.clip(d + rng.integers(-M // 64 - 2, M // 64 + 3, size=s), 0, M)
        for k in range(4):
            y, x = int(rng.integers(0, s[0])), int(rng.integers(0, s[1]))
            d[y, x], e[y, x] = (0, M) if k % 2 else (M, 0)
        dec.append(d)
        src.append(e)
    return dec, src


def frame_shapes(h, w, fmt):
    return [(h, w)] + [(h // 2, w // 2) if fmt == "yuv420" else (h, w)] * 2


# ---- CPU: the fixtures -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(FIXTURES))
def test_oracle_vs_fixture(oracle, name):
    """The oracle's decode against the reference's: at most one level apart, and only at a handful of samples (rounding
    ties of two fp32 orders, whose count grows with M); every frame holds 0, M and, at 16 bits, samples >= 32768."""
    import pipeline

    fmt, bd = FIXTURES[name]
    M = 2**bd - 1
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    mine = pipeline.decode_video(data)
    gold = fixture_frames(name)
    assert sorted(mine) == sorted(gold)
    n_diff = n_all = 0
    for k, planes in gold.items():
        f, b, d = mine[k]
        assert (f, b) == (fmt, bd)
        assert any(int((p == 0).sum()) for p in planes) and any(int((p == M).sum()) for p in planes), (name, k)
        high_count(planes, bd, f"{name} frame {k}")
        for a, g in zip(int_planes(d, bd), planes):
            assert np.abs(a - g).max() <= 1, (name, k)
            n_diff += int((a != g).sum())
            n_all += a.size
    print(f"{name}: oracle and reference differ at {n_diff} of {n_all} samples (rounding ties)")
    assert n_diff <= n_all // 50


@pytest.mark.parametrize("name", list(FIXTURES))
def test_host_writers_vs_reference_bytes(name, tmp_path):
    """io's writers on the reference's frames write the reference writers' bytes: YUV 2-byte samples only at 10 bits
    (above, the low byte of each sample, as the reference's cast leaves it), PPM 2-byte samples MSB first."""
    import coolchic_b200  # noqa: F401
    from coolchic_b200.io import FrameData
    from coolchic_b200.io.io import save_frame_data_to_file

    fmt, bd = FIXTURES[name]
    M = np.float32(2**bd - 1)
    ext = ".ppm" if fmt == "rgb" else ".yuv"
    out = str(tmp_path / ("o" + ext))
    for k, planes in sorted(fixture_frames(name).items()):
        t = [torch.from_numpy(p.astype(np.float32) / M) for p in planes]
        data = {c: x[None, None] for c, x in zip("yuv", t)} if fmt == "yuv420" else torch.stack(t)[None]
        save_frame_data_to_file(FrameData(bd, fmt, data), out, append=k != 0)
    assert open(out, "rb").read() == open(os.path.join(GOLDEN, name + ext), "rb").read()


def test_yuv_reader_bitdepth_from_name(tmp_path, monkeypatch):
    """The yuv reader's bit depth comes from the file name, as the reference's does (io/io.py): "_8b" anywhere in the
    path is 8 bits, anything else 10 bits, 2-byte little-endian samples; "444" anywhere is 4:4:4."""
    import coolchic_b200  # noqa: F401
    from coolchic_b200.io.io import read_samples

    monkeypatch.chdir(tmp_path)
    h, w = 4, 6
    for name, bd, fmt in [("a_6x4_8b.yuv", 8, "yuv420"), ("a_6x4_10b.yuv", 10, "yuv420"),
                          ("a_6x4_12b.yuv", 10, "yuv420"), ("a_6x4_16b_444.yuv", 10, "yuv444"),
                          ("a_6x4_444_8b.yuv", 8, "yuv444"), ("a_6x4.yuv", 10, "yuv420")]:
        n = h * w + 2 * (h * w if fmt == "yuv444" else (h // 2) * (w // 2))
        vals = (np.arange(n) * 37) % (2**bd)
        vals.astype(np.uint8 if bd == 8 else "<u2").tofile(name)
        s = read_samples(name, 0)
        assert (s.bitdepth, s.frame_data_type, tuple(s.img_size)) == (bd, fmt, (h, w)), name
        assert np.array_equal(s.samples.astype(np.int64), vals), name


# ---- CPU: negative controls ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_sign_extending_checker_is_detected(fmt):
    """Widening the int16 container without a view to uint16 changes the SSE of every 16-bit case."""
    rng = np.random.default_rng(16)
    dec, src = analysis_planes(rng, frame_shapes(40, 56, fmt), 16)
    high_count(src, 16, f"{fmt} 16-bit source")
    right = [int(((d - s) ** 2).sum()) for d, s in zip(dec, src)]
    wrong = sse_sign_extended(dec, src)
    assert all(a != b for a, b in zip(right, wrong))
    # and on the sources of the analysis tests below
    for shapes in (frame_shapes(181, 179, "rgb"), frame_shapes(352, 356, "yuv420")):
        d, s = analysis_planes(np.random.default_rng(3), shapes, 16)
        assert sse_sign_extended(d, s) != [int(((a - b) ** 2).sum()) for a, b in zip(d, s)]
    print("negative control sign_extension: detected")


@pytest.mark.parametrize("bd", BITDEPTHS[1:])
def test_tail_rounded_at_m_minus_1_is_detected(oracle, bd):
    """The oracle's tail passes check_levels at this bit depth; the same prediction rounded on the M - 1 grid fails."""
    for fmt in ("rgb", "yuv444"):
        residue, motion, refs, gf = recon_inputs(fmt, bd, False, 8)
        x = inter(residue, motion, refs, gf, 8)
        pre = oracle.inter_predict(residue, motion, refs[0], None, gf, 8)
        err = assert_within(pre, x, f"{fmt} {bd}-bit oracle prediction")
        check_levels(oracle.finish_frame(pre, bd, fmt), x, bd, fmt, "oracle", window=err)
        M1 = 2**bd - 2
        bad = (np.round(np.clip(pre.astype(np.float64), 0, 1) * M1) / M1).astype(np.float32)
        with pytest.raises(AssertionError):
            check_levels(bad, x, bd, fmt, "rounded at M - 1", window=err)
    print(f"negative control rounding at M - 1, {bd} bits: detected")


# ---- GPU: decode against the reference -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(FIXTURES))
def test_decode_video_vs_reference(ctx, oracle, name, tmp_path):
    """decode_video with .yuv / .ppm output: frames equal to the oracle's, within one level of the reference's at the
    oracle's own rounding ties, and the file byte-equal to what the reference's writer wrote."""
    import pipeline

    from coolchic_b200.bitstream.decode import decode_video

    fmt, bd = FIXTURES[name]
    ext = ".ppm" if fmt == "rgb" else ".yuv"
    path = os.path.join(GOLDEN, name + ".cool")
    out = str(tmp_path / ("o" + ext))
    frames = decode_video(path, decoded_path=out)
    mine = pipeline.decode_video(open(path, "rb").read())
    gold = fixture_frames(name)
    assert sorted(frames) == [str(k) for k in sorted(gold)]
    n_diff = n_oracle = 0
    for k, planes in gold.items():
        fd = frames[str(k)]
        assert (fd.frame_data_type, fd.bitdepth) == (fmt, bd)
        got = int_planes(fd.data, bd)
        for a, o, g in zip(got, int_planes(mine[k][2], bd), planes):
            assert np.array_equal(a, o), (name, k)
            assert np.abs(a - g).max() <= 1, (name, k)
            n_diff += int((a != g).sum())
            n_oracle += int((o != g).sum())
    assert n_diff == n_oracle
    print(f"{name}: {n_diff} samples differ from the reference (rounding ties)")
    # the file: the reference writer's bytes for these frames (the host writers, pinned to the reference's bytes by
    # test_host_writers_vs_reference_bytes), and the reference's own file but at the bytes of those tie samples
    got = open(out, "rb").read()
    gold_bytes = open(os.path.join(GOLDEN, name + ext), "rb").read()
    from coolchic_b200.io.io import save_frame_data_to_file

    host = str(tmp_path / ("h" + ext))
    for k in sorted(gold):
        save_frame_data_to_file(frames[str(k)], host, append=k != 0)
    assert got == open(host, "rb").read()
    assert len(got) == len(gold_bytes)
    n_bytes = int((np.frombuffer(got, np.uint8) != np.frombuffer(gold_bytes, np.uint8)).sum())
    assert n_bytes <= 2 * n_diff and (n_diff > 0 or got == gold_bytes)


# ---- GPU: frame tails and packing at every bit depth ------------------------------------------------------------------
def _exact(x):
    """A float64 T of fp32 input values: no rounding before the tail."""
    return T(torch.from_numpy(np.asarray(x, dtype=np.float64)))


@pytest.mark.gpu
@pytest.mark.parametrize("bd", BITDEPTHS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_finish_frame(ctx, oracle, fmt, bd):
    rng = np.random.default_rng(bd)
    M = 2**bd - 1
    x = rng.uniform(-0.3, 1.3, size=(3, 37, 50)).astype(np.float32)
    x[0, 0, :8] = (np.arange(8) + 0.5) / M          # ties of the rounding grid at the bottom
    x[1, 0, :8] = (M - 8 + np.arange(8) + 0.5) / M  # and at the top
    got = ctx.finish_frame(torch.from_numpy(x[None]).cuda(), bd, fmt)
    want = oracle.finish_frame(x, bd, fmt)
    if fmt == "yuv420":
        got = {k: got[k][0, 0].cpu().numpy() for k in "yuv"}
        assert all(np.array_equal(got[k], want[k]) for k in "yuv")
    else:
        got = got[0].cpu().numpy()
        assert np.array_equal(got, want)
    n_tie, n_diff = check_levels(got, _exact(x), bd, fmt, f"finish_frame {fmt} {bd}")
    print(f"{fmt} {bd}: {n_tie} samples at a rounding tie, {n_diff} differ")


# the shapes of test_gpu_decode.py::test_fused_frame_tail_equals_separate_kernels, one per (format, bit depth)
FUSED_SHAPES = {"rgb": [((96, 160), (0, 4)), ((64, 64), (0, 1)), ((33, 47), (0, 2))],
                "yuv444": [((33, 47), (0, 2)), ((96, 160), (0, 4)), ((64, 64), (0, 1))],
                "yuv420": [((96, 160), (0, 4)), ((50, 70), (0, 3))]}


@pytest.mark.gpu
@pytest.mark.parametrize("bd", BITDEPTHS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_fused_frame_tail(ctx, oracle, seed_stream, fmt, bd):
    """The tail fused into the synthesis kernel against ccd_finish_frame on the raw output, the oracle, and the
    restatement's levels within the raw output's measured error of a tie."""
    hw, lr = FUSED_SHAPES[fmt][bd % len(FUSED_SHAPES[fmt])]
    h, d, nnb, lb, lat = _stream(ctx, seed_stream, (hw, lr, None, None, None, (bd, fmt), 5))
    raw = ctx.decode_coolchic(d, nnb, lb)
    sep = ctx.finish_frame(raw, bd, fmt)
    fin, _ = ctx.decode_many([d], [nnb], [lb], finish=[(bd, fmt)])
    nn = oracle.decode_nn(d, nnb)
    want = oracle.finish_frame(oracle.synthesize(d, nn, lat), bd, fmt)
    if fmt == "yuv420":
        got = {k: fin[0][k][0, 0].cpu().numpy() for k in "yuv"}
        for k in "yuv":
            assert torch.equal(fin[0][k], sep[k]) and np.array_equal(got[k], want[k]), k
    else:
        got = fin[0][0].cpu().numpy()
        assert torch.equal(fin[0], sep) and np.array_equal(got, want)
    x = intra(h, nn, lat)
    err = assert_within(raw[0].cpu().numpy(), x, f"{hw} raw")
    n_tie, n_diff = check_levels(got, x, bd, fmt, f"fused {fmt} {bd}", window=err)
    print(f"{fmt} {bd} {hw}: {n_tie} samples within the error of a rounding tie, {n_diff} differ")


@pytest.mark.gpu
@pytest.mark.parametrize("is_b,fs", [(False, 8), (True, 8), (False, 2), (True, 2)])
@pytest.mark.parametrize("bd", BITDEPTHS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_reconstruct_frame(ctx, oracle, fmt, bd, is_b, fs):
    """P / B reconstruction (grid_sample bilinear and sinc-8) against the oracle bit for bit and the restatement's
    levels, from references whose samples cover the whole range."""
    from coolchic_b200.io import FrameData

    residue, motion, refs, gf = recon_inputs(fmt, bd, is_b, fs)
    r444 = [to444(r) for r in refs]
    want = oracle.finish_frame(oracle.inter_predict(residue, motion, r444[0], r444[1] if is_b else None, gf, fs), bd, fmt)

    def to_fd(r):
        if fmt == "yuv420":
            return FrameData(bd, fmt, {k: torch.from_numpy(v[None, None]).cuda() for k, v in r.items()})
        return FrameData(bd, fmt, torch.from_numpy(r[None]).cuda())

    res_d, mot_d = torch.from_numpy(residue[None]).cuda(), torch.from_numpy(motion[None]).cuda()
    got = ctx.reconstruct_frame(res_d, mot_d, [to_fd(r) for r in refs], is_b, fmt, bd, gf, fs)
    got = {k: got[k][0, 0].cpu().numpy() for k in "yuv"} if fmt == "yuv420" else got[0].cpu().numpy()
    if fmt == "yuv420":
        assert all(np.array_equal(got[k], want[k]) for k in "yuv")
    else:
        assert np.array_equal(got, want)
    x = inter(residue, motion, r444, gf, fs)
    pre = ctx.inter_predict(res_d, mot_d, [FrameData(bd, "rgb", torch.from_numpy(r[None]).cuda()) for r in r444],
                            is_b, "rgb", gf, fs)
    err = assert_within(pre[0].cpu().numpy(), x, f"{fmt} {bd} prediction")
    n_tie, n_diff = check_levels(got, x, bd, fmt, f"reconstruct {fmt} {bd}", window=err)
    print(f"{fmt} {bd} {'B' if is_b else 'P'} fs{fs}: {n_tie} samples within the error of a tie, {n_diff} differ")


@pytest.mark.gpu
@pytest.mark.parametrize("bd", BITDEPTHS)
@pytest.mark.parametrize("fmt", FORMATS)
def test_pack_frame(ctx, fmt, bd):
    """Planar and HWC packing (odd sizes where the format allows), and pack_frames in one launch and one by one,
    against the integers the frame was made of."""
    rng = np.random.default_rng(100 + bd)
    h, w = (36, 50) if fmt == "yuv420" else (37, 53)
    M = 2**bd - 1
    planes = [rng.integers(0, M + 1, size=s) for s in frame_shapes(h, w, fmt)]
    for p in planes:
        p[0, :2] = (0, M)
    high_count(planes, bd, f"pack {fmt} {bd}")
    ts = [torch.from_numpy((p.astype(np.float32) / np.float32(M))).cuda() for p in planes]
    data = {k: t[None, None] for k, t in zip("yuv", ts)} if fmt == "yuv420" else torch.stack(ts)[None]
    assert all(np.array_equal(a, b) for a, b in zip(int_planes(data, bd), planes))
    dt = np.uint8 if bd <= 8 else np.uint16
    want = np.concatenate([p.reshape(-1) for p in planes]).astype(dt)
    got = ctx.pack_frame(data, bd, fmt).cpu().numpy().view(dt)
    assert np.array_equal(got.astype(np.int64), want.astype(np.int64))
    if fmt != "yuv420":
        got = ctx.pack_frame(data, bd, fmt, interleaved=True).cpu().numpy().view(dt)
        assert np.array_equal(got.astype(np.int64), np.stack(planes, -1).reshape(-1))
    flat = torch.cat([t.reshape(-1) for t in ts] * 3)
    n_fr = flat.numel() // 3
    sizes = [p.size for p in planes]
    batch = []
    for i in range(3):
        parts = torch.split(flat[i * n_fr:(i + 1) * n_fr], sizes)
        batch.append({k: v.view(1, 1, *p.shape) for k, v, p in zip("yuv", parts, planes)} if fmt == "yuv420"
                     else flat[i * n_fr:(i + 1) * n_fr].view(1, 3, h, w))
    launches = ctx.launch_count()
    got = ctx.pack_frames(batch, bd, fmt).cpu().numpy().view(dt)
    assert ctx.launch_count() == launches + 1
    assert np.array_equal(got.astype(np.int64), np.tile(want, 3).astype(np.int64))
    loose = [{k: v.clone() for k, v in b.items()} if fmt == "yuv420" else b.clone() for b in batch]
    assert np.array_equal(ctx.pack_frames(loose, bd, fmt).cpu().numpy().view(dt), np.tile(want, 3))


# ---- GPU: the analyses at 12 and 16 bits -------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("bd", [12, 16])
def test_frame_distortion_and_ssim(ctx, bd):
    """frame_distortion (SSE, max_abs, error map) and frame_ssim (cs / ssim per scale, map) against numpy int64 /
    float64, planar and HWC; one frame at M everywhere (every MS-SSIM level sum at its maximum, 65535 * 4^j at 16
    bits) against itself and against a textured source."""
    M = 2**bd - 1
    rng = np.random.default_rng(bd)
    cases = [(181, 179, "rgb", "hwc"), (176, 190, "yuv444", "planar"), (352, 356, "yuv420", "planar"),
             (40, 57, "rgb", "planar"), (38, 56, "yuv420", "planar")]
    frames, srcs, lays, ints = [], [], [], []
    for h, w, fmt, lay in cases:
        dec, src = analysis_planes(rng, frame_shapes(h, w, fmt), bd)
        high_count(src, bd, f"{h}x{w} {fmt} {bd}-bit source")
        frames.append(_frame(ctx, dec, fmt, bd))
        srcs.append(_source(ctx, src, bd, lay))
        lays.append(lay)
        ints.append((dec, src))
    full = [np.full((176, 180), M, dtype=np.int64)] * 3
    _, tex = analysis_planes(rng, frame_shapes(176, 180, "rgb"), bd)
    for src, lay in ((full, "hwc"), (tex, "planar")):
        frames.append(_frame(ctx, full, "rgb", bd))
        srcs.append(_source(ctx, src, bd, lay))
        lays.append(lay)
        ints.append((full, src))
    dist = ctx.frame_distortion(frames, srcs, lays, want_maps=True)
    for r, (dec, src) in zip(dist, ints):
        _check_dist(r, dec, src, bd, r["map"])
        assert r["sse"] != sse_sign_extended(dec, src) or bd < 16 or r["sse"] == [0, 0, 0]
    assert M in dist[0]["max_abs"]  # decoded and source M apart: the largest squared error a sample can have
    big = [i for i, (h, w, fmt, _) in enumerate(cases) if min(h, w) >> (fmt == "yuv420") >= 176] + [5, 6]
    res = ctx.frame_ssim([frames[i] for i in big], [srcs[i] for i in big], [lays[i] for i in big], want_maps=True)
    for i, r in zip(big, res):
        dec, src = ints[i]
        for c in range(3):
            cs, ssim, m0 = check_scales(dec[c], src[c], M)
            assert max(abs(a - b) for a, b in zip(r["cs"][c], cs)) < 1e-10, (i, c, r["cs"][c], cs)
            assert max(abs(a - b) for a, b in zip(r["ssim"][c], ssim)) < 1e-10, (i, c, r["ssim"][c], ssim)
            assert np.abs(r["maps"][c].cpu().numpy() - m0).max() < 1e-6
    assert res[-2]["cs"] == [[1.0] * 5] * 3 and res[-2]["ssim"] == [[1.0] * 5] * 3


def _pb_case(fmt, bd, is_b, fs, oracle):
    """Inputs of a P / B frame, its source integers (the oracle's decode, moved a few steps, with samples at 0, M, and
    pixels M away from the decoded sample) and the source's layout."""
    residue, motion, refs, gf = recon_inputs(fmt, bd, is_b, fs)
    r444 = [to444(r) for r in refs]
    fin = oracle.finish_frame(oracle.inter_predict(residue, motion, r444[0], r444[1] if is_b else None, gf, fs), bd, fmt)
    M = 2**bd - 1
    rng = np.random.default_rng(bd + 7 * is_b)
    src = []
    for k in int_planes(fin, bd):
        s = np.clip(k + rng.integers(-M // 32, M // 32 + 1, size=k.shape), 0, M)
        s[0, :4] = np.where(k[0, :4] > M // 2, 0, M)  # M or nearly M away
        s[1, :2] = (0, M)
        src.append(s)
    return residue, motion, refs, r444, gf, src, ("hwc" if fmt == "rgb" else "planar")


@pytest.mark.gpu
@pytest.mark.parametrize("is_b,fs", [(False, 8), (True, 2)])
@pytest.mark.parametrize("fmt", FORMATS)
@pytest.mark.parametrize("bd", [12, 16])
def test_inter_stats_and_analysis(ctx, oracle, bd, fmt, is_b, fs):
    """inter_stats' sums against math.fsum on the oracle's prediction and the source read as k / M; inter_analysis'
    SSE of every variant against numpy int64 on the oracle's frames, and its flow statistics against float64."""
    from coolchic_b200.bitstream.motion import VARIANT_NAMES, variant_inputs, variants_of
    from coolchic_b200.io import FrameData

    residue, motion, refs, r444, gf, src, lay = _pb_case(fmt, bd, is_b, fs, oracle)
    high_count(src, bd, f"{fmt} {bd}-bit {'B' if is_b else 'P'} source")
    M = 2**bd - 1
    dt = np.int16 if bd > 8 else np.uint8
    flat = np.stack(src, -1).reshape(-1) if lay == "hwc" else np.concatenate([p.reshape(-1) for p in src])
    s_dev = torch.from_numpy(flat.astype(dt)).cuda()

    def to_fd(r):
        if fmt == "yuv420":
            return FrameData(bd, fmt, {k: torch.from_numpy(v[None, None]).cuda() for k, v in r.items()})
        return FrameData(bd, fmt, torch.from_numpy(r[None]).cuda())

    res_d, mot_d = torch.from_numpy(residue[None]).cuda(), torch.from_numpy(motion[None]).cuda()
    args = (res_d, mot_d, [to_fd(r) for r in refs], is_b, fmt, bd, gf, fs)
    # prediction statistics
    st = ctx.inter_stats(*args, source=s_dev, layout=lay, want_maps=True)
    probe = residue.copy()
    probe[:3], probe[3] = 0.0, 0.5
    pred = oracle.inter_predict(probe, motion, r444[0], r444[1] if is_b else None, gf, fs)
    assert np.array_equal(st["pred"].cpu().numpy(), pred)
    orig = np.stack([np.repeat(np.repeat(p, 2, 0), 2, 1) if p.shape != src[0].shape else p for p in src])
    orig = orig.astype(np.float32) / np.float32(M)
    alpha = np.clip(residue[3] + np.float32(0.5), 0, 1).astype(np.float32)
    beta = np.clip(residue[4] + np.float32(0.5), 0, 1).astype(np.float32) if is_b else np.zeros_like(alpha)
    dummy = (np.float32(0) + r444[0]) + (r444[1] if is_b else np.float32(0))
    dummy = (dummy / np.float32(2 if is_b else 1)).astype(np.float32)
    e, f = (pred - orig).astype(np.float32), (dummy - orig).astype(np.float32)
    want = [math.fsum(alpha.ravel().tolist()), math.fsum(beta.ravel().tolist()),
            math.fsum((e * e).astype(np.float32).ravel().tolist()), math.fsum((f * f).astype(np.float32).ravel().tolist())]
    for got, wt in zip(st["sums"], want):
        assert abs(got - wt) <= 1e-12 * max(abs(wt), 1e-300), (got, wt)
    # motion analysis
    a = ctx.inter_analysis(*args, source=s_dev, layout=lay, want_maps=True)
    n_checked = 0
    for k, v in enumerate(VARIANT_NAMES):
        if v not in variants_of("B" if is_b else "P"):
            assert a["sse"][k] is None
            continue
        r, m, g = variant_inputs(residue, motion, gf, v)
        fin = oracle.finish_frame(oracle.inter_predict(r, m, r444[0], r444[1] if is_b else None, g, fs), bd, fmt)
        assert a["sse"][k] == _frame_sse(fin, src, fmt, bd), v
        if v == "decoded":
            assert a["sse"][k] != sse_sign_extended(int_planes(fin, bd), src) or bd < 16
        n_checked += 1
    assert n_checked == (7 if is_b else 5)
    for got, wt in zip(a["refs"], flow_stats(motion, gf, 2 if is_b else 1)):
        for x, y in zip(got["sum"], wt["sum"]):
            assert abs(x - y) <= 1e-12 * max(abs(y), 1e-300), (x, y)
        assert got["max"] == wt["max"] and got["outside"] == wt["outside"]
        assert torch.equal(got["flow"].cpu(), torch.from_numpy(wt["flow"]))


# ---- GPU: end to end through the file readers ---------------------------------------------------------------------------
def _ppm_source(name, path, seed):
    """A 16-bit (or 13-bit) PPM source per frame of an rgb fixture: the reference's frame moved a few steps, with samples
    M away from it; returns the integer planes per display index."""
    from coolchic_b200.io.io import write_ppm

    _, bd = FIXTURES[name]
    M = 2**bd - 1
    rng = np.random.default_rng(seed)
    out = {}
    for k, planes in fixture_frames(name).items():
        s = [np.clip(p + rng.integers(-M // 40, M // 40 + 1, size=p.shape), 0, M) for p in planes]
        for p, q in zip(s, planes):
            p[0, :3] = np.where(q[0, :3] > M // 2, 0, M)
        write_ppm(torch.from_numpy(np.stack(s).astype(np.float32)) / np.float32(M), bd, path.format(k))
        out[k] = s
    return out


@pytest.mark.gpu
def test_cc_eval_16bit_ppm(ctx, oracle, tmp_path):
    """cc_eval.py on a 16-bit stream and a 16-bit PPM source: the PSNR columns against check_psnr of numpy int64 SSEs of
    the oracle's frame; the grid analysis' PSNRs against the oracle's variants."""
    from test_grids import _check_analysis

    from coolchic_b200.io.io import read_samples

    name = "img_37x53_rgb_16bit"
    path = os.path.join(GOLDEN, name + ".cool")
    src_path = str(tmp_path / "src.ppm")
    src = _ppm_source(name, str(tmp_path / "src{}.ppm"), 9)
    os.rename(str(tmp_path / "src0.ppm"), src_path)
    s = read_samples(src_path, 0)
    assert s.bitdepth == 16 and np.array_equal(s.samples.astype(np.int64), np.stack(src[0], -1))
    high_count(src[0], 16, "cc_eval source")
    import pipeline

    dec = int_planes(pipeline.decode_video(open(path, "rb").read())[0][2], 16)
    sse = [int(((d - q) ** 2).sum()) for d, q in zip(dec, src[0])]
    assert sse != sse_sign_extended(dec, src[0])
    psnr, planes = check_psnr(sse, [p.size for p in dec], 16)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", path, "--original", src_path, "--grids"],
                       capture_output=True, text=True, cwd=ROOT)
    assert r.returncode == 0, r.stderr
    lines = r.stdout.splitlines()
    row = lines[lines.index(next(x for x in lines if x.startswith("frame_idx"))) + 1].split()
    assert row[:2] == ["0", "I"]
    got = [float(v) for v in row[2:6]]
    assert all(abs(g - w) < 1e-6 for g, w in zip(got, [psnr] + planes)), (got, psnr, planes)
    assert re.search(r"grids frame 0 I residue psnr_db " + f"{psnr:.6f}", r.stdout)
    print(f"cc_eval 16-bit: psnr_db {psnr:.6f}, planes {planes}")
    _check_analysis(ctx, oracle, name, open(path, "rb").read(), src_path, [src[0]])
