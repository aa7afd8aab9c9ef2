"""Quality analysis (coolchic_b200.bitstream.quality, ccd_frame_distortion, ccd_inter_stats) and the source readers
(coolchic_b200.io.io.read_samples / load_frame_data_from_file).

The readers are checked against what the unmodified reference's load_frame_data_from_file returns for a few of its
own test sources (oracle/gen_golden_originals.py).  The GPU tests compare the distortion with numpy int64 on the
golden GOPs and kodim14, against sources made of the reference-decoded frames plus seeded integer noise, and the
prediction statistics with the oracle's inter prediction and math.fsum."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT

ORIGINALS = {"kodim15_192x128_01p_yuv420_10b.yuv": 1, "kodim15_192x128_01p_yuv444_8b.yuv": 1,
             "192x128_kodim15.png": 1, "D-BQSquare-3frames_224x128_60p_yuv420_8b.yuv": 3}
GOPS = [("gop5_64x96_yuv420", "yuv420"), ("gop3_40x56_rgb", "rgb"), ("gop3_48x72_yuv420_bilinear", "yuv420"),
        ("gop3_40x56_rgb_bicubic", "rgb"), ("gop3_48x72_yuv420_sinc6", "yuv420"), ("gop4_40x56_rgb_sinc12", "rgb"),
        # every network weight live (oracle/gen_golden_dense.py): alpha and beta vary per pixel and differ
        ("gop3_40x56_rgb_sinc8_dense", "rgb"), ("gop3_48x72_yuv420_bicubic_dense", "yuv420")]


# ---- checker: the reference's formulas restated on integer errors ------------------------------------------------
def dist_to_db(dist):
    """metrics/mse.py:18-21."""
    return -10 * math.log10(max(dist, 10 ** (-100 / 10)))


def check_psnr(sse, n, bitdepth):
    """(psnr_db, [psnr per plane]) of loss.py:88-118: pixel-weighted MSE over the planes."""
    m2 = float(2**bitdepth - 1) ** 2
    return dist_to_db(sum(sse) / m2 / sum(n)), [dist_to_db(s / m2 / k) for s, k in zip(sse, n)]


def check_pred_db(sse, n):
    """training/test.py:188-199."""
    return -10 * math.log10(sse / n + 1e-10)


def _planes_int(fd, bitdepth):
    """Integer planes (int64) of a decoded FrameData (any device)."""
    M = 2**bitdepth - 1
    if fd.frame_data_type == "yuv420":
        ts = [fd.data[k][0, 0] for k in "yuv"]
    else:
        ts = [fd.data[0, c] for c in range(3)]
    return [np.rint(t.cpu().numpy().astype(np.float32) * np.float32(M)).astype(np.int64) for t in ts]


def _check_dist(r, dec, src, bitdepth, map_=None):
    """sse / max_abs exactly, the error map bit for bit."""
    d = [a - b for a, b in zip(dec, src)]
    assert r["sse"] == [int((x * x).sum()) for x in d]
    assert r["max_abs"] == [int(np.abs(x).max()) for x in d]
    if map_ is not None:
        h, w = dec[0].shape
        e = d[0] * d[0]
        for x in d[1:]:
            x2 = x * x
            e = e + (x2 if x2.shape == (h, w) else np.repeat(np.repeat(x2, 2, 0), 2, 1))
        M = 2**bitdepth - 1
        want = e.astype(np.float32) / np.float32(M * M)
        assert np.array_equal(map_.cpu().numpy().view(np.uint32), want.view(np.uint32))


# ---- CPU: readers ----------------------------------------------------------------------------------------------
def test_read_samples_match_reference():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.io.io import load_frame_data_from_file, read_samples

    gold = np.load(os.path.join(GOLDEN, "originals_frames.npz"))
    for name, n in ORIGINALS.items():
        path = os.path.join(GOLDEN, name)
        for i in range(n):
            s = read_samples(path, i)
            b, h, w = (int(v) for v in gold[f"{name}/{i}/meta"])
            fmt = str(gold[f"{name}/{i}/type"])
            assert (s.bitdepth, tuple(s.img_size), s.frame_data_type) == (b, (h, w), fmt)
            assert s.samples.dtype == (np.uint8 if b <= 8 else np.uint16)
            keys = "yuv" if fmt == "yuv420" else "012"
            want = [gold[f"{name}/{i}/{c}"].astype(np.int64) for c in keys]
            if s.layout == "hwc":
                got = [s.samples[:, :, c].astype(np.int64) for c in range(3)]
            else:
                assert s.layout == "planar"
                sizes = [x.size for x in want]
                flat = s.samples.astype(np.int64)
                got = [flat[sum(sizes[:c]):sum(sizes[:c + 1])].reshape(want[c].shape) for c in range(3)]
            for g, wt in zip(got, want):
                assert np.array_equal(g, wt)
            fd = load_frame_data_from_file(path, i)
            assert (fd.bitdepth, fd.frame_data_type, tuple(fd.img_size)) == (b, fmt, (h, w))
            vals = [fd.data[c][0, 0] for c in "yuv"] if fmt == "yuv420" else [fd.data[0, c] for c in range(3)]
            for v, wt in zip(vals, want):
                ref = wt.astype(np.float32) / np.float32(2**b - 1)
                assert v.dtype.is_floating_point and np.array_equal(v.numpy().view(np.uint32), ref.view(np.uint32))


@pytest.mark.parametrize("bitdepth", [8, 10, 16])
def test_ppm_roundtrip(tmp_path, bitdepth):
    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200.io.io import read_samples, write_ppm

    rng = np.random.default_rng(bitdepth)
    M = 2**bitdepth - 1
    k = rng.integers(0, M + 1, size=(3, 6, 10))
    k[0, 0, 0], k[1, 0, 0] = 0, M
    path = str(tmp_path / "x.ppm")
    write_ppm(torch.from_numpy(k.astype(np.float32)) / M, bitdepth, path)
    s = read_samples(path, 0)
    assert (s.layout, s.bitdepth, tuple(s.img_size), s.frame_data_type) == ("hwc", bitdepth, (6, 10), "rgb")
    assert s.samples.dtype == (np.uint8 if bitdepth <= 8 else np.uint16)
    assert np.array_equal(s.samples.astype(np.int64), k.transpose(1, 2, 0))


def test_malformed_sources(tmp_path, monkeypatch):
    from PIL import Image

    import coolchic_b200  # noqa: F401
    from coolchic_b200.io.io import read_samples

    def bad(path, idx=0):
        with pytest.raises(ValueError):
            read_samples(str(path), idx)

    monkeypatch.chdir(tmp_path)  # bare names: the naming rules (_8b, 444) read the whole path
    bad("missing_8x8_yuv420_8b.yuv")
    bad("x.bmp")
    yuv = "seq_8x4_yuv420_8b.yuv"
    np.zeros(2 * 48, np.uint8).tofile(yuv)
    assert read_samples(str(yuv), 1).samples.size == 48
    bad(yuv, 2)
    bad(yuv, -1)
    short = "seq_8x4_yuv420_10b.yuv"
    np.zeros(48, np.uint8).tofile(short)  # half a 10-bit frame
    bad(short)
    noname = "seq_8by4_yuv420_8b.yuv"
    np.zeros(48, np.uint8).tofile(noname)
    bad(noname)
    for i, body in enumerate([b"P5 2 2 255\n" + bytes(12), b"P6 2 2 1000\n" + bytes(24), b"P6 2 2 255\n" + bytes(11),
                              b"P6 2 x 255\n" + bytes(12), b"P6 2 2", b"P6\n2  2 255\n" + bytes(12)]):
        p = tmp_path / f"b{i}.ppm"
        p.write_bytes(body)
        bad(p)
    ok = tmp_path / "ok.ppm"
    ok.write_bytes(b"P6\n2 2\n255\n" + bytes(range(12)))
    assert read_samples(str(ok), 0).samples.reshape(-1).tolist() == list(range(12))
    bad(ok, 1)
    gray = tmp_path / "g.png"
    Image.fromarray(np.zeros((4, 4), np.uint8), mode="L").save(gray)
    bad(gray)
    rgba = tmp_path / "a.png"
    px = np.arange(64, dtype=np.uint8).reshape(4, 4, 4)
    Image.fromarray(px, mode="RGBA").save(rgba)
    assert np.array_equal(read_samples(str(rgba), 0).samples, px[:, :, :3])
    bad(rgba, 1)
    (tmp_path / "junk.png").write_bytes(b"not a png")
    bad(tmp_path / "junk.png")


def test_psnr_formulas():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.quality import FrameQuality, dist_to_db as q_db, pred_to_db

    assert q_db(0.0) == 100.0 and dist_to_db(0.0) == 100.0
    assert abs(q_db(1e-4) - 40.0) < 1e-12
    assert abs(pred_to_db(0.0, 10) - 100.0) < 1e-12  # the 1e-10 term, not a clamp
    assert abs(pred_to_db(3e-12 * 30, 30) - check_pred_db(3e-12 * 30, 30)) < 1e-12
    assert pred_to_db(1e-12 * 30, 30) < 100.0
    q = FrameQuality(display_idx=0, frame_type="I", img_size=(4, 6), bitdepth=8, frame_data_type="yuv420", n_bytes=30,
                     sse=[100, 7, 0], n_samples=[24, 6, 6], max_abs=[3, 2, 0])
    psnr, planes = check_psnr([100, 7, 0], [24, 6, 6], 8)
    assert abs(q.psnr_db - psnr) < 1e-9 and q.psnr_v_db == 100.0
    assert [abs(a - b) < 1e-9 for a, b in zip([q.psnr_y_db, q.psnr_u_db, q.psnr_v_db], planes)] == [True] * 3
    # pixel-weighted mean of the plane MSEs (loss.py:88-118)
    assert abs(q.mse - (24 * q.mse_y + 6 * q.mse_u + 6 * q.mse_v) / 36) < 1e-15
    assert q.rate_bpp == 8 * 30 / 24


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _noisy(k, bitdepth, rng, amp=3):
    return np.clip(k.astype(np.int64) + rng.integers(-amp, amp + 1, size=k.shape), 0, 2**bitdepth - 1)


def _gop_sources(name, fmt, seed):
    """Per display frame: integer planes (int64) of the reference-decoded frame plus seeded noise."""
    gold = np.load(os.path.join(GOLDEN, name + "_frames.npz"))
    rng = np.random.default_rng(seed)
    n = len({k.split("_")[0] for k in gold.files})
    if fmt == "yuv420":
        return [[_noisy(gold[f"{i}_{c}"], 8, rng) for c in "yuv"] for i in range(n)]
    return [[_noisy(gold[str(i)][c], 8, rng) for c in range(3)] for i in range(n)]


def _write_yuv(path, frames, bitdepth=8):
    dt = np.uint8 if bitdepth == 8 else np.dtype("<u2")
    np.concatenate([np.concatenate([p.reshape(-1) for p in fr]) for fr in frames]).astype(dt).tofile(path)


def _write_rgb(path, planes):
    from PIL import Image

    import torch

    from coolchic_b200.io.io import write_ppm

    hwc = np.stack(planes, -1).astype(np.uint8)
    if path.endswith(".png"):
        Image.fromarray(hwc, mode="RGB").save(path)
    else:
        write_ppm(torch.from_numpy(hwc.transpose(2, 0, 1).astype(np.float32)) / 255, 8, path)


def _decode_cpu(data, **kw):
    from coolchic_b200.bitstream.decode import decode_video_bytes

    return decode_video_bytes(data, **kw)


@pytest.mark.gpu
@pytest.mark.parametrize("name", [g[0] for g in GOPS if g[1] == "yuv420"])
def test_video_quality_yuv_gop(ctx, name, tmp_path, monkeypatch):
    """video_quality on a 4:2:0 GOP: every frame's SSE / max_abs against numpy int64, PSNR against the checker,
    error map bit-equal; then the same source with frame_offset and the decoded frames against themselves."""
    from coolchic_b200.bitstream.quality import video_quality

    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    dec = _decode_cpu(data)
    srcs = _gop_sources(name, "yuv420", seed=len(name))
    h, w = srcs[0][0].shape
    monkeypatch.chdir(tmp_path)  # bare names: the naming rules (_8b, 444) read the whole path
    path = f"src_{w}x{h}_30p_yuv420_8b.yuv"
    _write_yuv(path, [srcs[0]] + srcs)  # one leading frame: the video starts at frame_offset 1
    q = video_quality(data, path, frame_offset=1, want_maps=True)
    assert list(q) == [str(i) for i in range(len(dec))]
    for k, fq in q.items():
        i = int(k)
        di = _planes_int(dec[k], 8)
        _check_dist({"sse": fq.sse, "max_abs": fq.max_abs}, di, srcs[i], 8, fq.error_map)
        psnr, planes = check_psnr(fq.sse, [x.size for x in di], 8)
        assert abs(fq.psnr_db - psnr) < 1e-9
        assert all(abs(a - b) < 1e-9 for a, b in zip([fq.psnr_y_db, fq.psnr_u_db, fq.psnr_v_db], planes))
        assert fq.frame_type == ("I" if i == 0 else fq.frame_type) and fq.rate_bpp > 0
        if fq.frame_type != "I":
            assert fq.pred_map is not None and 0 <= fq.alpha_mean <= 1
            assert fq.frame_type == "B" or fq.beta_mean == 0
    # the decoded frames themselves as the source: MSE 0, 100 dB
    same = f"self_{w}x{h}_30p_yuv420_8b.yuv"
    _write_yuv(same, [_planes_int(dec[str(i)], 8) for i in range(len(dec))])
    for fq in video_quality(data, same).values():
        assert fq.sse == [0, 0, 0] and fq.mse == 0 and fq.psnr_db == 100.0 and fq.max_abs == [0, 0, 0]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [g[0] for g in GOPS if g[1] == "rgb"])
def test_frame_distortion_rgb_gop(ctx, name, tmp_path):
    """RGB GOP frames against PNG / PPM sources read back by read_samples: one frame_distortion call for all."""
    import torch

    from coolchic_b200.io.io import read_samples

    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    dec = _decode_cpu(data, output_device="cuda")
    srcs = _gop_sources(name, "rgb", seed=len(name))
    h, w = srcs[0][0].shape
    frames, tens, lays, want = [], [], [], []
    for i, planes in enumerate(srcs):
        for ext in (".png", ".ppm"):
            p = str(tmp_path / f"f{i}{ext}")
            _write_rgb(p, planes)
            s = read_samples(p, 0)
            frames.append(dec[str(i)])
            tens.append(torch.from_numpy(s.samples.reshape(-1)).to(ctx.torch_device))
            lays.append(s.layout)
            want.append(planes)
    launches = ctx.launch_count()
    res = ctx.frame_distortion(frames, tens, lays, want_maps=True)
    assert ctx.launch_count() == launches + 1
    for fd, r, planes in zip(frames, res, want):
        _check_dist(r, _planes_int(fd, 8), planes, 8, r["map"])


@pytest.mark.gpu
@pytest.mark.parametrize("ext", [".png", ".ppm"])
def test_video_quality_kodim14(ctx, kodim14, ext, tmp_path):
    from coolchic_b200.bitstream.quality import video_quality

    dec = _decode_cpu(kodim14["data"])
    di = _planes_int(dec["0"], 8)
    rng = np.random.default_rng(14)
    src = [_noisy(x, 8, rng, amp=5) for x in di]
    path = str(tmp_path / ("kodim14" + ext))
    _write_rgb(path, src)
    fq = video_quality(kodim14["data"], path, want_maps=True)["0"]
    _check_dist({"sse": fq.sse, "max_abs": fq.max_abs}, di, src, 8, fq.error_map)
    psnr, _ = check_psnr(fq.sse, [x.size for x in di], 8)
    assert abs(fq.psnr_db - psnr) < 1e-9
    assert fq.n_bytes <= len(kodim14["data"]) and fq.pred_psnr_db == 0 and fq.alpha_mean == 0
    _write_rgb(path, di)
    fq = video_quality(kodim14["data"], path)["0"]
    assert fq.mse == 0 and fq.psnr_db == 100.0


def _to444(fd):
    """convert_420_to_444 (nearest) of a reference frame, as numpy [3, H, W]."""
    if fd.frame_data_type != "yuv420":
        return fd.data[0].cpu().numpy()
    up = [np.repeat(np.repeat(fd.data[c][0, 0].cpu().numpy(), 2, 0), 2, 1) for c in "uv"]
    return np.stack([fd.data["y"][0, 0].cpu().numpy()] + up)


@pytest.mark.gpu
@pytest.mark.parametrize("name,fmt", GOPS)
def test_inter_stats(ctx, oracle, name, fmt):
    """k_inter_stats on every P / B frame: the prediction bit-equal to the oracle's inter prediction with alpha = 1
    and a zero residue, alpha / beta maps bit-equal, the four sums against math.fsum and repeatable."""
    import torch

    from coolchic_b200.bitstream import decode

    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, fmt, seed=7)
    seen = []

    def recon(fh, cc_out, refs, dev):
        seen.append((fh, dict(cc_out), [r.to(ctx.torch_device) for r in refs]))
        return decode._reconstruct(fh, cc_out, refs, dev)

    from coolchic_b200.bitstream.header import VideoHeader

    vh = VideoHeader()
    vh.read_header(memoryview(data))
    cs = vh.get_coding_structure()
    decode.decode_video_bytes(data, output_device="cuda", reconstruct_fn=recon)
    n_inter = 0
    for coding_idx, (fh, cc, refs) in enumerate(seen):
        ft = fh.get_value("frame_type")
        if ft == "I":
            continue
        n_inter += 1
        disp = cs.get_frame_from_coding_order(coding_idx).display_order
        is_b = ft == "B"
        planes = srcs[disp]
        h, w = planes[0].shape
        if fmt == "yuv420":
            src = torch.from_numpy(np.concatenate([p.reshape(-1) for p in planes]).astype(np.uint8)).to(ctx.torch_device)
            layout = "planar"
            orig = np.stack([planes[0]] + [np.repeat(np.repeat(p, 2, 0), 2, 1) for p in planes[1:]])
        else:
            src = torch.from_numpy(np.stack(planes, -1).reshape(-1).astype(np.uint8)).to(ctx.torch_device)
            layout = "hwc"
            orig = np.stack(planes)
        orig = orig.astype(np.float32) / np.float32(255)
        args = (cc["residue"], cc["motion"], refs, is_b, fmt, 8, fh.get_value("global_flow"),
                fh.get_value("warp_filter_size"))
        st = ctx.inter_stats(*args, source=src, layout=layout, want_maps=True)
        st2 = ctx.inter_stats(*args, source=src, layout=layout)
        assert st["sums"] == st2["sums"]
        res = cc["residue"][0].cpu().numpy()
        mot = cc["motion"][0].cpu().numpy()
        r444 = [_to444(r) for r in refs[:2 if is_b else 1]]
        probe = res.copy()
        probe[:3] = 0.0
        probe[3] = 0.5
        want_pred = oracle.inter_predict(probe, mot, r444[0], r444[1] if is_b else None, fh.get_value("global_flow"),
                                         fh.get_value("warp_filter_size"))
        pred = st["pred"].cpu().numpy()
        assert np.array_equal(pred, want_pred), (name, coding_idx)
        alpha = np.clip(res[3] + np.float32(0.5), 0, 1).astype(np.float32)
        beta = np.clip(res[4] + np.float32(0.5), 0, 1).astype(np.float32) if is_b else np.zeros_like(alpha)
        assert np.array_equal(st["alpha"].cpu().numpy(), alpha) and np.array_equal(st["beta"].cpu().numpy(), beta)
        dummy = (np.float32(0) + r444[0]) + (r444[1] if is_b else np.float32(0))
        dummy = (dummy / np.float32(2 if is_b else 1)).astype(np.float32)
        e, f = (pred - orig).astype(np.float32), (dummy - orig).astype(np.float32)
        want = [math.fsum(alpha.ravel().tolist()), math.fsum(beta.ravel().tolist()),
                math.fsum((e * e).astype(np.float32).ravel().tolist()), math.fsum((f * f).astype(np.float32).ravel().tolist())]
        for got, wt in zip(st["sums"], want):
            assert abs(got - wt) <= 1e-12 * max(abs(wt), 1e-300), (name, coding_idx, got, wt)
        # the reference's own fp32 torch formula (test.py:188-190) on this prediction
        ref_db = float(-10 * torch.log10(((torch.from_numpy(pred) - torch.from_numpy(orig)) ** 2).mean() + 1e-10))
        assert abs(check_pred_db(st["sums"][2], 3 * h * w) - ref_db) < 1e-3
    assert n_inter == len(seen) - 1


@pytest.mark.gpu
def test_launches(ctx, tmp_path, monkeypatch):
    """video_quality = decode_video_bytes' launches + one k_inter_stats per P / B frame + one k_frame_dist."""
    from coolchic_b200.bitstream.quality import video_quality

    name = "gop5_64x96_yuv420"
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, "yuv420", seed=3)
    h, w = srcs[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"g_{w}x{h}_yuv420_8b.yuv"
    _write_yuv(path, srcs)
    _decode_cpu(data, output_device="cuda")  # warm
    n0 = ctx.launch_count()
    _decode_cpu(data, output_device="cuda")
    n_decode = ctx.launch_count() - n0
    n0 = ctx.launch_count()
    q = video_quality(data, path)
    n_pb = sum(fq.frame_type != "I" for fq in q.values())
    assert n_pb == 4
    assert ctx.launch_count() - n0 == n_decode + n_pb + 1


@pytest.mark.gpu
def test_batch_one_launch(ctx):
    """2 x SM + 5 Kodak-size frames (mixed 8 / 10-bit, planar and HWC sources) in one k_frame_dist launch."""
    import torch

    from coolchic_b200.io.framedata import FrameData

    n = 2 * torch.cuda.get_device_properties(ctx.device).multi_processor_count + 5
    h, w = 512, 768
    g = torch.Generator(device=ctx.torch_device).manual_seed(5)
    frames, srcs, lays = [], [], []
    for i in range(n):
        b = 10 if i % 3 == 1 else 8
        M = 2**b - 1
        k = torch.randint(0, M + 1, (3, h, w), generator=g, device=ctx.torch_device, dtype=torch.int32)
        s = (k + torch.randint(-2, 3, (3, h, w), generator=g, device=ctx.torch_device, dtype=torch.int32)).clamp(0, M)
        frames.append(FrameData(b, "yuv444" if i % 2 else "rgb", (k.float() / M).view(1, 3, h, w)))
        if i % 2:
            srcs.append(s.reshape(-1).to(torch.uint8 if b == 8 else torch.int16))
            lays.append("planar")
        else:
            srcs.append(s.permute(1, 2, 0).reshape(-1).to(torch.uint8 if b == 8 else torch.int16))
            lays.append("hwc")
    n0 = ctx.launch_count()
    res = ctx.frame_distortion(frames, srcs, lays)
    assert ctx.launch_count() == n0 + 1
    for i in (0, 1, n // 2, n - 1):
        d = (frames[i].data[0] * (2**frames[i].bitdepth - 1)).round().long() - (
            srcs[i].view(3, h, w) if lays[i] == "planar" else srcs[i].view(h, w, 3).permute(2, 0, 1)).long()
        assert res[i]["sse"] == [int((d[c] ** 2).sum()) for c in range(3)]
        assert res[i]["max_abs"] == [int(d[c].abs().max()) for c in range(3)]


@pytest.mark.gpu
def test_off_grid_and_mismatch(ctx, tmp_path, monkeypatch):
    import torch

    from coolchic_b200._native import CcdError
    from coolchic_b200.bitstream.quality import video_quality
    from coolchic_b200.io.framedata import FrameData

    h, w = 8, 12
    y = torch.full((1, 1, h, w), 10 / 255, device=ctx.torch_device)
    u = torch.full((1, 1, h // 2, w // 2), 20 / 255, device=ctx.torch_device)
    v = u.clone()
    src = torch.zeros(h * w * 3 // 2, dtype=torch.uint8, device=ctx.torch_device)
    good = FrameData(8, "yuv420", {"y": y, "u": u, "v": v})
    u2 = u.clone()
    u2[0, 0, 1, 2] = 20.5 / 255
    v2 = v.clone()
    v2[0, 0, 3, 5] = 1.5
    off = FrameData(8, "yuv420", {"y": y, "u": u2, "v": v2})
    r = ctx.frame_distortion([good], [src], ["planar"])[0]
    assert r["sse"] == [100 * h * w, 400 * h * w // 4, 400 * h * w // 4]
    with pytest.raises(CcdError) as e:
        ctx.frame_distortion([good, off], [src, src], ["planar", "planar"])
    assert e.value.code == -1
    assert e.value.bad_index == [-1, h * w + 1 * (w // 2) + 2]

    name = "gop3_48x72_yuv420_bilinear"
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, "yuv420", seed=1)
    monkeypatch.chdir(tmp_path)
    n0 = ctx.launch_count()
    for bad_name, frames in [("a_72x48_yuv444_8b.yuv", srcs), ("a_72x48_yuv420_10b.yuv", srcs),
                             ("a_70x48_yuv420_8b.yuv", srcs), ("a_72x48_yuv420_8b.yuv", srcs[:2])]:
        _write_yuv(bad_name, frames, 8)
        with pytest.raises(ValueError):
            video_quality(data, bad_name)
    with pytest.raises(ValueError):
        video_quality(data, "a_72x48_yuv420_8b.yuv", frame_offset=1)
    assert ctx.launch_count() == n0


@pytest.mark.gpu
def test_cc_eval_cli(ctx, tmp_path, monkeypatch):
    name = "gop5_64x96_yuv420"
    srcs = _gop_sources(name, "yuv420", seed=9)
    h, w = srcs[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"g_{w}x{h}_yuv420_8b.yuv"
    _write_yuv(path, srcs)
    maps = "m.npz"
    out = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", os.path.join(GOLDEN, name + ".cool"),
                          "--original", path, "--maps", maps], capture_output=True, text=True, check=True).stdout
    lines = out.splitlines()
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    rows = lines[i + 1:i + 1 + len(srcs)]
    assert [r.split()[0] for r in rows] == [str(k) for k in range(len(srcs))]
    assert lines[i + 1 + len(srcs)].startswith("mean psnr_db")
    z = np.load(maps)
    assert z["frame0_error"].shape == (h, w) and z["frame1_pred"].shape == (3, h, w)
