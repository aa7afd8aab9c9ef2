"""Motion analysis (coolchic_b200.bitstream.motion, ccd_inter_analysis, DESIGN §4.9).

CPU: every variant of every P / B frame of the golden GOPs restated through the oracle (its inter prediction on the
variant's inputs, then its frame tail), from the reference's raw residue and motion with the reference-decoded frames
as references, against a seeded synthetic source; the host's PSNR / delta assembly against test_quality's checker; the
flow statistics of a float64 numpy restatement on crafted flows.

GPU: the kernel's SSE of every variant against ccd_frame_distortion of ccd_reconstruct_frame on the variant's inputs,
exactly; the flow statistics against the numpy restatement; repeatability, launches, the CLI and the refused calls."""
import ctypes
import math
import os
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from test_quality import _gop_sources, _write_yuv, check_psnr

GOPS = [("gop5_64x96_yuv420", "yuv420"), ("gop3_40x56_rgb", "rgb"), ("gop3_48x72_yuv420_bilinear", "yuv420"),
        ("gop3_40x56_rgb_bicubic", "rgb"), ("gop3_48x72_yuv420_sinc6", "yuv420"), ("gop4_40x56_rgb_sinc12", "rgb"),
        ("arch_gop3_7x9_sinc10", "rgb"), ("arch_gop3_7x9_sinc14", "rgb")]


# ---- checkers ----------------------------------------------------------------------------------------------------
def flow_stats(motion, global_flow, n_ref):
    """Per reference, the flow statistics of ccdec.h restated in float64 numpy: sums (math.fsum), max, outside count,
    and the fp32 flow map."""
    _, h, w = motion.shape
    gf = (list(global_flow) + [0, 0, 0, 0])[:4]
    ys, xs = np.mgrid[0:h, 0:w].astype(np.float64)
    out = []
    for r in range(n_ref):
        gx, gy = gf[2 * r], gf[2 * r + 1]
        fx, fy = motion[2 * r].astype(np.float64), motion[2 * r + 1].astype(np.float64)
        mag = np.sqrt(fx * fx + fy * fy)
        sx, sy = (xs + gx) + fx, (ys + gy) + fy
        outside = int(((sx < 0) | (sx > w - 1) | (sy < 0) | (sy > h - 1)).sum())
        flow = np.stack([motion[2 * r] + np.float32(gx), motion[2 * r + 1] + np.float32(gy)]).astype(np.float32)
        out.append({"sum": [math.fsum((fx + gx).ravel().tolist()), math.fsum((fy + gy).ravel().tolist()),
                            math.fsum(mag.ravel().tolist())], "max": float(mag.max()), "outside": outside, "flow": flow})
    return out


def _frame_sse(fin, src, fmt, bitdepth):
    """Per-plane SSE of a finished frame (oracle layout) against integer source planes."""
    M = 2**bitdepth - 1
    planes = [fin[k] for k in "yuv"] if fmt == "yuv420" else list(fin)
    return [int(((np.rint(p.astype(np.float32) * np.float32(M)).astype(np.int64) - s) ** 2).sum())
            for p, s in zip(planes, src)]


def _to444(fr):
    if not isinstance(fr, dict):
        return fr
    up = lambda p: np.repeat(np.repeat(p, 2, 0), 2, 1)  # noqa: E731
    return np.stack([fr["y"], up(fr["u"]), up(fr["v"])])


def _golden_inter_frames(name):
    """Per P / B frame in coding order: (frame header, residue, motion, reference frames) from the reference's raw
    outputs and decoded frames, and the golden frame it decodes to."""
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.header import CoolChicHeader, FrameHeader, VideoHeader

    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    gold = np.load(os.path.join(GOLDEN, name + "_frames.npz"))
    raw = np.load(os.path.join(GOLDEN, name + "_raw.npz"))
    v = VideoHeader()
    rest = v.read_header(data)
    out, i = [], 0
    for _ in range(v.get_coding_structure().get_max_coding_order() + 1):
        f = FrameHeader()
        rest = f.read_header(rest)
        ft, fmt, bd = f.get_value("frame_type"), f.get_value("frame_data_type"), f.get_value("bitdepth")
        for _ in range(1 if ft == "I" else 2):
            c = CoolChicHeader()
            rest = c.read_header(rest)
            rest = rest[c.get_value("nn_n_bytes") + c.get_value("n_bytes_latent"):]
        if ft == "I":
            i += 1
            continue
        M = 2**bd - 1

        def frame(idx):
            if fmt == "yuv420":
                return {k: gold[f"{idx}_{k}"].astype(np.float32) / np.float32(M) for k in "yuv"}
            return gold[str(idx)].astype(np.float32) / np.float32(M)

        refs = [_to444(frame(j)).astype(np.float32) for j in f.get_value("index_references")]
        out.append((f, raw[f"c{i}"], raw[f"c{i + 1}"], refs, frame(f.get_value("display_index"))))
        i += 2
    return out


# ---- CPU -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,fmt", GOPS)
def test_variants_through_oracle(oracle, name, fmt):
    """Each variant restated through the oracle; decoded reproduces the golden frame; the host's PSNR and deltas match
    the checker on those SSEs; a P frame has no beta variants."""
    from coolchic_b200.bitstream.motion import VARIANT_NAMES, motion_analysis, variant_inputs, variants_of

    srcs = _gop_sources(name, fmt, seed=11)
    n_pb = 0
    for f, residue, motion, refs, golden in _golden_inter_frames(name):
        n_pb += 1
        ft, bd = f.get_value("frame_type"), f.get_value("bitdepth")
        gf, fs = f.get_value("global_flow"), f.get_value("warp_filter_size")
        is_b = ft == "B"
        src = srcs[f.get_value("display_index")]
        sse = {}
        for v in VARIANT_NAMES:
            if v not in variants_of(ft):
                with pytest.raises(ValueError):
                    variant_inputs(residue, motion, gf, v)
                sse[v] = None
                continue
            r, m, g = variant_inputs(residue, motion, gf, v)
            fin = oracle.finish_frame(oracle.inter_predict(r, m, refs[0], refs[1] if is_b else None, g, fs), bd, fmt)
            if v == "decoded":
                M = 2**bd - 1
                for key in ("yuv" if fmt == "yuv420" else [None]):
                    a, b = (fin[key], golden[key]) if key else (fin, golden)
                    assert np.array_equal(np.rint(a * M), np.rint(b * M)), (name, ft, key)
            sse[v] = _frame_sse(fin, src, fmt, bd)
        assert (sse["ref0_only"] is None) == (not is_b) and (sse["ref1_only"] is None) == (not is_b)
        assert sse["no_prediction"] != sse["decoded"] and sse["no_motion"] != sse["decoded"]
        h, w = src[0].shape
        n = [x.size for x in src]
        fake = {"sse": [sse[v] for v in VARIANT_NAMES],
                "refs": [{"sum": [0.0, 0.0, 0.0], "max": 0.0, "outside": 0}] * (2 if is_b else 1)}
        ma = motion_analysis(fake, ft, bd, (h, w), fmt, gf)
        base, _ = check_psnr(sse["decoded"], n, bd)
        for v in VARIANT_NAMES:
            if sse[v] is None:
                assert ma.psnr_db(v) is None and ma.plane_psnr_db(v) is None and ma.delta_db(v) is None
                continue
            psnr, planes = check_psnr(sse[v], n, bd)
            assert abs(ma.psnr_db(v) - psnr) < 1e-9
            assert all(abs(a - b) < 1e-9 for a, b in zip(ma.plane_psnr_db(v), planes))
            assert abs(ma.delta_db(v) - (psnr - base)) < 1e-9
        assert ma.delta_db("decoded") == 0.0
    assert n_pb >= 2


def test_variant_inputs():
    """The input changes of the variant table, on numpy and torch inputs, without touching the originals."""
    import torch

    from coolchic_b200.bitstream.motion import VARIANT_NAMES, variant_inputs

    rng = np.random.default_rng(0)
    res, mot = rng.standard_normal((5, 3, 4)).astype(np.float32), rng.standard_normal((4, 3, 4)).astype(np.float32)
    gf = [1, -2, 3, 4]
    res0, mot0 = res.copy(), mot.copy()
    for v in VARIANT_NAMES:
        for r0, m0 in ((res, mot), (torch.from_numpy(res)[None], torch.from_numpy(mot)[None])):
            r, m, g = variant_inputs(r0, m0, gf, v)
            r, m = np.asarray(r).reshape(5, 3, 4), np.asarray(m).reshape(4, 3, 4)
            want_r, want_m, want_g = res.copy(), mot.copy(), gf
            if v in ("no_local_motion", "no_motion"):
                want_m[:] = 0
            if v == "no_motion":
                want_g = [0, 0, 0, 0]
            if v in ("ref0_only", "ref1_only"):
                want_r[4] = 0.5 if v == "ref0_only" else -0.5
            if v == "no_residue":
                want_r[:3] = 0
            if v == "no_prediction":
                want_r[3] = -0.5
            assert np.array_equal(r, want_r) and np.array_equal(m, want_m) and g == want_g, v
    assert np.array_equal(res, res0) and np.array_equal(mot, mot0) and gf == [1, -2, 3, 4]
    with pytest.raises(ValueError):
        variant_inputs(res[:4], mot[:2], gf[:2], "ref1_only")
    with pytest.raises(ValueError):
        variant_inputs(res, mot, gf, "nothing")


def test_flow_stats_restatement():
    """The float64 restatement on crafted flows: borders inclusive, the global shift counted, sums and max exact."""
    from coolchic_b200.bitstream.motion import motion_analysis

    h, w = 4, 6
    mot = np.zeros((4, h, w), np.float32)
    mot[0, 0, 0] = -0.25          # x + gx + fx = -0.25 + 0: outside
    mot[1, 3, 5] = 0.0
    mot[0, 1, 2], mot[1, 1, 2] = 3.0, 4.0   # |local| 5
    st = flow_stats(mot, [0, 0, 1, -1], 2)
    assert st[0]["outside"] == 1 + 1  # (0, 0) and (2, 1) + (3, 4) = (5, 5): y = 5 > 3
    assert st[0]["max"] == 5.0 and st[0]["sum"] == [-0.25 + 3.0, 4.0, 0.25 + 5.0]
    # reference 1: zero local flow shifted by (1, -1): the last column and the first row fall outside
    assert st[1]["outside"] == h + w - 1 and st[1]["max"] == 0.0 and st[1]["sum"] == [h * w, -h * w, 0.0]
    assert np.array_equal(st[1]["flow"], np.stack([np.ones((h, w)), -np.ones((h, w))]).astype(np.float32))
    # the exact border: x + gx + fx == w - 1 is inside
    edge = np.zeros((2, h, w), np.float32)
    edge[0] = 0.5
    assert flow_stats(edge, [0, 0], 1)[0]["outside"] == h
    edge[0] = 0.0
    assert flow_stats(edge, [0, 0], 1)[0]["outside"] == 0
    res = {"sse": [[1, 2, 3]] * 7, "refs": st}
    ma = motion_analysis(res, "B", 8, (h, w), "rgb", [0, 0, 1, -1])
    assert ma.refs[1].global_flow == (1, -1) and ma.refs[1].mean_flow == (1.0, -1.0)
    assert ma.refs[0].mean_local == (0.25 + 5.0) / (h * w) and ma.refs[0].outside_fraction == 2 / (h * w)


# ---- GPU -----------------------------------------------------------------------------------------------------------
def _device_inter_frames(ctx, data):
    """(frame header, raw residue / motion, references on the device) of every P / B frame of a decode, coding order."""
    from coolchic_b200.bitstream import decode

    seen = []

    def recon(fh, cc_out, refs, dev):
        if fh.get_value("frame_type") != "I":
            seen.append((fh, dict(cc_out), [r.to(ctx.torch_device) for r in refs]))
        return decode._reconstruct(fh, cc_out, refs, dev)

    decode.decode_video_bytes(data, output_device="cuda", reconstruct_fn=recon)
    return seen


def _source_tensor(ctx, planes, fmt, bitdepth=8):
    import torch

    dt = np.uint8 if bitdepth <= 8 else np.int16
    if fmt == "yuv420":
        return torch.from_numpy(np.concatenate([p.reshape(-1) for p in planes]).astype(dt)).to(ctx.torch_device), "planar"
    return torch.from_numpy(np.stack(planes, -1).reshape(-1).astype(dt)).to(ctx.torch_device), "hwc"


def check_frame(ctx, fh, cc, refs, src, layout, global_flow):
    """The kernel on one frame against reconstruct + frame_distortion per variant, and against the restated
    statistics; a second call bit-identical.  Returns the analysis."""
    import torch

    from coolchic_b200.bitstream.motion import VARIANT_NAMES, variant_inputs, variants_of
    from coolchic_b200.io.framedata import FrameData

    ft, fmt, bd = fh.get_value("frame_type"), fh.get_value("frame_data_type"), fh.get_value("bitdepth")
    fs = fh.get_value("warp_filter_size")
    is_b = ft == "B"
    args = (cc["residue"], cc["motion"], refs, is_b, fmt, bd, global_flow, fs)
    n0 = ctx.launch_count()
    a = ctx.inter_analysis(*args, source=src, layout=layout, want_maps=True)
    assert ctx.launch_count() == n0 + 1
    b = ctx.inter_analysis(*args, source=src, layout=layout)
    assert a["sse"] == b["sse"]
    for ra, rb in zip(a["refs"], b["refs"]):
        assert (ra["sum"], ra["max"], ra["outside"]) == (rb["sum"], rb["max"], rb["outside"])
    for k, v in enumerate(VARIANT_NAMES):
        if v not in variants_of(ft):
            assert a["sse"][k] is None
            continue
        r, m, g = variant_inputs(cc["residue"], cc["motion"], global_flow, v)
        fin = ctx.reconstruct_frame(r, m, refs, is_b, fmt, bd, g, fs)
        want = ctx.frame_distortion([FrameData(bd, fmt, fin)], [src], [layout])[0]["sse"]
        assert a["sse"][k] == want, (v, a["sse"][k], want)
    mot = cc["motion"][0].cpu().numpy()
    st = flow_stats(mot, global_flow, 2 if is_b else 1)
    assert len(a["refs"]) == len(st)
    for got, want in zip(a["refs"], st):
        for x, y in zip(got["sum"], want["sum"]):
            assert abs(x - y) <= 1e-12 * max(abs(y), 1e-300), (x, y)
        assert got["max"] == want["max"] and got["outside"] == want["outside"]
        assert torch.equal(got["flow"].cpu(), torch.from_numpy(want["flow"]))
    return a


@pytest.mark.gpu
@pytest.mark.parametrize("crafted", [False, True])
@pytest.mark.parametrize("name,fmt", GOPS)
def test_kernel_vs_reconstruction(ctx, name, fmt, crafted):
    """Every P / B frame of the fixture, with its own global flow and then with a crafted one per reference (passed to
    the kernel and to the reconstructions alike)."""
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, fmt, seed=5)
    frames = _device_inter_frames(ctx, data)
    assert frames
    for fh, cc, refs in frames:
        h, w = cc["residue"].shape[-2:]
        gf = fh.get_value("global_flow")
        if crafted:  # shifts that reach past the border, different per reference
            gf = [w // 3 + 1, -(h // 4) - 1, -(w // 2), h // 3 + 2][:len(gf)]
        src, layout = _source_tensor(ctx, srcs[fh.get_value("display_index")], fmt)
        check_frame(ctx, fh, cc, refs, src, layout, gf)


@pytest.mark.gpu
def test_1080p_b_frame_sinc14(ctx, seed_stream):
    """A synthetic 1080p 4:2:0 B frame at sinc-14 (source: the decoded frame with seeded noise), checked the same way."""
    import torch

    from coolchic_b200 import synth

    data = synth.make_video_stream(ctx, seed_stream, 1080, 1920, 3, "yuv420", 8, 14, seed=3)
    frames = _device_inter_frames(ctx, data)
    b = [f for f in frames if f[0].get_value("frame_type") == "B"]
    assert len(b) == 1
    fh, cc, refs = b[0]
    fin = ctx.reconstruct_frame(cc["residue"], cc["motion"], refs, True, "yuv420", 8, fh.get_value("global_flow"), 14)
    g = torch.Generator(device=ctx.torch_device).manual_seed(14)
    parts = []
    for k in "yuv":
        x = (fin[k].reshape(-1) * 255).round().to(torch.int32)
        parts.append((x + torch.randint(-4, 5, x.shape, generator=g, device=x.device, dtype=torch.int32)).clamp(0, 255))
    src = torch.cat(parts).to(torch.uint8)
    a = check_frame(ctx, fh, cc, refs, src, "planar", fh.get_value("global_flow"))
    assert a["sse"][0] != a["sse"][6]


@pytest.mark.gpu
@pytest.mark.parametrize("name", [g[0] for g in GOPS if g[1] == "yuv420"])
def test_video_quality_motion(ctx, name, tmp_path, monkeypatch):
    """video_quality(motion=True): decoded SSE = the frame's own SSE, one extra launch per P / B frame, I frames None,
    everything else as without motion."""
    from coolchic_b200.bitstream.quality import video_quality

    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, "yuv420", seed=len(name) + 1)
    h, w = srcs[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"src_{w}x{h}_30p_yuv420_8b.yuv"
    _write_yuv(path, srcs)
    video_quality(data, path)  # warm
    n0 = ctx.launch_count()
    plain = video_quality(data, path)
    n_plain = ctx.launch_count() - n0
    n0 = ctx.launch_count()
    q = video_quality(data, path, motion=True, want_maps=True)
    n_motion = ctx.launch_count() - n0
    n_pb = 0
    for k, fq in q.items():
        assert fq.sse == plain[k].sse and fq.pred_psnr_db == plain[k].pred_psnr_db
        if fq.frame_type == "I":
            assert fq.motion is None
            continue
        n_pb += 1
        m = fq.motion
        assert m.sse["decoded"] == fq.sse and abs(m.psnr_db("decoded") - fq.psnr_db) < 1e-12
        assert len(m.refs) == (2 if fq.frame_type == "B" else 1)
        assert all(r.flow_map.shape == (2, h, w) for r in m.refs)
    assert n_pb >= 2 and n_motion == n_plain + n_pb


@pytest.mark.gpu
def test_cc_eval_motion_cli(ctx, tmp_path, monkeypatch):
    name = "gop5_64x96_yuv420"
    srcs = _gop_sources(name, "yuv420", seed=9)
    h, w = srcs[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"g_{w}x{h}_yuv420_8b.yuv"
    _write_yuv(path, srcs)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", os.path.join(GOLDEN, name + ".cool"),
                          "--original", path, "--motion", "--maps", "m.npz"], capture_output=True, text=True,
                         check=True).stdout
    lines = out.splitlines()
    i = next(k for k, ln in enumerate(lines) if ln.startswith("frame_idx"))
    types = {ln.split()[0]: ln.split()[1] for ln in lines[i + 1:i + 1 + len(srcs)]}
    inter = [k for k, t in types.items() if t != "I"]
    assert len(inter) == 4
    z = np.load("m.npz")
    for k in inter:
        j = lines.index(next(ln for ln in lines if ln.startswith(f"motion frame {k} ")))
        assert lines[j + 1].split() == ["variant", "psnr_db", "psnr_y_db", "psnr_u_db", "psnr_v_db", "delta_db"]
        n_var = 7 if types[k] == "B" else 5
        rows = lines[j + 2:j + 2 + n_var]
        assert rows[0].split()[0] == "decoded" and float(rows[0].split()[-1]) == 0.0
        assert all(len(r.split()) == 6 for r in rows)
        n_ref = 2 if types[k] == "B" else 1
        assert [ln.split()[0] for ln in lines[j + 2 + n_var:j + 2 + n_var + n_ref]] == [f"ref{r}" for r in range(n_ref)]
        assert all(z[f"frame{k}_flow{r}"].shape == (2, h, w) for r in range(n_ref))
    assert not any(ln.startswith("motion frame 0 ") for ln in lines)


@pytest.mark.gpu
def test_refused_calls(ctx):
    """Bad calls are refused before any launch, with the codes of ccd_reconstruct_frame and ccd_inter_stats; a
    non-finite flow is an argument error naming its pixel."""
    import torch

    from coolchic_b200._native import CcdError, CcdInterAnalysis
    from coolchic_b200.io.framedata import FrameData

    dev = ctx.torch_device
    h, w = 8, 12
    ref = FrameData(8, "yuv420", {"y": torch.zeros((1, 1, h, w), device=dev), "u": torch.zeros((1, 1, h // 2, w // 2), device=dev),
                                  "v": torch.zeros((1, 1, h // 2, w // 2), device=dev)})
    res = torch.zeros((1, 5, h, w), device=dev)
    mot = torch.zeros((1, 4, h, w), device=dev)
    src = torch.zeros(h * w * 3 // 2, dtype=torch.uint8, device=dev)

    def call(mutate, layout=0):
        f, keep, _, _ = ctx._inter_frame(res, mot, [ref, ref], True, "yuv420", 8, [0, 0, 0, 0], 8)
        mutate(f)
        an = CcdInterAnalysis(d_src=src.data_ptr(), src_layout=layout)
        rc = ctx._lib.ccd_inter_analysis(ctx._h, ctypes.byref(f), ctypes.byref(an), ctx._stream())
        torch.cuda.synchronize()
        return rc, an

    n0 = ctx.launch_count()
    assert call(lambda f: None)[0] == 0
    assert ctx.launch_count() == n0 + 1
    n0 = ctx.launch_count()
    assert call(lambda f: setattr(f, "n_res_ch", 4))[0] == -1
    assert call(lambda f: setattr(f, "n_mot_ch", 2))[0] == -1
    assert call(lambda f: None, layout=1)[0] == -1  # HWC source of a 4:2:0 frame
    assert call(lambda f: setattr(f, "bitdepth", 0))[0] == -1

    def tiny(fs):
        def m(f):
            f.h, f.w, f.frame_data_type, f.warp_filter_size = 1, 1, 0, fs
        return m

    assert call(tiny(2))[0] == -4 and call(tiny(4))[0] == -4
    assert ctx.launch_count() == n0
    mot[0, 3, 2, 5] = float("nan")
    mot[0, 0, 6, 1] = float("inf")
    with pytest.raises(CcdError) as e:
        ctx.inter_analysis(res, mot, [ref, ref], True, "yuv420", 8, [0, 0, 0, 0], 8, source=src)
    assert e.value.code == -1 and e.value.bad_index == [2 * w + 5]
