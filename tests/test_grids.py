"""Latent-grid analysis (coolchic_b200.bitstream.grids, ccd_synthesize_many).

The variants are checked against the oracle: ccoracle.synthesize on the decoded latents with the masked grids set to
zero, then ccoracle.finish_frame (I frames) or ccoracle.inter_predict + finish_frame with the decoded frames as
references (P / B).  The PSNRs of video_grid_analysis are checked against a numpy SSE of those oracle frames, taken to
integers, and the source."""
import glob
import math
import os
import re
import subprocess
import sys
import time

import numpy as np
import pytest
from conftest import GOLDEN, ROOT

SINGLE = ["kodim14"] + sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(GOLDEN, "*.cool"))
                              if os.path.basename(p).startswith(("arch_", "img_")) and "_gop" not in p)
GOPS = sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(GOLDEN, "*.cool"))
              if os.path.basename(p).startswith(("gop", "arch_gop")))


def _parse(name):
    """(coding structure, per coding index: (frame header, {name: (header, nn bytes, latent bytes)}))."""
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream import decode
    from coolchic_b200.bitstream.header import VideoHeader

    buf = memoryview(open(os.path.join(GOLDEN, name + ".cool"), "rb").read())
    vh = VideoHeader()
    buf = vh.read_header(buf)
    cs = vh.get_coding_structure()
    frames = []
    for _ in range(cs.get_max_coding_order() + 1):
        fh, ccs, buf = decode._parse_frame(buf)
        frames.append((fh, {n: (h, bytes(nb), bytes(lb)) for n, (h, nb, lb) in ccs.items()}))
    return cs, frames


def _zeroed(oracle, desc, lat, mask):
    _, offs = oracle.latent_layout(desc)
    out = np.array(lat, dtype=np.int8, copy=True)
    for g in range(desc.n_grids):
        if (mask >> g) & 1:
            out[offs[g]:offs[g] + desc.grid_h[g] * desc.grid_w[g]] = 0
    return out


def _planes(x):
    """The three planes of a frame (numpy or torch, FrameData.data layout) as numpy float32."""
    if isinstance(x, dict):
        return [np.asarray(x[k].cpu() if hasattr(x[k], "cpu") else x[k]).reshape(x[k].shape[-2:]) for k in "yuv"]
    a = np.asarray(x.cpu() if hasattr(x, "cpu") else x)
    return [a.reshape(3, *a.shape[-2:])[c] for c in range(3)]


def _equal(got, want):
    return all(np.array_equal(g.view(np.uint32), w.view(np.uint32)) for g, w in zip(_planes(got), _planes(want)))


def _to444(fd):
    if fd.frame_data_type != "yuv420":
        return fd.data[0].cpu().numpy()
    up = [np.repeat(np.repeat(fd.data[c][0, 0].cpu().numpy(), 2, 0), 2, 1) for c in "uv"]
    return np.stack([fd.data["y"][0, 0].cpu().numpy()] + up)


def _oracle_frame(oracle, fh, ccs, refs, name=None, mask=0):
    """The oracle's finished frame with the grids of `mask` zeroed in Cool-chic `name`; ccs: {name: (desc, nn, lat)}."""
    raw = {n: oracle.synthesize(d, nn, _zeroed(oracle, d, lat, mask if n == name else 0)) for n, (d, nn, lat) in ccs.items()}
    b, fmt = fh.get_value("bitdepth"), fh.get_value("frame_data_type")
    if fh.get_value("frame_type") == "I":
        return oracle.finish_frame(raw["residue"], b, fmt)
    r444 = [_to444(r) for r in refs]
    x = oracle.inter_predict(raw["residue"], raw["motion"], r444[0], r444[1] if fh.get_value("frame_type") == "B" else None,
                             fh.get_value("global_flow"), fh.get_value("warp_filter_size"))
    return oracle.finish_frame(x, b, fmt)


def _psnr(sse, n, bitdepth):
    m2 = float(2**bitdepth - 1) ** 2
    db = lambda d: -10 * math.log10(max(d, 10 ** (-100 / 10)))  # noqa: E731  metrics/mse.py:18-21
    return db(sum(sse) / m2 / sum(n)), [db(s / m2 / k) for s, k in zip(sse, n)]


# ---- CPU ---------------------------------------------------------------------------------------------------------
def test_masks_every_golden_coolchic():
    from coolchic_b200._desc import desc_from_header
    from coolchic_b200.bitstream.grids import synthesis_masks

    n = 0
    for name in SINGLE + GOPS:
        for _, ccs in _parse(name)[1]:
            for h, _, _ in ccs.values():
                d = desc_from_header(h)
                hyper = sum(1 << g for g in range(d.n_grids) if d.grid_is_hyper[g])
                syn_grids = [g for g in range(d.n_grids) if not d.grid_is_hyper[g]]
                syn, drop, coarse = synthesis_masks(d)
                assert syn == syn_grids
                assert drop == [1 << g for g in syn_grids]
                assert len(coarse) == len(syn) - 1
                for k, m in enumerate(coarse, 1):
                    kept = [g for g in syn if not (m >> g) & 1]
                    assert kept == syn[-k:]
                assert all(m & hyper == 0 and m >> d.n_grids == 0 for m in drop + coarse)
                n += 1
    assert n > len(SINGLE)


def test_oracle_masked_grid_changes_output(oracle, kodim14):
    from coolchic_b200.bitstream.grids import synthesis_masks

    d = kodim14["desc"]
    nn = oracle.decode_nn(d, kodim14["nn_bytes"])
    lat = kodim14["latents"]
    full = oracle.synthesize(d, nn, lat)
    syn, drop, _ = synthesis_masks(d)
    assert len(syn) == 7
    for g, m in zip(syn, drop):
        assert not np.array_equal(oracle.synthesize(d, nn, _zeroed(oracle, d, lat, m)), full), g


# ---- GPU ---------------------------------------------------------------------------------------------------------
def _decoded(ctx, name):
    """Per coding index: (frame header, {name: (desc, nn ints, latents on the device)}, finish request of the residue)."""
    from coolchic_b200 import _native
    from coolchic_b200._desc import desc_from_header
    from coolchic_b200.bitstream import decode

    cs, frames = _parse(name)
    flat = [(i, n, desc_from_header(h), nb, lb) for i, (_, ccs) in enumerate(frames) for n, (h, nb, lb) in ccs.items()]
    _, lats = ctx.decode_many([f[2] for f in flat], [f[3] for f in flat], [f[4] for f in flat], want_latents=True)
    out = [(fh, {}, decode._finish_request(fh, {n: v for n, v in ccs.items()})) for fh, ccs in frames]
    for (i, n, d, nb, _), lat in zip(flat, lats):
        out[i][1][n] = (d, _native.decode_nn(d, nb), lat)
    return cs, out


@pytest.mark.gpu
@pytest.mark.parametrize("name", SINGLE)
def test_single_image_parity(ctx, oracle, name):
    """Every drop and coarse mask, raw and finished, against the oracle; mask 0 is the decode; latents are read only."""
    from coolchic_b200.bitstream.grids import synthesis_masks

    _, frames = _decoded(ctx, name)
    fh, ccs, fin = frames[0]
    d, nn, lat = ccs["residue"]
    _, nb, lb = _parse(name)[1][0][1]["residue"]
    before = lat.clone()
    lat_np = lat.cpu().numpy()
    _, drop, coarse = synthesis_masks(d)
    masks = [0] + drop + coarse
    n = len(masks)
    raw = ctx.synthesize([d] * n, [nn] * n, [lat] * n, masks)
    assert fin is not None
    done = ctx.synthesize([d] * n, [nn] * n, [lat] * n, masks, finish=[fin] * n)
    dec_raw, _ = ctx.decode_many([d], [nb], [lb])
    dec_fin, _ = ctx.decode_many([d], [nb], [lb], finish=[fin])
    assert np.array_equal(raw[0].cpu().numpy(), dec_raw[0].cpu().numpy())
    assert _equal(done[0], dec_fin[0])
    for m, r, f in zip(masks, raw, done):
        want = oracle.synthesize(d, nn, _zeroed(oracle, d, lat_np, m))
        assert np.array_equal(r[0].cpu().numpy(), want), (name, m)
        assert _equal(f, oracle.finish_frame(want, *fin)), (name, m)
    assert np.array_equal(lat.cpu().numpy(), before.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("name", GOPS)
def test_gop_variants(ctx, oracle, name):
    """Every drop mask of the motion and the residue, and every coarse mask of the residue, of every P / B frame:
    reconstructed with the decoded references, against the oracle's inter prediction of the oracle variant."""
    from coolchic_b200.bitstream import decode
    from coolchic_b200.bitstream.grids import synthesis_masks

    cs, frames = _decoded(ctx, name)
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    dec = decode.decode_video_bytes(data, output_device="cuda")
    n_checked = 0
    for c, (fh, ccs, _) in enumerate(frames):
        if fh.get_value("frame_type") == "I":
            continue
        refs = [dec[str(r)] for r in cs.get_frame_from_coding_order(c).index_references]
        np_ccs = {n: (d, nn, lat.cpu().numpy()) for n, (d, nn, lat) in ccs.items()}
        variants = []
        for n, (d, _, _) in ccs.items():
            _, drop, coarse = synthesis_masks(d)
            variants += [(n, m) for m in drop + (coarse if n == "residue" else [])]
        outs = ctx.synthesize([ccs[n][0] for n, _ in variants], [ccs[n][1] for n, _ in variants],
                              [ccs[n][2] for n, _ in variants], [m for _, m in variants])
        base = ctx.synthesize([ccs[n][0] for n in ccs], [ccs[n][1] for n in ccs], [ccs[n][2] for n in ccs], [0] * len(ccs))
        base = dict(zip(ccs, base))
        for (n, m), o in zip(variants, outs):
            cc = {**base, n: o}
            got = ctx.reconstruct_frame(cc["residue"], cc["motion"], refs, fh.get_value("frame_type") == "B",
                                        fh.get_value("frame_data_type"), fh.get_value("bitdepth"),
                                        fh.get_value("global_flow"), fh.get_value("warp_filter_size"))
            assert _equal(got, _oracle_frame(oracle, fh, np_ccs, refs, n, m)), (name, c, n, m)
            n_checked += 1
    assert n_checked > 0


def _launches(ctx, fn):
    """Kernels one fn() call launches, by the library's own count (after a warm-up call)."""
    import torch

    fn()
    torch.cuda.synchronize()
    n0 = ctx.launch_count()
    fn()
    torch.cuda.synchronize()
    return ctx.launch_count() - n0


def _variant_list(ctx, n):
    """n variants of mixed architectures: the single-image fixtures in turn, every other one with its frame tail, drop
    masks on two of three.  Returns (streams, descs, nn ints, latents, nn bytes, latent bytes, masks, finish)."""
    from coolchic_b200.bitstream.grids import synthesis_masks

    streams = []
    for name in SINGLE:
        _, frames = _decoded(ctx, name)
        _, ccs, fin = frames[0]
        _, nb, lb = _parse(name)[1][0][1]["residue"]
        streams.append((ccs["residue"], nb, lb, fin))
    jobs = [streams[i % len(streams)] for i in range(n)]
    drops = [synthesis_masks(j[0][0])[1] for j in jobs]
    return (streams, [j[0][0] for j in jobs], [j[0][1] for j in jobs], [j[0][2] for j in jobs], [j[1] for j in jobs],
            [j[2] for j in jobs], [d[i % len(d)] if i % 3 else 0 for i, d in enumerate(drops)],
            [j[3] if i % 2 else None for i, j in enumerate(jobs)])


def _traced():
    """Run in a fresh process (test_traced_kernels_and_copies): one variant of each fixture through synthesize and
    through decode_many, each in one torch.profiler session after a warm-up call, as test_gpu_staging._copies takes
    them.  Prints the kernel names of both, the synthesize call's copies each way and the launch counts of both."""
    import json

    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    ctx = _native.get_context(0)
    streams, descs, nns, lats, nbs, lbs, masks, fins = _variant_list(ctx, len(SINGLE))
    out = {}
    for key, fn in (("syn", lambda: ctx.synthesize(descs, nns, lats, masks, finish=fins)),
                    ("dec", lambda: ctx.decode_many(descs, nbs, lbs, finish=fins))):
        fn()
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            time.sleep(0.05)
            n0 = ctx.launch_count()
            fn()
            torch.cuda.synchronize()
            launches = ctx.launch_count() - n0
            time.sleep(0.05)
        names = [e.name for e in prof.events()]
        out[key] = {"kernels": sorted(m.group(0) for m in (re.search(r"\bk_\w+", n) for n in names
                                                           if not n.startswith(("Memcpy", "Memset"))) if m),
                    "launches": launches, "htod": sum(n.startswith("Memcpy HtoD") for n in names),
                    "dtoh": sum(n.startswith("Memcpy DtoH") for n in names)}
    print(json.dumps(out))


@pytest.mark.gpu
def test_traced_kernels_and_copies(ctx):
    """One variant of each fixture: the kernels of decoding them but the entropy launches, and one copy each way.  The
    trace is taken in a fresh process: in a process that has already run profiler sessions (this suite's other tests),
    later sessions were seen to miss records, up to 21 of 50 kernels."""
    import json

    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.join(ROOT, 'oracle')!r}, {ROOT!r}]; "
            "import test_grids; test_grids._traced()")
    out = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True, cwd=here).stdout
    r = json.loads(out.strip().splitlines()[-1])
    syn, dec = r["syn"], r["dec"]
    assert len(syn["kernels"]) == syn["launches"] and len(dec["kernels"]) == dec["launches"], "incomplete trace"
    assert (syn["htod"], syn["dtoh"]) == (1, 1)
    assert not any("k_entropy" in k for k in syn["kernels"])
    assert syn["kernels"] == [k for k in dec["kernels"] if "k_entropy" not in k]


@pytest.mark.gpu
def test_launches(ctx):
    """2 x SM + 5 variants of mixed architectures in one call: the launches of decoding them without the entropy
    launches, by the library's own count.  Alone, each stream's decode makes exactly one entropy launch more than its
    synthesis; together they make one entropy launch per ARM configuration, the same as one variant of each."""
    import torch

    n = 2 * torch.cuda.get_device_properties(ctx.device).multi_processor_count + 5
    streams, descs, nns, lats, nbs, lbs, masks, fins = _variant_list(ctx, n)
    k = len(streams)
    for i in range(k):
        n_syn = _launches(ctx, lambda: ctx.synthesize(descs[i:i + 1], nns[i:i + 1], lats[i:i + 1], masks[i:i + 1],
                                                      finish=fins[i:i + 1]))
        n_dec = _launches(ctx, lambda: ctx.decode_many(descs[i:i + 1], nbs[i:i + 1], lbs[i:i + 1], finish=fins[i:i + 1]))
        assert n_syn == n_dec - 1, SINGLE[i]
    n_entropy = (_launches(ctx, lambda: ctx.decode_many(descs[:k], nbs[:k], lbs[:k], finish=fins[:k]))
                 - _launches(ctx, lambda: ctx.synthesize(descs[:k], nns[:k], lats[:k], masks[:k], finish=fins[:k])))
    assert 1 <= n_entropy <= k
    n_syn = _launches(ctx, lambda: ctx.synthesize(descs, nns, lats, masks, finish=fins))
    n_dec = _launches(ctx, lambda: ctx.decode_many(descs, nbs, lbs, finish=fins))
    assert n_syn == n_dec - n_entropy

@pytest.mark.gpu
def test_errors(ctx):
    import ctypes

    from coolchic_b200 import _native
    from coolchic_b200._native import CcdError

    _, frames = _decoded(ctx, "kodim14")
    d, nn, lat = frames[0][1]["residue"]
    hyper = [g for g in range(d.n_grids) if d.grid_is_hyper[g]]
    assert hyper
    for mask in (1 << hyper[0], 1 << d.n_grids, 1 << 31):
        with pytest.raises(CcdError) as e:
            ctx.synthesize([d], [nn], [lat], [mask])
        assert e.value.code == -1 and "zero_grids" in str(e.value)
    out = ctx._empty_frame(d.img_h, d.img_w, "rgb")
    nn64 = np.ascontiguousarray(nn, dtype=np.int64)
    for lat_p, out_p in ((None, out.data_ptr()), (lat.data_ptr(), None)):
        job = _native.CcdSynthJob(desc=ctypes.pointer(d), nn_ints=nn64.ctypes.data, d_latents=lat_p, d_out=out_p)
        rc = ctx._lib.ccd_synthesize_many(ctx._h, ctypes.byref(job), 1, ctx._stream())
        with pytest.raises(CcdError) as e:
            _native._check(rc)
        assert e.value.code == -1 and "null" in str(e.value) and job.status == -1
    raw = ctx.synthesize([d], [nn], [lat], [0])[0]
    dec, _ = ctx.decode_many([d], [_parse("kodim14")[1][0][1]["residue"][1]], [_parse("kodim14")[1][0][1]["residue"][2]])
    assert np.array_equal(raw.cpu().numpy(), dec[0].cpu().numpy())


def _noisy(k, rng, amp=3):
    return np.clip(k.astype(np.int64) + rng.integers(-amp, amp + 1, size=k.shape), 0, 255)


def _ints(x, bitdepth):
    M = np.float32(2**bitdepth - 1)
    return [np.rint(p.astype(np.float32) * M).astype(np.int64) for p in _planes(x)]


def _check_analysis(ctx, oracle, name, data, path, src, counts=None):
    """Every drop / coarse PSNR of video_grid_analysis against the oracle variants, bits against video_rate."""
    from coolchic_b200.bitstream import decode
    from coolchic_b200.bitstream.grids import synthesis_masks, video_grid_analysis
    from coolchic_b200.bitstream.rate import video_rate

    res = video_grid_analysis(data, path)
    rates = video_rate(data)
    cs, frames = _decoded(ctx, name)
    dec = decode.decode_video_bytes(data, output_device="cuda")
    assert list(res) == list(rates) == [str(i) for i in range(len(frames))]
    for c, (fh, ccs, _) in enumerate(frames):
        f = cs.get_frame_from_coding_order(c)
        disp, b = f.display_order, fh.get_value("bitdepth")
        fg = res[str(disp)]
        refs = [dec[str(r)] for r in f.index_references]
        np_ccs = {n: (d, nn, lat.cpu().numpy()) for n, (d, nn, lat) in ccs.items()}
        n_samples = [x.size for x in src[disp]]

        def psnr(x):
            return _psnr([int(((a - s) ** 2).sum()) for a, s in zip(_ints(x, b), src[disp])], n_samples, b)

        base = psnr(_oracle_frame(oracle, fh, np_ccs, refs))
        assert abs(fg.psnr_db - base[0]) < 1e-9
        assert list(fg.coolchics) == list(ccs)
        for n, rows in fg.coolchics.items():
            d = ccs[n][0]
            syn, drop, coarse = synthesis_masks(d)
            assert [r.bits for r in rows] == rates[str(disp)].coolchics[n].grid_bits
            assert [r.bpp for r in rows] == rates[str(disp)].coolchics[n].grid_bpp
            for r in rows:
                assert r.size == (d.grid_h[r.grid], d.grid_w[r.grid]) and r.is_hyper == bool(d.grid_is_hyper[r.grid])
                if r.is_hyper:
                    assert r.drop_psnr_db is None and r.coarse_psnr_db is None
                    continue
                want, planes = psnr(_oracle_frame(oracle, fh, np_ccs, refs, n, 1 << r.grid))
                assert abs(r.drop_psnr_db - want) < 1e-9 and np.allclose(r.drop_psnr_planes_db, planes, rtol=0, atol=1e-9)
                assert abs(r.drop_delta_db - (want - base[0])) < 1e-9
                k = len(syn) - syn.index(r.grid)  # grids kept from the coarsest down to this one
                if n == "residue" and k < len(syn):
                    want, _ = psnr(_oracle_frame(oracle, fh, np_ccs, refs, n, coarse[k - 1]))
                    assert abs(r.coarse_psnr_db - want) < 1e-9
                else:
                    assert r.coarse_psnr_db is None
    return res


@pytest.mark.gpu
def test_analysis_kodim14(ctx, oracle, kodim14, tmp_path):
    from test_quality import _write_rgb

    from coolchic_b200.bitstream import decode

    dec = decode.decode_video_bytes(kodim14["data"])
    rng = np.random.default_rng(14)
    src = [_noisy(x, rng, amp=5) for x in _ints(dec["0"].data, 8)]
    path = str(tmp_path / "kodim14.png")
    _write_rgb(path, src)
    res = _check_analysis(ctx, oracle, "kodim14", kodim14["data"], path, [src])
    rows = res["0"].coolchics["residue"]
    assert sum(r.is_hyper for r in rows) == 3 and sum(r.coarse_psnr_db is not None for r in rows) == 6


@pytest.mark.gpu
def test_analysis_gop_and_cli(ctx, oracle, tmp_path, monkeypatch):
    """A 4:2:0 I-B-P GOP against a noisy YUV source; one synthesize and one distortion call per frame; the cc_eval.py
    --grids table."""
    from test_quality import _gop_sources, _write_yuv

    from coolchic_b200 import _native

    name = "gop3_48x72_yuv420_bilinear"
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, "yuv420", seed=11)
    h, w = srcs[0][0].shape
    monkeypatch.chdir(tmp_path)
    path = f"src_{w}x{h}_30p_yuv420_8b.yuv"
    _write_yuv(path, srcs)
    calls = {"synthesize": 0, "frame_distortion": 0}
    for fn in calls:
        orig = getattr(_native.Context, fn)

        def counted(self, *a, _fn=fn, _orig=orig, **k):
            calls[_fn] += 1
            return _orig(self, *a, **k)

        monkeypatch.setattr(_native.Context, fn, counted)
    res = _check_analysis(ctx, oracle, name, data, path, srcs)
    assert {res[k].frame_type for k in res} == {"I", "P", "B"}
    assert calls == {"synthesize": len(res), "frame_distortion": len(res)}
    monkeypatch.undo()

    def run(*extra):
        return subprocess.run([sys.executable, os.path.join(ROOT, "cc_eval.py"), "-i", os.path.join(GOLDEN, name + ".cool"),
                               "--original", os.path.join(tmp_path, path)] + list(extra), capture_output=True, text=True,
                              check=True, cwd=tmp_path).stdout.splitlines()

    plain, grids = run(), run("--grids")
    keep = lambda lines: [ln for ln in lines if not ln.startswith("Decoding frame")]  # noqa: E731  (timings)
    assert keep(grids)[:len(keep(plain))] == keep(plain)
    table = keep(grids)[len(keep(plain)):]
    n_tables = 0
    for i, ln in enumerate(table):
        if not ln.startswith("grids frame"):
            continue
        _, _, key, ftype, cc, _, psnr = ln.split()
        fg = res[key]
        assert ftype == fg.frame_type and abs(float(psnr) - fg.psnr_db) < 1e-6
        assert table[i + 1].split() == ["grid", "size", "hyper", "bits", "bpp", "drop_psnr_db", "drop_delta_db",
                                        "coarse_psnr_db"]
        rows = fg.coolchics[cc]
        for r, ln2 in zip(rows, table[i + 2:i + 2 + len(rows)]):
            v = ln2.split()
            assert int(v[0]) == r.grid and v[1] == f"{r.size[0]}x{r.size[1]}" and int(v[2]) == int(r.is_hyper)
            for s, x in zip(v[3:], (r.bits, r.bpp, r.drop_psnr_db, r.drop_delta_db, r.coarse_psnr_db)):
                assert (s == "n/a") if x is None else abs(float(s) - x) < 1e-6
        n_tables += 1
    assert n_tables == sum(len(fg.coolchics) for fg in res.values())
