"""The decoder on networks with every weight live.

synth.adapt_nn copies the sample stream's network (7 grids, a 48-wide synthesis with 3 outputs, a 14 + 6 ARM) into a
target architecture and pads the rest with zeros: residue channels 3 / 4 (alpha, beta), the second flow of a B frame,
synthesis units past 48, latent grids past the seventh and ARM units past 14 + 6 only ever met zero weights.  Here
synth.liven_nn fills them (make_coolchic(live=...)), and the reference fixtures of oracle/gen_golden_dense.py pin the
result to the unmodified reference.  Five deliberate bugs of the float64 restatement (test_reference64.py) and of the
numpy DMMA ARM (test_arm_f64.py) pass on every older fixture and fail on the new ones."""
import glob
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from test_arm_f64 import FAST_SHAPES, _blob_bytes, arm_ints, contexts, eval_f64, eval_int64, fits_f64, pack
from test_rate import _check_against_checker, _coolchics, model_indices
from test_reference64 import REF_FIXTURES, assert_within, cpu_seed, intra, reference_fixture  # noqa: F401

DENSE = ["img_64x96_rgb_vhop_dense", "img_96x128_rgb_12grids_dense", "gop3_40x56_rgb_sinc8_dense",
         "gop3_48x72_yuv420_bicubic_dense"]


def _syn(*layers, **fields):
    ov = {"n_layer_synthesis": len(layers), **{f"syn_layer_{i}": lay for i, lay in enumerate(layers)}}
    ov.update(fields)
    return ov


def _arm(n_ctx, hidden, cf, ifce_res=(0, 2)):
    return {"spatial_context_arm": n_ctx, "n_hidden_layers_arm": hidden, "output_feature_ifce": cf,
            "ifce_resolution": list(ifce_res) if cf else None}


# id -> (size, latent_resolution, header overrides, kind of Cool-chic, final upsampling, seed)
# the float tail matrix: k_tail_syn<CINP, C> for CINP 4 / 8 / 16 (2, 4, 7, 12 and 16 grids; 2 grids: the int8 stack)
# x C 2 ... 5, 0 / 1 / 2 residual 3x3 layers, hidden widths 8 ... 127, widths that take TMA staging (a multiple of 16)
# and plain loads, sizes that are not multiples of the 32 x 16 tile
HIDS = (8, 16, 48, 64, 127)
SIZES = ((37, 45), (48, 64), (33, 100))
TAIL = {}
for _i, (_lat, _C) in enumerate([(lat, C) for lat in ((0, 1), (0, 3), (0, 6), (0, 11), (0, 15)) for C in (2, 3, 4, 5)]):
    _n3, _hid, _size = _i % 3, HIDS[_i % 5], SIZES[(_i + _i // 4) % 3]
    _layers = [f"{_hid}-1-linear-relu", f"{_C}-1-linear-none"] + [
        f"{_C}-3-residual-{'relu' if _l < _n3 - 1 else 'none'}" for _l in range(_n3)]
    _kind = "motion" if _C == 2 or (_C == 4 and _i % 2) else ("intra" if _C == 3 else "residue")
    TAIL[f"nl{_lat[1] + 1}_C{_C}_n3{_n3}_hid{_hid}_{_size[0]}x{_size[1]}"] = (_size, _lat, _syn(*_layers), _kind, None,
                                                                              20 + _i)
# k_syn_fused through the per-stream path (upsampling kernel sizes 6 / 5)
FUSED = {
    "ups65_C3_hid48": ((37, 61), (0, 3), {"ups_k_size": 6, "ups_preconcat_k_size": 5}, "intra", None, 41),
    "ups65_C5_n3_1_hid64": ((40, 56), (0, 4), _syn("64-1-linear-relu", "5-1-linear-none", "5-3-residual-relu",
                                                   ups_k_size=6, ups_preconcat_k_size=5), "residue", None, 42),
}
# the reference's decoder presets (cfg/dec), every weight live
PRESETS = {
    "intra_lop": ((40, 56), (0, 6), {**_arm(6, 2, 2), **_syn("8-1-linear-relu", "3-1-linear-none",
                                                             "3-3-residual-none")}, "intra", None, 51),
    "intra_mop": ((40, 56), (0, 6), {**_arm(10, 2, 4), **_syn("16-1-linear-relu", "3-1-linear-none", "3-3-residual-relu",
                                                              "3-3-residual-none")}, "intra", None, 52),
    "intra_hop": ((40, 56), (0, 6), {**_arm(14, 2, 6), **_syn("48-1-linear-relu", "3-1-linear-none", "3-3-residual-relu",
                                                              "3-3-residual-none")}, "intra", None, 53),
    "intra_vhop": ((40, 56), (0, 6), {**_arm(20, 2, 6), **_syn("64-1-linear-relu", "3-1-linear-none",
                                                               "3-3-residual-relu", "3-3-residual-none")}, "intra", None,
                   54),
}
for _C in (4, 5):
    for _name, _a, _hid in (("vlop", (6, 1, 0), 8), ("lop", (6, 2, 0), 16), ("mop", (10, 2, 2), 16),
                            ("hop", (10, 2, 4), 48)):
        PRESETS[f"residue_{_name}_C{_C}"] = ((48, 72), (0, 6), {**_arm(*_a), **_syn(
            f"{_hid}-1-linear-relu", f"{_C}-1-linear-none", f"{_C}-3-residual-none")}, "residue", None, 60 + _C + _hid)
for _C in (2, 4):
    PRESETS[f"motion_lop_C{_C}"] = ((44, 60), (2, 6), {**_arm(6, 1, 0), **_syn("8-1-linear-relu", f"{_C}-1-linear-none")},
                                    "motion", "nearest", 70 + _C)
    PRESETS[f"motion_mop_C{_C}"] = ((44, 60), (2, 6), {**_arm(6, 2, 2, (2, 2)), **_syn("16-1-linear-relu",
                                                                                       f"{_C}-1-linear-none")},
                                    "motion", "nearest", 80 + _C)
ALL = {**TAIL, **FUSED, **PRESETS}


def live_stream(backend, ss, case, live=True):
    """(header, desc, nn ints, nn bytes, latent bytes, latents) of one fabricated Cool-chic."""
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    size, lat, ov, kind, fin, seed = case
    cc, h, lat_t = synth.make_coolchic(backend, ss, size, lat, None, seed=seed, final_upsampling_type=fin,
                                       overrides=dict(ov), live=kind if live else None)
    h2 = type(h)()
    rest = h2.read_header(cc)
    d = desc_from_header(h2)
    n_nn, n_lat = h2.get_value("nn_n_bytes"), h2.get_value("n_bytes_latent")
    nb, lb = bytes(rest[:n_nn]), bytes(rest[n_nn:n_nn + n_lat])
    return h2, d, backend.decode_nn(d, nb), nb, lb, lat_t.cpu().numpy()


def _dead(d, nn):
    from coolchic_b200 import synth

    sec = synth.split_nn(d, nn)
    dead = []
    for key in ("arm.weight", "synthesis.weight"):
        for name, w in sec[key].items():
            w2 = np.abs(w).reshape(w.shape[0], w.shape[1], -1).sum(axis=2)
            dead += [(f"{key}.{name}", "row", int(r)) for r in np.flatnonzero(w2.sum(axis=1) == 0)]
            dead += [(f"{key}.{name}", "col", int(c)) for c in np.flatnonzero(w2.sum(axis=0) == 0)]
    return dead


def dead_parts(d, nn, ss):
    """Every synthesis and ARM weight tensor's output rows and input columns (the hidden units and inputs) with no
    nonzero weight, but those the sample stream ``ss`` itself has at zero: [(tensor, 'row' | 'col', index)]."""
    own = set(_dead(ss.desc, ss.nn))
    return [p for p in _dead(d, nn) if p not in own]


_LIVE_CACHE = {}


def _cpu_live(cpu_seed, name):  # noqa: F811
    if name not in _LIVE_CACHE:
        _LIVE_CACHE[name] = live_stream(*cpu_seed, ALL[name])
    return _LIVE_CACHE[name]


# ------------------------------------------------------------------------------------------------------------------
# CPU: liveness, the oracle against the restatement, the reference fixtures, the negative controls, the ARM bound
@pytest.mark.parametrize("name", list(ALL))
def test_every_weight_is_live(oracle, cpu_seed, name):  # noqa: F811
    h, d, nn, _, _, lat = _cpu_live(cpu_seed, name)
    assert dead_parts(d, nn, cpu_seed[1]) == [], name
    raw = oracle.synthesize(d, nn, lat)
    assert all(float(raw[c].std()) > 0 for c in range(raw.shape[0])), name
    kind = ALL[name][3]
    if kind == "residue":  # alpha / beta below 0, inside (0, 1) and above 1
        for c in range(3, raw.shape[0]):
            a = raw[c] + 0.5
            assert (a < 0).any() and ((a > 0) & (a < 1)).any() and (a > 1).any(), (name, c)
    if kind == "motion":  # flows of a few pixels, with fractions
        p5, p95 = np.percentile(raw, [5, 95])
        assert -5 < p5 < -1 and 1 < p95 < 5 and (raw != np.round(raw)).mean() > 0.9, name
    # the ARM keeps the fast layout: arm_fits_f64, and the library plans the fast blob
    from coolchic_b200 import _native

    cf = d.n_ifce_out if d.flag_ifce else 0
    a = arm_ints(d, nn)
    if (d.n_ctx, cf) in FAST_SHAPES and a["feat_bound"] is not None:  # (an IFCE of many grids is never fast)
        assert fits_f64(a), name
        # the same network with one stabiliser weight past the bound plans the generic blob, larger by exactly the
        # difference of the two layouts
        from coolchic_b200 import synth

        t = synth.split_nn(d, nn.copy())
        t["arm.weight"]["stab"][0, 0] = 2**40
        big, _ = synth.join_nn(d, t)
        assert not fits_f64(arm_ints(d, big))
        p_fast, p_gen = _native.entropy_plan(d, nn), _native.entropy_plan(d, big)
        base = [s - r * (16 + 32 * 4 + 16 + 4) - w * 64 for r, w, s in (p_fast, p_gen)]
        assert base[1] - base[0] == _blob_bytes(d, False) - _blob_bytes(d, True), name


def test_adapt_nn_alone_leaves_dead_weights(cpu_seed):  # noqa: F811
    """Without liven_nn, every architecture beyond the sample keeps whole rows and columns at zero: the gap this file
    closes."""
    names = ["intra_vhop", "residue_hop_C5", "motion_mop_C4", next(n for n in TAIL if n.startswith("nl12")),
             next(n for n in TAIL if "hid127" in n)]
    for name in names:
        _, d, nn, _, _, _ = live_stream(*cpu_seed, ALL[name], live=False)
        dead = dead_parts(d, nn, cpu_seed[1])
        print(f"{name} through adapt_nn alone: {len(dead)} dead rows / columns")
        assert dead, name


@pytest.mark.parametrize("name", list(ALL))
def test_oracle_vs_restatement(oracle, cpu_seed, name):  # noqa: F811
    h, d, nn, _, _, lat = _cpu_live(cpu_seed, name)
    assert_within(oracle.synthesize(d, nn, lat), intra(h, nn, lat), f"{name} oracle raw")


@pytest.mark.parametrize("name", DENSE)
def test_dense_fixtures_vs_restatement(oracle, name):
    # alpha and beta vary: the a-priori bound of a prediction puts too many samples near a tie, so the window is the
    # oracle's measured error, as above 10 bits
    reference_fixture(oracle, name, measured_window=True)


@pytest.mark.parametrize("name", DENSE)
def test_dense_fixtures_are_live(oracle, cpu_seed, name):  # noqa: F811
    """Every Cool-chic of the committed fixtures has no dead row or column, and varying outputs (alpha / beta and
    both flows of the B frame included)."""
    from coolchic_b200._desc import desc_from_header

    raw = np.load(os.path.join(GOLDEN, name + "_raw.npz"))
    for i, (h, nb, _) in enumerate(_coolchics(open(os.path.join(GOLDEN, name + ".cool"), "rb").read())):
        d = desc_from_header(h)
        assert dead_parts(d, oracle.decode_nn(d, bytes(nb)), cpu_seed[1]) == [], (name, i)
        r = raw[f"c{i}"]
        assert all(float(r[c].std()) > 0 for c in range(r.shape[0])), (name, i)
        if r.shape[0] == 5 and d.latent_res_lo == 0:  # a B residue: alpha and beta differ, neither is 0.5
            a, b = np.clip(r[3] + 0.5, 0, 1), np.clip(r[4] + 0.5, 0, 1)
            assert np.abs(a - b).mean() > 0.1 and abs(a.mean() - 0.5) + abs(b.mean() - 0.5) > 0.01, (name, i)


# each bug of the restatement: passes on every older reference fixture, fails on the dense ones listed
LIVE_CONTROLS = {
    "swap_ab": ["gop3_40x56_rgb_sinc8_dense", "gop3_48x72_yuv420_bicubic_dense"],
    "drop_flow1_y": ["gop3_40x56_rgb_sinc8_dense", "gop3_48x72_yuv420_bicubic_dense"],
    "drop_grids7": ["img_96x128_rgb_12grids_dense"],
    "drop_hidden48": ["img_64x96_rgb_vhop_dense"],
}


@pytest.mark.parametrize("bug", list(LIVE_CONTROLS))
def test_negative_controls_pass_the_old_fixtures_and_fail_the_dense_ones(oracle, bug):
    for name in REF_FIXTURES:
        r = reference_fixture(oracle, name, bug)
        assert r <= 1.0, f"negative control {bug} fails on the older {name} ({r:.3g})"
    print(f"negative control {bug}: passes on all {len(REF_FIXTURES)} older reference fixtures")
    for name in LIVE_CONTROLS[bug]:
        fired = []
        r = reference_fixture(oracle, name, bug, measured_window=True, failures=fired)
        print(f"negative control {bug} on the reference's {name}: max |err| / bound = {r:.3g}; " +
              ("; ".join(fired) or "every frame's levels within the tie windows"))
        assert r > 1.0, f"negative control {bug} passes against the reference's {name}"
        # what rejects the bug is the reference's own integer samples, off a rounding tie of the un-bugged value
        assert any("off a tie differ" in m for m in fired), (bug, name, fired)
    print(f"negative control {bug}: detected by the dense fixtures")


def _golden_arms(dense):
    from coolchic_b200._desc import desc_from_header

    for path in sorted(glob.glob(os.path.join(GOLDEN, "*.cool"))):
        if path.endswith("_dense.cool") != dense:
            continue
        for k, (h, nb, _) in enumerate(_coolchics(open(path, "rb").read())):
            d = desc_from_header(h)
            from coolchic_b200 import _native

            yield f"{os.path.basename(path)}#{k}", d, _native.decode_nn(d, bytes(nb))


def test_arm_negative_control_tile3(cpu_seed):  # noqa: F811
    """The fourth n-tile of the DMMA ARM (units 24 ... 31, only the 20 + 6 shape has it) packed with a wrong column
    permutation: equal to the int64 ARM on every older golden ARM, different on the dense 20 + 6 ones."""
    rng = np.random.default_rng(5)
    n_old = 0
    for label, d, nn in _golden_arms(False):
        a = arm_ints(d, nn)
        cf = d.n_ifce_out if d.flag_ifce else 0
        if (d.n_ctx, cf) not in FAST_SHAPES or a["feat_bound"] is None:
            continue
        X = contexts(a, rng, 1024)
        got, want = eval_f64(a, pack(a, "tile3_perm"), X), eval_int64(a, X)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), label
        n_old += 1
    print(f"negative control tile3_perm: passes on {n_old} older golden ARMs")
    n_new = 0
    for label, d, nn in _golden_arms(True):
        if (d.n_ctx, d.n_ifce_out if d.flag_ifce else 0) != (20, 6):
            continue
        a = arm_ints(d, nn)
        X = contexts(a, rng, 1024)
        got, want = eval_f64(a, pack(a, "tile3_perm"), X), eval_int64(a, X)
        ok = eval_f64(a, pack(a), X)
        assert np.array_equal(ok[0], want[0]) and np.array_equal(ok[1], want[1]), label
        assert not (np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])), label
        n_new += 1
    assert n_new >= 1
    print(f"negative control tile3_perm: detected on {n_new} dense 20 + 6 ARMs")


@pytest.mark.parametrize("name", [n for n in PRESETS])
def test_dense_preset_arms_f64(oracle, cpu_seed, name):  # noqa: F811
    """The numpy DMMA evaluation equals the int64 ARM on the dense preset ARMs, which fit the f64 bound."""
    _, d, nn, _, _, _ = _cpu_live(cpu_seed, name)
    a = arm_ints(d, nn)
    cf = d.n_ifce_out if d.flag_ifce else 0
    if (d.n_ctx, cf) not in FAST_SHAPES:
        pytest.skip("generic ARM shape")
    assert fits_f64(a)
    X = contexts(a, np.random.default_rng(2))
    got, want = eval_f64(a, pack(a), X), eval_int64(a, X)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


# ------------------------------------------------------------------------------------------------------------------
# GPU
def _launches(d, name):
    """Library launches of one decode_many job: the entropy kernel, then the batched tail (a k_ups_level_b per
    cascade level but the last, k_tail_syn) or the per-stream one with k_syn_fused (k_ups_first, k_ups_pre +
    k_ups_convt per level, k_syn_fused)."""
    nl = sum(1 for g in range(d.n_grids) if not d.grid_is_hyper[g])
    if name in FUSED:
        return 1 + 1 + 2 * (nl - 1) + 1
    return 1 + (nl - 2) + 1


def _device_check(oracle, h, d, nn, lat, out, what):
    want = oracle.synthesize(d, nn, lat)
    got = out[0].cpu().numpy()
    assert np.array_equal(got, want), (what, np.argwhere(got != want)[:5].tolist())
    assert_within(got, intra(h, nn, lat), f"{what} device raw")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(TAIL) + list(FUSED))
def test_float_tail_matrix(ctx, oracle, cpu_seed, name):  # noqa: F811
    h, d, nn, nb, lb, lat = _cpu_live(cpu_seed, name)
    n0 = ctx.launch_count()
    out, lats = ctx.decode_many([d], [nb], [lb], want_latents=True)
    n = ctx.launch_count() - n0
    assert n == _launches(d, name), (name, n)
    assert np.array_equal(lats[0].cpu().numpy(), lat)
    _device_check(oracle, h, d, nn, lat, out[0], name)


@pytest.mark.gpu
def test_all_presets_in_one_call(ctx, oracle, cpu_seed):  # noqa: F811
    """Every reference preset in one decode_many call (the jobs of one (CINP, C) group differ in n3 and width): each
    output equals its decode alone, the oracle, and the restatement within its bound."""
    import torch

    names = list(PRESETS) + list(TAIL)
    items = [_cpu_live(cpu_seed, n) for n in names]
    outs, _ = ctx.decode_many([it[1] for it in items], [it[3] for it in items], [it[4] for it in items])
    for name, (h, d, nn, nb, lb, lat), out in zip(names, items, outs):
        alone, _ = ctx.decode_many([d], [nb], [lb])
        assert torch.equal(out, alone[0]), name
        _device_check(oracle, h, d, nn, lat, out, f"{name} in one call")


def _entropy_streams(cpu_seed, oracle):  # noqa: F811
    """Stream records (test_entropy_edges.Stream) of the dense 20 + 6 and 14 + 6 Cool-chics."""
    from test_entropy_edges import Stream

    from coolchic_b200._desc import desc_from_header

    out = []
    for name in DENSE:
        for k, (h, nb, lb) in enumerate(_coolchics(open(os.path.join(GOLDEN, name + ".cool"), "rb").read())):
            d = desc_from_header(h)
            if (d.n_ctx, d.n_ifce_out) in ((20, 6), (14, 6)):
                nn = oracle.decode_nn(d, bytes(nb))
                lat, _ = oracle.decode_latents(d, nn, bytes(lb))
                mu, sc = model_indices(d, nn, lat)
                out.append(Stream(f"{name}#{k}", d, nn, bytes(nb), bytes(lb), lat.astype(np.int64), mu, sc))
    for name in ("intra_vhop", "intra_hop"):
        h, d, nn, nb, lb, lat = _cpu_live(cpu_seed, name)
        mu, sc = model_indices(d, nn, lat)
        out.append(Stream(name, d, nn, nb, lb, lat.astype(np.int64), mu, sc))
    assert {(s.desc.n_ctx, s.desc.n_ifce_out) for s in out} == {(20, 6), (14, 6)}
    return out


@pytest.mark.gpu
def test_dense_arm_streams(ctx, oracle, cpu_seed):  # noqa: F811
    """Dense 20 + 6 and 14 + 6 streams: device encode = oracle encode, decode = the latents under the default, a
    one-warp and an all-warp producer mask; the rate pass against the checker; then 2 x SM + 5 of them in one call."""
    import torch
    from test_entropy_edges import DEFAULT_MASK, _check_stream

    streams = _entropy_streams(cpu_seed, oracle)
    try:
        for s in streams:
            _check_stream(ctx, oracle, ctx.set_producer_mask, s)
            _check_against_checker(ctx, oracle, s.desc, s.nb, s.lb)
        n = 2 * torch.cuda.get_device_properties(ctx.device).multi_processor_count + 5
        batch = [streams[i % len(streams)] for i in range(n)]
        alone = [ctx.decode_many([s.desc], [s.nb], [s.lb])[0][0] for s in streams]
        for mask in (DEFAULT_MASK, 0x0001):
            ctx.set_producer_mask(mask)
            outs, lats = ctx.decode_many([s.desc for s in batch], [s.nb for s in batch], [s.lb for s in batch],
                                         want_latents=True)
            for i, s in enumerate(batch):
                assert np.array_equal(lats[i].cpu().numpy(), s.lat), (i, hex(mask))
                assert torch.equal(outs[i], alone[i % len(streams)]), (i, hex(mask))
    finally:
        ctx.set_producer_mask(DEFAULT_MASK)


def _traced_vhop():
    """Run in a fresh process: the k_entropy names of the decode of the dense 20 + 6 fixture, in a torch.profiler
    trace."""
    import time

    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native
    from coolchic_b200._desc import desc_from_header

    ctx = _native.get_context(0)
    (h, nb, lb), = _coolchics(open(os.path.join(GOLDEN, "img_64x96_rgb_vhop_dense.cool"), "rb").read())
    d = desc_from_header(h)
    ctx.decode_many([d], [bytes(nb)], [bytes(lb)])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        time.sleep(0.05)
        ctx.decode_many([d], [bytes(nb)], [bytes(lb)])
        torch.cuda.synchronize()
        time.sleep(0.05)
    print(json.dumps(sorted({m.group(0) for m in (re.search(r"k_entropy<[^>]*>", e.name) for e in prof.events()) if m})))


@pytest.mark.gpu
def test_dense_vhop_runs_the_fast_20_6_kernel(ctx):
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.join(ROOT, 'oracle')!r}, {ROOT!r}]; "
            "import test_live_networks; test_live_networks._traced_vhop()")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True, cwd=here).stdout
    assert json.loads(r.strip().splitlines()[-1]) == ["k_entropy<20, 6, true>"]


def _gold_frames(name, fmt):
    g = np.load(os.path.join(GOLDEN, name + ("_frames.npz" if "gop" in name else ".npz")))
    if name.startswith("img"):
        return {0: list(g["rgb"].astype(np.int64))}
    n = len({k.split("_")[0] for k in g.files})
    return {i: [g[f"{i}_{k}"].astype(np.int64) for k in "yuv"] if fmt == "yuv420" else list(g[str(i)].astype(np.int64))
            for i in range(n)}


@pytest.mark.gpu
@pytest.mark.parametrize("name", DENSE)
def test_decode_video_vs_reference(ctx, oracle, name):
    """decode_video of the dense fixtures: every frame equal to the oracle's pipeline, and within one level of the
    reference's only where the oracle itself is (rounding ties)."""
    import pipeline
    from test_bitdepths import int_planes

    from coolchic_b200.bitstream.decode import decode_video

    fmt = "yuv420" if "yuv420" in name else "rgb"
    frames = decode_video(os.path.join(GOLDEN, name + ".cool"))
    mine = pipeline.decode_video(open(os.path.join(GOLDEN, name + ".cool"), "rb").read())
    gold = _gold_frames(name, fmt)
    assert sorted(frames) == [str(k) for k in sorted(gold)]
    n_diff = n_oracle = 0
    for k, planes in gold.items():
        got = int_planes(frames[str(k)].data, 8)
        for a, o, g in zip(got, int_planes(mine[k][2], 8), planes):
            assert np.array_equal(a, o), (name, k)
            assert np.abs(a - g).max() <= 1, (name, k)
            n_diff += int((a != g).sum())
            n_oracle += int((o != g).sum())
    assert n_diff == n_oracle
    print(f"{name}: {n_diff} samples differ from the reference (rounding ties)")


@pytest.mark.gpu
@pytest.mark.parametrize("name", [n for n in DENSE if "gop" in n])
def test_dense_gop_inter_frames(ctx, oracle, name):
    """Every P / B frame of the dense GOPs: reconstruct_frame against the oracle's prediction and tail, and the motion
    analysis (every variant; ref0_only / ref1_only against a beta that varies per pixel) with test_motion's checker."""
    from test_motion import _device_inter_frames, _source_tensor, check_frame
    from test_quality import _gop_sources, _to444

    fmt = "yuv420" if "yuv420" in name else "rgb"
    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    srcs = _gop_sources(name, fmt, seed=7)
    frames = _device_inter_frames(ctx, data)
    assert {f[0].get_value("frame_type") for f in frames} == {"P", "B"}
    for fh, cc, refs in frames:
        is_b = fh.get_value("frame_type") == "B"
        res = cc["residue"][0].cpu().numpy()
        beta = np.clip(res[4] + 0.5, 0, 1) if is_b else None
        if is_b:
            assert 0 < float(beta.mean()) < 1 and float(beta.std()) > 0.1
        gf, fs = fh.get_value("global_flow"), fh.get_value("warp_filter_size")
        args = (cc["residue"], cc["motion"], refs, is_b, fmt, 8, gf, fs)
        fin = ctx.reconstruct_frame(*args)
        r444 = [_to444(r) for r in refs]
        pre = oracle.inter_predict(res, cc["motion"][0].cpu().numpy(), r444[0], r444[1] if is_b else None, gf, fs)
        want = oracle.finish_frame(pre, 8, fmt)
        if fmt == "yuv420":
            for k in "yuv":
                assert np.array_equal(fin[k][0, 0].cpu().numpy(), want[k]), (name, k)
        else:
            assert np.array_equal(fin[0].cpu().numpy(), want), name
        src, layout = _source_tensor(ctx, srcs[fh.get_value("display_index")], fmt)
        check_frame(ctx, fh, cc, refs, src, layout, gf)

