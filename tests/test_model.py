"""Entropy-model analysis (coolchic_b200.bitstream.model, ccd_latent_rate_edited, ccd_rate_sweep): the rate of the
decoded latents under the coder's model with some ARM inputs read as 0, and the scale-calibration sweep.

The library reads an input as 0 by zeroing its row of the fixed-point weights.  The checker here restates every
variant the other way, by zeroing the INPUTS of the numpy ARM of test_rate (X[..., t] = 0, V[..., c] = 0), so the GPU
tests check the host edit independently; the CPU tests show on every golden model that the two are the same thing."""
import ctypes
import glob
import os
import subprocess
import sys

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from test_rate import CTX_DY, CTX_DX, GENERIC_ARM, _coolchics, _fixed_point, _golden, _latent_offsets, model_freq

GOLDENS = sorted(glob.glob(os.path.join(GOLDEN, "*.cool")))


# ---------------------------------------------------------------------------------------------- checker
def arm_model(d, nn):
    """(layers, Ws, Bs, {grid: (Wi, Bi)}) of the fixed-point ARM and IFCE, as test_rate.model_indices builds them."""
    from coolchic_b200 import synth

    sec = synth.split_nn(d, nn)
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim, H = d.n_ctx + cf, d.arm_hidden
    s_w, s_b = int(d.qshift[0]), int(d.qshift[1])
    ifce_cols = np.arange(dim) >= dim - cf if cf else np.zeros(dim, dtype=bool)
    aw, ab = sec["arm.weight"], sec["arm.bias"]
    layers = [_fixed_point(aw[f"mlp.{2 * l}"], ab[f"mlp.{2 * l}"], s_w, s_b,
                           ifce_cols if l == 0 else np.zeros(dim, dtype=bool), True, l == H) for l in range(H + 1)]
    if d.arm_stab:
        Ws, Bs = _fixed_point(aw["stab"], ab["stab"], s_w, s_b, ifce_cols, False)
    else:
        Ws, Bs = np.zeros((dim, 2), np.int64), np.zeros(2, np.int64)
    ifce = {}
    for g in range(d.n_grids):
        n_in = int(d.grid_ifce_in[g]) if cf else 0
        if n_in:
            ifce[g] = _fixed_point(sec["ifce.weight"][f"grid{g}"], sec["ifce.bias"][f"grid{g}"], int(d.qshift[2]),
                                   int(d.qshift[3]), np.zeros(n_in, dtype=bool), False)
    return layers, Ws, Bs, ifce


def arm_out(layers, Ws, Bs, X):
    """(o0, o1) of the integer ARM on inputs X [N, dim] (armint.py:180-203)."""
    x = X << 16
    s = Bs + x @ Ws
    for W, B in layers[:-1]:
        x = np.maximum(B + x @ W, 0) >> 16
    return (layers[-1][1] + x @ layers[-1][0] + s) >> 24


def ifce_features(Wi, Bi, V):
    acc = Bi + (V << 16) @ Wi
    return (acc >> 24).astype(np.float32).astype(np.int64)  # fp32 round trip


def bits_of(mask):
    return [b for b in range(64) if (int(mask) >> b) & 1]


def variant_indices(d, nn, latents, zero_ctx=0, zero_ifce_out=0, zero_ifce_grids=0):
    """(mu_idx, sc_idx) of every symbol (decode order) under the variant, by zeroing inputs: spatial input t,
    IFCE feature c, and every IFCE channel that reads a grid of zero_ifce_grids."""
    layers, Ws, Bs, ifce = arm_model(d, nn)
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim = d.n_ctx + cf
    offs = _latent_offsets(d)
    lat = np.asarray(latents).astype(np.int64)
    grids = [lat[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]].reshape(d.grid_h[g], d.grid_w[g]) for g in range(d.n_grids)]
    mu_idx, sc_idx = np.zeros(lat.size, np.int64), np.zeros(lat.size, np.int64)
    for g in range(d.n_grids):
        h, w = grids[g].shape
        X = np.zeros((h, w, dim), np.int64)
        P = np.pad(grids[g], ((4, 0), (4, 4)))
        for t in range(d.n_ctx):
            X[:, :, t] = P[4 + CTX_DY[t]:4 + CTX_DY[t] + h, 4 + CTX_DX[t]:4 + CTX_DX[t] + w]
        if g in ifce:
            n_in = int(d.grid_ifce_in[g])
            yy, xx = np.arange(h) >> 1, np.arange(w) >> 1
            V = np.zeros((h, w, n_in), np.int64)
            if g < d.n_grids - 1:  # the first grid decoded has one all-zero input
                sh = 0
                for c in range(n_in):
                    if c > 0 and (d.grid_h[g + c], d.grid_w[g + c]) != (d.grid_h[g + 1 + c], d.grid_w[g + 1 + c]):
                        sh += 1
                    V[:, :, c] = grids[g + 1 + c][(yy >> sh)[:, None], (xx >> sh)[None, :]]
                    if (zero_ifce_grids >> (g + 1 + c)) & 1:
                        V[:, :, c] = 0
            X[:, :, d.n_ctx:] = ifce_features(*ifce[g], V)
        for t in bits_of(zero_ctx):
            X[:, :, t] = 0
        for c in bits_of(zero_ifce_out):
            X[:, :, d.n_ctx + c] = 0
        o = arm_out(layers, Ws, Bs, X.reshape(h * w, dim))
        sl = slice(offs[g], offs[g] + h * w)
        mu_idx[sl] = np.clip(o[:, 0] + 16384, 0, 32767)
        sc_idx[sl] = np.clip(o[:, 1] + 1280, 0, 2560)
    return mu_idx, sc_idx


def _grid_sums(d, per_symbol):
    offs = _latent_offsets(d)
    return [float(np.sum(per_symbol[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]])) for g in range(d.n_grids)]


def _model_bits(oracle, lat, mu_idx, sc_idx):
    freq = model_freq(oracle, lat, mu_idx, sc_idx)
    return freq, 24.0 - np.log2(freq.astype(np.float64))


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("path", GOLDENS, ids=os.path.basename)
def test_weight_edit_is_input_zeroing(path, oracle):
    """Zeroing row i of the first layer (residual +I included) and of the stabiliser gives, on random inputs, exactly
    the ARM with input i read as 0; zeroing row c of an IFCE weight gives exactly the IFCE with channel c read as 0.
    Every single-input mask of every golden model: 0 to 2+ hidden layers, the 3x3 / five-layer architectures."""
    from coolchic_b200._desc import desc_from_header

    rng = np.random.default_rng(0)
    for h, nb, _ in _coolchics(open(path, "rb").read()):
        d = desc_from_header(h)
        layers, Ws, Bs, ifce = arm_model(d, oracle.decode_nn(d, nb))
        dim = Ws.shape[0]
        X = rng.integers(-64, 64, size=(512, dim)).astype(np.int64)
        X[:, d.n_ctx:] = rng.integers(-4096, 4096, size=(512, dim - d.n_ctx))
        for i in range(dim):
            Xz = X.copy()
            Xz[:, i] = 0
            L = [(W.copy(), B) for W, B in layers]
            L[0][0][i, :] = 0
            Ws_e = Ws.copy()
            Ws_e[i, :] = 0
            assert np.array_equal(arm_out(L, Ws_e, Bs, X), arm_out(layers, Ws, Bs, Xz)), (path, i)
        for g, (Wi, Bi) in ifce.items():
            V = rng.integers(-64, 64, size=(512, Wi.shape[0])).astype(np.int64)
            for c in range(Wi.shape[0]):
                Vz = V.copy()
                Vz[:, c] = 0
                We = Wi.copy()
                We[c, :] = 0
                assert np.array_equal(ifce_features(We, Bi, V), ifce_features(Wi, Bi, Vz)), (path, g, c)


def test_static_bits_formula():
    """The static baseline of a histogram equals the ideal static code of the symbols themselves: the sum over
    symbols of -log2(p(s)) with p the symbol's frequency, from np.bincount."""
    from coolchic_b200.bitstream import model

    rng = np.random.default_rng(1)
    for n, spread in ((1, 1), (1000, 3), (50000, 20)):
        sym = np.clip(np.round(rng.laplace(0, spread, size=n)), -64, 63).astype(np.int64)
        counts = np.bincount(sym + 64, minlength=128)
        p = counts[sym + 64] / n
        assert model.static_bits(counts) == pytest.approx(float(np.sum(-np.log2(p))), rel=1e-12, abs=1e-9)
    assert model.static_bits(np.zeros(128)) == 0.0


@pytest.mark.parametrize("path", GOLDENS, ids=os.path.basename)
def test_variant_table(path):
    """The variants of every golden Cool-chic: ctx_0 .. ctx_{n_ctx - 1}, no_ifce with IFCE, no_hyper only with
    hyperlatent grids, and the masks of the definition."""
    from coolchic_b200._desc import desc_from_header
    from coolchic_b200.bitstream import model

    for h, _, _ in _coolchics(open(path, "rb").read()):
        d = desc_from_header(h)
        v = model.variant_edits(d)
        hyper = [g for g in range(d.n_grids) if d.grid_is_hyper[g]]
        want = ["decoded"] + [f"ctx_{k}" for k in range(d.n_ctx)] + (["no_ifce"] if d.flag_ifce else []) + \
            (["no_hyper"] if d.flag_ifce and hyper else []) + ["no_context"]
        assert list(v) == want
        assert v["ctx_0"][0] == v["no_context"][0] == (1 << d.n_ctx) - 1
        assert v[f"ctx_{d.n_ctx - 1}"] == (1 << (d.n_ctx - 1), 0, 0)
        if hyper:
            assert v["no_hyper"] == (0, 0, sum(1 << g for g in hyper))


# ---------------------------------------------------------------------------------------------- GPU
def _cc(ctx, data, k=0):
    """(desc, NN integers, device latents, host latents) of the k-th Cool-chic of a bitstream."""
    from coolchic_b200 import _native
    from coolchic_b200._desc import desc_from_header

    h, nb, lb = _coolchics(data)[k]
    d = desc_from_header(h)
    _, lats = ctx.decode_many([d], [nb], [lb], want_latents=True)
    return d, _native.decode_nn(d, nb), lats[0], lats[0].cpu().numpy()


def _1080p(ctx, seed_stream):
    from coolchic_b200 import synth

    return synth.make_image_stream(ctx, seed_stream, 1080, 1920)


def _variant_run(ctx, d, nn, lat, names=None):
    from coolchic_b200.bitstream import model

    ed = model.variant_edits(d)
    names = list(ed) if names is None else names
    res = ctx.latent_rate([d] * len(names), [nn] * len(names), [lat] * len(names), want_freq=True,
                          edits=[ed[n] for n in names])
    return ed, dict(zip(names, res))


def _assert_bits_match(bits, freq):
    # bits = fp32(24 - log2(f64(freq))): one ulp, as test_rate allows for the device log2
    want = (24.0 - np.log2(freq.astype(np.float64))).astype(np.float32)
    assert np.all(np.abs(bits.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)) <= 1)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kodim14"] + GENERIC_ARM + ["1080p"])
def test_decoded_equals_video_rate(ctx, seed_stream, name):
    """The all-zero edit is ccd_latent_rate, bit for bit: per-symbol bits, freq and grid sums."""
    data = _1080p(ctx, seed_stream) if name == "1080p" else _golden(name)
    d, nn, lat, _ = _cc(ctx, data)
    plain = ctx.latent_rate([d], [nn], [lat], want_freq=True, want_mu_sc=True)[0]
    ed = ctx.latent_rate([d], [nn], [lat], want_freq=True, want_mu_sc=True, edits=[(0, 0, 0)])[0]
    for k in ("bits", "freq", "mu_sc"):
        assert np.array_equal(plain[k].cpu().numpy(), ed[k].cpu().numpy())
    assert plain["grid_bits"] == ed["grid_bits"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["kodim14"] + GENERIC_ARM + ["gop5_64x96_yuv420:2", "gop5_64x96_yuv420:3"])
def test_every_variant_equals_checker(ctx, oracle, case):
    """Every variant of kodim14 (IFCE and hyperlatents), of the generic-ARM fixtures and of a P/B frame's residue and
    motion Cool-chics: freq of every symbol equals the input-zeroing checker's, bits to one ulp of it, grid sums to
    1e-12 of the host's."""
    name, _, k = case.partition(":")
    d, nn, lat, lat_h = _cc(ctx, _golden(name), int(k or 0))
    ed, res = _variant_run(ctx, d, nn, lat)
    for v, e in ed.items():
        freq, exact = _model_bits(oracle, lat_h, *variant_indices(d, nn, lat_h, *e))
        assert np.array_equal(res[v]["freq"].cpu().numpy().view(np.uint32), freq), v
        _assert_bits_match(res[v]["bits"].cpu().numpy(), freq)
        np.testing.assert_allclose(res[v]["grid_bits"], _grid_sums(d, exact), rtol=1e-12, atol=1e-9)


@pytest.mark.gpu
def test_1080p_variants_equal_checker(ctx, oracle, seed_stream):
    """ctx_0 and no_ifce of the 1080p seven-grid frame (the fast <14, 6> kernel) against the checker."""
    d, nn, lat, lat_h = _cc(ctx, _1080p(ctx, seed_stream))
    assert d.n_grids == 7
    ed, res = _variant_run(ctx, d, nn, lat, ["ctx_0", "no_ifce"])
    for v in ("ctx_0", "no_ifce"):
        freq, _ = _model_bits(oracle, lat_h, *variant_indices(d, nn, lat_h, *ed[v]))
        assert np.array_equal(res[v]["freq"].cpu().numpy().view(np.uint32), freq), v


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["kodim14", "gop5_64x96_yuv420:2"])
def test_identities(ctx, case):
    """Bit for bit: under no_ifce the grids without IFCE input, and under no_hyper the grids whose IFCE reads no
    hyperlatent grid, keep their decoded bits."""
    name, _, k = case.partition(":")
    d, nn, lat, _ = _cc(ctx, _golden(name), int(k or 0))
    ed, res = _variant_run(ctx, d, nn, lat)
    offs = _latent_offsets(d)
    dec = res["decoded"]["bits"].cpu().numpy()

    def grid(a, g):
        return a[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]]

    n_same = 0
    for g in range(d.n_grids):
        if d.grid_ifce_in[g] == 0:
            assert np.array_equal(grid(res["no_ifce"]["bits"].cpu().numpy(), g), grid(dec, g))
            n_same += 1
        reads = [g + 1 + c for c in range(d.grid_ifce_in[g]) if g + 1 + c < d.n_grids]
        if "no_hyper" in res and not any(d.grid_is_hyper[x] for x in reads):
            assert np.array_equal(grid(res["no_hyper"]["bits"].cpu().numpy(), g), grid(dec, g))
            n_same += 1
    assert n_same > 0
    assert ("no_hyper" in res) == (name == "kodim14")


def _sweep_check(ctx, oracle, d, nn, lat, lat_h, offsets):
    r = ctx.latent_rate([d], [nn], [lat], want_mu_sc=True)[0]
    sw = ctx.rate_sweep([d], [lat], [r["mu_sc"]], offsets)[0]
    ms = r["mu_sc"].cpu().numpy().view(np.uint32)
    mu, sc = (ms & 0xFFFF).astype(np.int64), (ms >> 16).astype(np.int64)
    for k, off in enumerate(offsets):
        _, exact = _model_bits(oracle, lat_h, mu, np.clip(sc + off, 0, 2560))
        np.testing.assert_allclose([b[k] for b in sw["bits"]], _grid_sums(d, exact), rtol=1e-12, atol=1e-9)
        if off == 0:
            # the same symbols' bits as the rate pass's grid sums, summed in another order (the sweep's threads own
            # other symbols than the rate pass's lanes): equal to rounding
            np.testing.assert_allclose([b[k] for b in sw["bits"]], r["grid_bits"], rtol=1e-12, atol=0)
    offs = _latent_offsets(d)
    for g in range(d.n_grids):
        s = lat_h[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]].astype(np.int64)
        assert np.array_equal(sw["hist"][g], np.bincount(s + 64, minlength=128))
    return sw, sc


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["kodim14", "gop5_64x96_yuv420:3"])
def test_sweep_equals_checker(ctx, oracle, case):
    name, _, k = case.partition(":")
    d, nn, lat, lat_h = _cc(ctx, _golden(name), int(k or 0))
    _sweep_check(ctx, oracle, d, nn, lat, lat_h, [-2560, -300, -64, -8, 0, 8, 64, 300, 2560])


@pytest.mark.gpu
@pytest.mark.parametrize("model_name", ["smin", "smax"])
def test_sweep_clamps_at_the_table_ends(ctx, oracle, model_name):
    """Crafted constant models pinned at sc_idx 0 / 2560: offsets past the end clamp there, so they cost exactly the
    bits of offset 0 (the same symbols summed in the same order), and every offset still equals the checker."""
    import torch
    from test_entropy_edges import MODELS, build_header, craft_latents, craft_nn

    _, _, _, d = build_header("17x33")
    m = MODELS[model_name]
    nn = craft_nn(d, m)
    lat_h, _, sc = craft_latents(d, m, "P4")
    assert set(np.unique(sc)) == {m.sc}
    lat = torch.from_numpy(lat_h.astype(np.int8)).cuda()
    offsets = [-64, -1, 0, 1, 64]
    sw, sc_used = _sweep_check(ctx, oracle, d, nn, lat, lat_h.astype(np.int8), offsets)
    assert set(np.unique(sc_used)) == {m.sc}
    past = [0, 1] if m.sc == 0 else [3, 4]
    for k in past:
        assert [b[k] for b in sw["bits"]] == [b[2] for b in sw["bits"]]


@pytest.mark.gpu
def test_launches_per_frame(ctx):
    """One k_latent_rate launch for every variant of a P/B frame's residue and motion Cool-chics, one k_rate_sweep
    launch for both; video_model_analysis makes one decode and these two per frame."""
    from coolchic_b200.bitstream import model, rate

    data = _golden("gop5_64x96_yuv420")
    _, frames, flat = rate._split_frames(data)
    ccs = _coolchics(data)
    n0 = ctx.launch_count()
    _, descs, nns, lats = rate._decode_latents([c[0] for c in ccs], [c[1] for c in ccs], [c[2] for c in ccs], ctx.device)
    n_decode = ctx.launch_count() - n0
    coding_idx, fh, idx, _ = next(f for f in frames if f[1].get_value("frame_type") in ("P", "B"))
    assert set(idx) == {"residue", "motion"}
    jobs = [(i, e) for i in idx.values() for e in model.variant_edits(descs[i]).values()]
    n0 = ctx.launch_count()
    res = ctx.latent_rate([descs[i] for i, _ in jobs], [nns[i] for i, _ in jobs], [lats[i] for i, _ in jobs],
                          want_mu_sc=True, edits=[e for _, e in jobs])
    assert ctx.launch_count() - n0 == 1
    firsts = [next(r for (j, e), r in zip(jobs, res) if j == i and e == (0, 0, 0)) for i in idx.values()]
    n0 = ctx.launch_count()
    ctx.rate_sweep([descs[i] for i in idx.values()], [lats[i] for i in idx.values()], [r["mu_sc"] for r in firsts],
                   model.SIGMA_OFFSETS)
    assert ctx.launch_count() - n0 == 1
    n0 = ctx.launch_count()
    model.video_model_analysis(data)
    assert ctx.launch_count() - n0 == n_decode + 2 * len(frames)


@pytest.mark.gpu
def test_two_calls_are_identical(ctx):
    from coolchic_b200.bitstream import model

    data = _golden("kodim14")
    a, b = model.video_model_analysis(data), model.video_model_analysis(data)
    for key in a:
        for name, c in a[key].coolchics.items():
            o = b[key].coolchics[name]
            assert c.variants == o.variants and c.sweep_bits == o.sweep_bits
            assert np.array_equal(c.hist, o.hist)


def _launches_refused(ctx, fn, code=-1):
    from coolchic_b200 import _native

    n0 = ctx.launch_count()
    with pytest.raises(_native.CcdError) as e:
        fn()
    assert e.value.code == code
    assert ctx.launch_count() == n0
    return e.value


@pytest.mark.gpu
def test_edit_argument_errors(ctx):
    """Refused before any launch: a zero_ctx bit >= n_ctx, a zero_ifce_out bit >= n_ifce_out, a zero_ifce_grids bit
    >= n_grids, any IFCE bit in a model without IFCE."""
    from coolchic_b200 import _native

    d, nn, lat, _ = _cc(ctx, _golden("kodim14"))
    for e in [(1 << d.n_ctx, 0, 0), (0, 1 << d.n_ifce_out, 0), (0, 0, 1 << d.n_grids)]:
        err = _launches_refused(ctx, lambda: ctx.latent_rate([d, d], [nn, nn], [lat, lat], edits=[(0, 0, 0), e]))
        assert "job 1" in str(err)
    plain = type(d).from_buffer_copy(d)
    plain.flag_ifce, plain.n_ifce_out = 0, 0
    for g in range(plain.n_grids):
        plain.grid_ifce_in[g] = 0
    nn0 = np.zeros(_native.load_library().ccd_nn_count(ctypes.byref(plain)), np.int64)
    ctx.latent_rate([plain], [nn0], [lat], edits=[(1, 0, 0)])  # a model without IFCE takes spatial edits
    for e in [(0, 1, 0), (0, 0, 1)]:
        _launches_refused(ctx, lambda: ctx.latent_rate([plain], [nn0], [lat], edits=[e]))


@pytest.mark.gpu
def test_sweep_argument_errors(ctx):
    """n_offsets outside 1 .. 32 and an offset outside [-2560, 2560] are refused before any launch; a latent outside
    [-64, 63] and an (mu_idx, sc_idx) outside its table are reported with the smallest bad decode-order index."""
    from coolchic_b200 import _native

    d, nn, lat, _ = _cc(ctx, _golden("kodim14"))
    ms = ctx.latent_rate([d], [nn], [lat], want_mu_sc=True)[0]["mu_sc"]
    lib = _native.load_library()

    def raw(n_offsets, offsets):
        job = (_native.CcdSweepJob * 1)()
        job[0].desc = ctypes.pointer(d)
        job[0].d_latents, job[0].d_mu_sc, job[0].n_offsets = lat.data_ptr(), ms.data_ptr(), n_offsets
        job[0].sc_offset[:len(offsets)] = offsets
        _native._check(lib.ccd_rate_sweep(ctx._h, job, 1, ctx._stream()), job)

    raw(32, list(range(-16, 16)))
    for n_off in (0, 33, -1):
        _launches_refused(ctx, lambda: raw(n_off, [0]))
    for off in (-2561, 2561):
        _launches_refused(ctx, lambda: ctx.rate_sweep([d], [lat], [ms], [0, off]))
    for bad_lat, bad_ms in ((64, None), (-65, None), (None, 32768), (None, 2561 << 16)):
        lat2, ms2 = lat.clone(), ms.clone()
        i_lat, i_ms = 200001, 123457
        if bad_lat is not None:
            lat2[i_lat] = bad_lat
        if bad_ms is not None:
            ms2[i_ms] = bad_ms
        with pytest.raises(_native.CcdError) as e:
            ctx.rate_sweep([d], [lat2], [ms2], [0])
        assert e.value.code == -1 and e.value.bad_index == [i_lat if bad_lat is not None else i_ms]
    lat2, ms2 = lat.clone(), ms.clone()
    lat2[200001], ms2[123457] = 64, 32768
    with pytest.raises(_native.CcdError) as e:
        ctx.rate_sweep([d], [lat2], [ms2], [0])
    assert e.value.bad_index == [123457]


@pytest.mark.gpu
def test_video_model_analysis_matches_video_rate(ctx):
    from coolchic_b200.bitstream import model, rate

    data = _golden("gop3_40x56_rgb_bicubic")
    fm, fr = model.video_model_analysis(data), rate.video_rate(data)
    assert list(fm) == list(fr)
    for key in fr:
        assert fm[key].frame_type == fr[key].frame_type and fm[key].img_size == fr[key].img_size
        assert set(fm[key].coolchics) == set(fr[key].coolchics)
        for name, c in fm[key].coolchics.items():
            r = fr[key].coolchics[name]
            assert c.variants["decoded"] == r.grid_bits
            assert c.grid_sizes == r.grid_sizes
            assert c.nn_bits == r.nn_module_bits
            assert "no_hyper" not in c.variants and c.hyper_net is None
            assert c.ifce_net == c.total("no_ifce") - c.total("decoded") - r.nn_module_bits["ifce"]
            assert c.ctx_curve[-1] == c.total("decoded") and len(c.ctx_curve) == c.n_ctx + 1
            assert [int(h.sum()) for h in c.hist] == [gh * gw for gh, gw in c.grid_sizes]


@pytest.mark.gpu
def test_cli_model(ctx):
    cmd = [sys.executable, os.path.join(ROOT, "cc_rate.py"), "-i", os.path.join(GOLDEN, "kodim14.cool")]
    plain = subprocess.run(cmd, capture_output=True, text=True, check=True).stdout
    out = subprocess.run(cmd + ["--model"], capture_output=True, text=True, check=True).stdout
    assert out.startswith(plain.rstrip("\n").split("\n")[0])
    assert "ARM net" not in plain
    for line in ("ARM net", "IFCE net", "hyperlatent net", "ctx_k bits"):
        assert line in out
    assert "n/a" not in out.split("hyperlatent net")[1].split("\n")[0]
