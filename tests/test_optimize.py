"""Lossless bitstream optimisation (DESIGN §4.11): candidate pricing (ccd_rate_candidates / k_rate_candidates) against
the exact rate checker of test_rate.py, the exp-Golomb recount, the header and payload rewrite, and optimize_bitstream's
output decoded by the GPU decoder and by the CPU oracle."""
import os

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from test_arm_f64 import FAST_SHAPES, arm_ints, fits_f64
from test_rate import CTX_DX, CTX_DY, _coolchics, _fixed_point, _golden, _latent_offsets, model_freq, model_indices

SMALL = ["img_48x64_rgb_arm8_1hidden", "img_40x56_yuv444_10bit_arm24", "arch_space_deep7", "arch_space_linear_6_2",
         "arch_space_ifce_16grids", "arch_space_ctx40", "img_96x128_rgb_12grids_dense", "gop3_40x56_rgb"]
DENSE = ["img_96x128_rgb_12grids_dense", "img_64x96_rgb_vhop_dense", "gop3_48x72_yuv420_bicubic_dense",
         "gop3_40x56_rgb_sinc8_dense"]


def _model_span(d):
    """[0, n): the ARM and IFCE integers at the start of the NN order, and where the ARM ends."""
    from coolchic_b200.bitstream.optimize import _sections

    sec = _sections(d)
    return sec[("arm", "bias")][1], sec[("ifce", "bias")][1]


def _draw(d, rng, n, deltas=(1, -1, 3, -3, 64, -64)):
    """n (index, delta) pairs: a sample over the ARM and IFCE integers, every ARM layer, the stabiliser and the IFCE."""
    from coolchic_b200 import synth

    secs, p, groups = synth.nn_sections(d), 0, []
    for key, items in secs.items():
        for _, shape in items:
            m = int(np.prod(shape))
            if key.startswith("arm") or key.startswith("ifce"):
                groups.append(range(p, p + m))
            p += m
    out = [(int(rng.choice(g)), int(rng.choice(deltas))) for g in groups if len(g)]
    while len(out) < n:
        g = groups[rng.integers(len(groups))]
        out.append((int(rng.choice(g)), int(rng.choice(deltas))))
    return out[:n]


def _fast_plan(d, nn):
    """The decoder's kernel choice (ccd_entropy_has_fast, the IFCE bound, arm_fits_f64), from test_arm_f64."""
    if (d.n_ctx, d.n_ifce_out) not in FAST_SHAPES:
        return False
    a = arm_ints(d, nn)
    return a["feat_bound"] is not None and fits_f64(a)


# ---- CPU: the delta evaluation the kernel makes, restated in numpy --------------------------------------------------
def _base_eval(d, nn, lat):
    """Per grid: inputs, every layer's input and hidden pre-activation, the IFCE sums and inputs, the output sums."""
    a = arm_ints(d, nn)
    from coolchic_b200 import synth

    sec = synth.split_nn(d, nn)
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim = d.n_ctx + cf
    offs = _latent_offsets(d)
    lat = np.asarray(lat).astype(np.int64)
    grids = [lat[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]].reshape(d.grid_h[g], d.grid_w[g]) for g in range(d.n_grids)]
    out = []
    for g in range(d.n_grids):
        h, w = grids[g].shape
        X = np.zeros((h, w, dim), np.int64)
        P = np.pad(grids[g], ((4, 0), (4, 4)))
        for t in range(d.n_ctx):
            X[:, :, t] = P[4 + CTX_DY[t]:4 + CTX_DY[t] + h, 4 + CTX_DX[t]:4 + CTX_DX[t] + w]
        n_in = int(d.grid_ifce_in[g]) if cf else 0
        V = np.zeros((h * w, max(n_in, 1)), np.int64)
        IA = np.zeros((h * w, max(cf, 1)), np.int64)
        if n_in:
            Wi, Bi = _fixed_point(sec["ifce.weight"][f"grid{g}"], sec["ifce.bias"][f"grid{g}"], int(d.qshift[2]),
                                  int(d.qshift[3]), np.zeros(n_in, dtype=bool), False)
            yy, xx = np.arange(h) >> 1, np.arange(w) >> 1
            Vg = np.zeros((h, w, n_in), np.int64)
            if g < d.n_grids - 1:
                sh = 0
                for c in range(n_in):
                    if c > 0 and (d.grid_h[g + c], d.grid_w[g + c]) != (d.grid_h[g + 1 + c], d.grid_w[g + 1 + c]):
                        sh += 1
                    Vg[:, :, c] = grids[g + 1 + c][(yy >> sh)[:, None], (xx >> sh)[None, :]]
            V = Vg.reshape(h * w, n_in)
            IA = Bi + (V << 16) @ Wi
            X[:, :, d.n_ctx:] = (IA.reshape(h, w, cf) >> 24).astype(np.float32).astype(np.int64)
        x = X.reshape(h * w, dim) << 16
        xs, ys = [x], []
        for W, B in a["layers"][:-1]:
            ys.append(B + xs[-1] @ W)
            xs.append(np.maximum(ys[-1], 0) >> 16)
        out.append(dict(xs=xs, ys=ys, V=V, IA=IA, S=a["Bs"] + x @ a["Ws"], A=a["layers"][-1][1] + xs[-1] @ a["layers"][-1][0]))
    return out, a


def _delta_indices(d, nn, base, a, idx, delta):
    """(mu_idx, sc_idx) of every symbol under the model with nn[idx] += delta, from the base evaluation: one changed
    fixed-point entry, a rank-1 change of the next layer, the later layers on the changed units."""
    from coolchic_b200 import synth

    nn2 = nn.copy()
    nn2[idx] += delta
    a2 = arm_ints(d, nn2)
    nh, cf = d.arm_hidden, (d.n_ifce_out if d.flag_ifce else 0)
    mu, sc = np.zeros(nn.size and sum(d.grid_h[g] * d.grid_w[g] for g in range(d.n_grids)), np.int64), None
    sc = np.zeros_like(mu)
    offs = _latent_offsets(d)
    n_arm = _model_span(d)[0]
    # the changed ARM entry
    change = None
    if idx < n_arm:
        pairs = [(("layer", l), a["layers"][l][k], a2["layers"][l][k], k) for l in range(nh + 1) for k in (0, 1)]
        pairs += [(("stab", 0), a["Ws"], a2["Ws"], 0), (("stab", 0), a["Bs"], a2["Bs"], 1)]
        for key, v0, v1, k in pairs:
            dif = np.argwhere(v1 != v0)
            if len(dif):
                change = (key, k, tuple(dif[0]), int(v1[tuple(dif[0])] - v0[tuple(dif[0])]))
                break
    sec2, sec1 = synth.split_nn(d, nn2), synth.split_nn(d, nn)

    def forward_from(b, l, Dx):
        """Changes of the output sums when the input of layer l moves by Dx [n, dim]."""
        for j in range(l, nh):
            W, _ = a["layers"][j]
            Dx = (np.maximum(b["ys"][j] + Dx @ W, 0) >> 16) - b["xs"][j + 1]
        return Dx @ a["layers"][nh][0]

    for g in range(d.n_grids):
        b = base[g]
        n = b["S"].shape[0]
        dS, dA = np.zeros((n, 2), np.int64), np.zeros((n, 2), np.int64)
        if change is not None:
            (kind, l), k, pos, dv = change
            if kind == "stab":
                x = b["xs"][0][:, pos[0]] if k == 0 else 1
                dS[:, pos[-1]] = dv * x
            elif l == nh:
                x = b["xs"][nh][:, pos[0]] if k == 0 else 1
                dA[:, pos[-1]] = dv * x
            else:
                o = pos[-1]
                x = b["xs"][l][:, pos[0]] if k == 0 else 1
                Dx = np.zeros_like(b["xs"][l + 1])
                Dx[:, o] = (np.maximum(b["ys"][l][:, o] + dv * x, 0) >> 16) - b["xs"][l + 1][:, o]
                dA = forward_from(b, l + 1, Dx)
        elif idx >= n_arm and cf and d.grid_ifce_in[g] and f"grid{g}" in sec2["ifce.weight"]:
            n_in = int(d.grid_ifce_in[g])
            W1, B1 = _fixed_point(sec2["ifce.weight"][f"grid{g}"], sec2["ifce.bias"][f"grid{g}"], int(d.qshift[2]),
                                  int(d.qshift[3]), np.zeros(n_in, dtype=bool), False)
            W0, B0 = _fixed_point(sec1["ifce.weight"][f"grid{g}"], sec1["ifce.bias"][f"grid{g}"], int(d.qshift[2]),
                                  int(d.qshift[3]), np.zeros(n_in, dtype=bool), False)
            dw, db = np.argwhere(W1 != W0), np.argwhere(B1 != B0)
            if len(dw) or len(db):
                if len(dw):
                    c, o = dw[0]
                    acc = b["IA"][:, o] + int(W1[c, o] - W0[c, o]) * (b["V"][:, c] << 16)
                else:
                    o = db[0][0]
                    acc = b["IA"][:, o] + int(B1[o] - B0[o])
                u = d.n_ctx + o
                Du = ((acc >> 24).astype(np.float32).astype(np.int64) << 16) - b["xs"][0][:, u]
                dS = Du[:, None] * a["Ws"][u][None, :]
                Dx = np.zeros_like(b["xs"][0])
                Dx[:, u] = Du
                dA = forward_from(b, 0, Dx)
        o = (b["A"] + dA + b["S"] + dS) >> 24
        sl = slice(offs[g], offs[g] + n)
        mu[sl] = np.clip(o[:, 0] + 16384, 0, 32767)
        sc[sl] = np.clip(o[:, 1] + 1280, 0, 2560)
    return mu, sc


@pytest.mark.parametrize("name", SMALL + ["kodim14"])
def test_delta_evaluation_matches_checker(oracle, name):
    """On every golden model, a seeded sample of one-integer edits in every ARM layer, the stabiliser and the IFCE:
    the delta evaluation gives the (mu, scale) indices and frequencies of a full checker pass on the edited integers."""
    import coolchic_b200  # noqa: F401
    from coolchic_b200._desc import desc_from_header

    h, nb, lb = _coolchics(_golden(name))[0]
    d = desc_from_header(h)
    nn = np.asarray(oracle.decode_nn(d, nb), dtype=np.int64)
    lat = oracle.decode_latents(d, nn, lb)[0].astype(np.int64)
    base, a = _base_eval(d, nn, lat)
    rng = np.random.default_rng(11)
    for idx, dl in _draw(d, rng, 6 if name == "kodim14" else 12):
        nn2 = nn.copy()
        nn2[idx] += dl
        mu, sc = model_indices(d, nn2, lat)
        mu_d, sc_d = _delta_indices(d, nn, base, a, idx, dl)
        assert np.array_equal(mu, mu_d) and np.array_equal(sc, sc_d), (name, idx, dl)
        assert np.array_equal(model_freq(oracle, lat, mu, sc), model_freq(oracle, lat, mu_d, sc_d))


def test_expgol_recount_is_the_minimum():
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream.expgolomb import exp_golomb_bits
    from coolchic_b200.bitstream.header import EXP_GOL_TABLE
    from coolchic_b200.bitstream.optimize import best_expgol_count

    rng = np.random.default_rng(5)
    for scale in (0, 1, 3, 40, 900, 60000):
        v = np.round(rng.laplace(0, scale + 1e-9, 200)).astype(np.int64)
        costs = [sum(exp_golomb_bits(v, [k] * v.size)) for k in EXP_GOL_TABLE]
        k = best_expgol_count(v)
        assert costs[k] == min(costs) and k == costs.index(min(costs))


def test_rewrite_decodes_to_the_golden_latents(oracle, kodim14):
    """A hand-edited ARM integer, the golden latents encoded again by the oracle under it, the header rewritten: the
    oracle decodes the new file to the golden latents and image, and the header round-trips."""
    from coolchic_b200._desc import desc_from_header
    from coolchic_b200.bitstream.expgolomb import encode_exp_golomb
    from coolchic_b200.bitstream.header import NN_KINDS, NN_MODULES, CoolChicHeader
    from coolchic_b200.bitstream.optimize import _sections

    d, h = kodim14["desc"], kodim14["header"]
    nn = np.asarray(oracle.decode_nn(d, kodim14["nn_bytes"]), dtype=np.int64)
    lat = np.asarray(kodim14["latents"]).astype(np.int8)
    nn2 = nn.copy()
    nn2[_model_span(d)[0] - 3] += 2  # an ARM bias
    sec = _sections(d)
    counts = []
    for m in NN_MODULES:
        for k in NN_KINDS:
            s, e = sec[(m, k)]
            counts += [int(h.get_value("nn_expgol_cnt").get_value(m, k))] * (e - s)
    payload, pad = encode_exp_golomb([int(v) for v in nn2], counts)
    lat_bytes = oracle.encode_latents(d, nn2, lat)
    raw = bytes(kodim14["data"])
    n_pre = len(raw) - len(kodim14["nn_bytes"]) - len(kodim14["lat_bytes"]) - h.get_value("n_bytes_header")
    h2 = CoolChicHeader()
    h2.read_header(raw[n_pre:])
    h2.set_value("nn_n_bytes", len(payload))
    h2.set_value("nn_n_bit_pad", pad)
    h2.set_value("n_bytes_latent", len(lat_bytes))
    hb = h2.to_bytes()
    h3 = CoolChicHeader()
    assert h3.read_header(hb + payload + lat_bytes) == payload + lat_bytes
    assert h3.to_bytes() == hb
    d3 = desc_from_header(h3)
    nn3 = np.asarray(oracle.decode_nn(d3, payload), dtype=np.int64)
    assert np.array_equal(nn3, nn2)
    lat3 = oracle.decode_latents(d3, nn3, lat_bytes)[0]
    assert np.array_equal(lat3.astype(np.int8), lat)


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _golden_coolchics(names):
    from coolchic_b200._desc import desc_from_header

    out = []
    for n in names:
        for h, nb, lb in _coolchics(_golden(n)):
            out.append((n, desc_from_header(h), nb, lb))
    return out


def _arm_space_names():
    import glob

    return sorted(os.path.basename(p)[:-5] for p in glob.glob(os.path.join(GOLDEN, "arch_space_*.cool")))


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kodim14", "gop5_64x96_yuv420", "img_40x56_rgb_9bit", "gop3_40x56_yuv420_16bit",
                                  "arch_129x7", "arch_40x56_five_layers"] + DENSE + SMALL)
def test_candidates_equal_latent_rate(ctx, name):
    """ccd_rate_candidates equals ccd_latent_rate on the edited integers bit for bit, per grid; its kernel flag equals
    the decoder's plan; two calls are identical; one k_rate_candidates launch per call."""
    from coolchic_b200 import _native

    rng = np.random.default_rng(sum(map(ord, name)))
    for _, d, nb, lb in _golden_coolchics([name]):
        nn = _native.decode_nn(d, nb)
        _, (lat,) = ctx.decode_many([d], [nb], [lb], want_latents=True)
        cands = _draw(d, rng, 24)
        n0 = ctx.launch_count()
        bits, fast = ctx.rate_candidates(d, nn, lat, cands)
        assert ctx.launch_count() - n0 == 1
        bits2, fast2 = ctx.rate_candidates(d, nn, lat, cands)
        assert np.array_equal(bits, bits2) and np.array_equal(fast, fast2)
        edited = []
        for idx, dl in cands:
            e = nn.copy()
            e[idx] += dl
            edited.append(e)
        ref = ctx.latent_rate([d] * (1 + len(cands)), [nn] + edited, [lat] * (1 + len(cands)))
        for j, r in enumerate(ref):
            assert list(bits[j]) == r["grid_bits"], (name, j, cands[j - 1] if j else None)
        assert fast[0] == _fast_plan(d, nn)
        for j, e in enumerate(edited):
            assert fast[j + 1] == _fast_plan(d, e), (name, cands[j])


@pytest.mark.gpu
def test_candidates_arm_space(ctx):
    """Every architecture of the test_arm_space table: a seeded draw priced against ccd_latent_rate."""
    import torch
    from coolchic_b200 import _native
    from test_arm_space import ARCHS, build

    rng = np.random.default_rng(3)
    for arch in ARCHS:
        s = build(arch)
        d, nn = s.desc, np.asarray(s.nn, dtype=np.int64)
        lat = torch.from_numpy(np.asarray(s.lat, dtype=np.int8)).to(ctx.torch_device)
        cands = _draw(d, rng, 6)
        edited = [nn.copy() for _ in cands]
        for e, (idx, dl) in zip(edited, cands):
            e[idx] += dl
        try:
            ref = ctx.latent_rate([d] * (1 + len(cands)), [nn] + edited, [lat] * (1 + len(cands)))
        except _native.CcdError as e:  # a rate pass that does not fit shared memory: pricing refuses it too
            assert e.code == -4  # CCD_ERR_UNSUPPORTED
            with pytest.raises(_native.CcdError):
                ctx.rate_candidates(d, nn, lat, cands)
            continue
        bits, fast = ctx.rate_candidates(d, nn, lat, cands)
        for j, r in enumerate(ref):
            assert list(bits[j]) == r["grid_bits"], (arch, j)


@pytest.mark.gpu
def test_candidate_refusals(ctx, kodim14):
    from coolchic_b200 import _native

    d = kodim14["desc"]
    nn = _native.decode_nn(d, kodim14["nn_bytes"])
    _, (lat,) = ctx.decode_many([d], [kodim14["nn_bytes"]], [kodim14["lat_bytes"]], want_latents=True)
    n_model = _model_span(d)[1]
    bad = [[(n_model, 1)], [(-1, 1)], [(0, 0)], [(0, 1)] * (_native.CCD_CAND_MAX + 1), []]
    for cands in bad:
        n0 = ctx.launch_count()
        with pytest.raises(_native.CcdError) as e:
            ctx.rate_candidates(d, nn, lat, cands)
        assert e.value.code == -1  # CCD_ERR_ARG
        assert ctx.launch_count() == n0


def _decode_all(ctx, data):
    """Frames of a bitstream through decode_video ({display index: FrameData}), and every Cool-chic's latents."""
    import tempfile

    from coolchic_b200.bitstream.decode import decode_video

    with tempfile.TemporaryDirectory() as t:
        p = os.path.join(t, "in.cool")
        open(p, "wb").write(data)
        frames = decode_video(p)
    from coolchic_b200._desc import desc_from_header

    ccs = _coolchics(data)
    descs = [desc_from_header(h) for h, _, _ in ccs]
    _, lats = ctx.decode_many(descs, [nb for _, nb, _ in ccs], [lb for _, _, lb in ccs], want_latents=True)
    return frames, descs, [nb for _, nb, _ in ccs], [lb for _, _, lb in ccs], lats


def _planes(fr):
    d = fr.data
    return [d[k].cpu().numpy() for k in ("y", "u", "v")] if isinstance(d, dict) else [d.cpu().numpy()]


def _check_lossless(ctx, oracle, data, out, rep):
    from coolchic_b200 import _native

    assert len(out) <= len(data) and rep.bytes_after == len(out)
    f0, d0, nb0, lb0, l0 = _decode_all(ctx, data)
    f1, d1, nb1, lb1, l1 = _decode_all(ctx, out)
    assert list(f0) == list(f1)
    for key in f0:
        for x, y in zip(_planes(f0[key]), _planes(f1[key])):
            assert np.array_equal(x, y)
    reps = rep.coolchics
    assert len(reps) == len(d1)
    for i in range(len(d1)):
        assert np.array_equal(l0[i].cpu().numpy(), l1[i].cpu().numpy())
        nn1 = _native.decode_nn(d1[i], nb1[i])
        assert np.array_equal(oracle.decode_latents(d1[i], nn1, lb1[i])[0], l1[i].cpu().numpy())
        bits = sum(ctx.latent_rate([d1[i]], [nn1], [l1[i]])[0]["grid_bits"])
        assert bits == reps[i].latent_bits_after
        nn0 = _native.decode_nn(d0[i], nb0[i])
        assert _fast_plan(d1[i], nn1) == _fast_plan(d0[i], nn0)


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kodim14", "gop5_64x96_yuv420", "gop3_40x56_rgb", "gop3_48x72_yuv420_sinc6",
                                  "gop3_40x56_yuv420_16bit", "gop3_39x57_rgb_13bit", "gop4_40x56_rgb_sinc12"] + DENSE)
def test_optimize_is_lossless(ctx, oracle, name):
    from coolchic_b200.bitstream.optimize import optimize_bitstream

    data = _golden(name)
    out, rep = optimize_bitstream(data, max_rounds=3 if name == "kodim14" else 6)
    _check_lossless(ctx, oracle, data, out, rep)
    again, rep2 = optimize_bitstream(out, max_rounds=2)
    assert len(again) <= len(out)
    _check_lossless(ctx, oracle, out, again, rep2)


@pytest.mark.gpu
def test_optimize_1080p(ctx, oracle, seed_stream):
    from coolchic_b200 import synth
    from coolchic_b200.bitstream.optimize import optimize_bitstream

    data = synth.make_image_stream(ctx, seed_stream, 1080, 1920)
    out, rep = optimize_bitstream(data, max_rounds=2)
    _check_lossless(ctx, oracle, data, out, rep)
