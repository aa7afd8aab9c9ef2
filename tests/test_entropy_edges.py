"""The entropy coder at the edges of its model: crafted ARMs and adversarial latents through every coder path.

Crafted models.  The ARM weight and bias q-steps are 2^-8, so every stabiliser weight integer q adds q * v index units
for a context value v and every bias integer adds one (build_arm: W = q * 2^8, x = v * 2^16, B = q_b * 2^24, output
>> 24; the last layer's o1 bias loses 4 << 8 = 1024 units, subtract_last).  Hidden and output weights are zero, so
(mu_idx, sc_idx) of a symbol is a closed form of its left neighbour (context 0), the one above (context 1) and the
co-located coarser latent (IFCE), clamped to [0, 32767] x [0, 2560]:

  C   constant: the biases alone, mu_idx / sc_idx anywhere on (and beyond) both axes;
  D   mu_idx follows the left neighbour at 3/4 of a symbol per unit, sc_idx the one above (clamping at both ends);
  D2  mu_idx at 2 symbols per unit of the left neighbour (clamps for |v| >= 32);
  DI  mu_idx driven through IFCE by the co-located coarser latent (the fp32 round trip, a floor in the ARM);
  G   D plus one hidden weight of 2^32 (a zero output weight follows it): arm_fits_int32 is false, the generic
      int64 kernel runs on a fast shape.

Adversarial latents are built in coding order, where the mode M = ((mu_idx + 128) >> 8) - 64 of every symbol is known:
P0 all mode; P1 a de Bruijn sequence B(3, 3) over {M-1, M, M+1} (period 28, so that every round alignment sees every
three-symbol hypothesis); P2 P1 with M-14, M+16 (the last window symbols) and M-15, M+17 (the first far ones) at 1/5;
P3 only -64 and 63; P4 uniform over [-64, 63]; P5 runs of 1 ... 12 far symbols between mode runs.  Every symbol is in
exactly one class: mode, near (M +- 1), window (the rest of M-14 ... M+16) or far; the coder's slow count is #far."""
import copy
import os
import re
import subprocess
import sys
import types
from typing import NamedTuple

import numpy as np
import pytest
from conftest import ROOT
from test_progressive import _check_staged
from test_rate import (_check_against_checker, _coding_order, _latent_offsets, _oracle_range_decode, _oracle_scales,
                       model_freq, model_indices)

WIN_HALF = 14  # CCD_WIN_HALF: the window is M - 14 ... M + 16
DEFAULT_MASK = 0x3777

# the shapes of test_gpu_decode.CASES: (H, W), latent_resolution, hyperlatent_resolution
GEOMS = {
    "64x96": ((64, 96), (0, 6), (4, 6)),    # hyperlatents
    "17x33": ((17, 33), (0, 4), None),      # odd sizes
    "129x7": ((129, 7), (0, 3), None),      # w <= 9: raster on every grid
    "40x250": ((40, 250), (0, 6), (4, 6)),  # 1-pixel-high coarse grids
    "256x384": ((256, 384), (0, 6), None),  # steady loop
}
PATTERNS = ["P0", "P1", "P2", "P3", "P4", "P5"]
MU_AXIS = [-200, 0, 127, 128, 16255, 16256, 16384, 16511, 32639, 32640, 32767, 32900]
SC_AXIS = [-50, 0, 1, 1280, 2559, 2560, 2700]


class Model(NamedTuple):
    mu: int = 16384  # mu_idx before context terms and the clamp
    sc: int = 1280
    qm: int = 0      # mu_idx units per unit of the left neighbour
    qs: int = 0      # sc_idx units per unit of the neighbour above
    qi: int = 0      # ARM weight of IFCE feature 0 (mu_idx += floor(qi * feat / 256))
    big: bool = False


MODELS = {
    "smin": Model(16384, 0),
    "smax": Model(16384, 2560),
    "Mlo": Model(0, 1280),        # M = -64: M - 1 is outside the support
    "Mhi": Model(32767, 1280),    # M = 64: the mode itself is outside the support
    "D": Model(16384, 1280, qm=192, qs=40),
}
EXTRA_MODELS = {
    "D2": Model(16384, 0, qm=512, qs=80),
    "DI": Model(16384 + 3, 640, qs=40, qi=100),
    "G": Model(16384, 1280, qm=192, qs=40, big=True),
}
# IFCE of the DI model: weight 48 on channel 0 (the co-located coarser latent v), bias 5; at the sample's IFCE q-steps
# (2^-6, 2^-5) the feature is 40 + 192 v (8 fractional bits)
IFCE_W, IFCE_B = 48, 5


def mode_of(mu_idx, half_down=False):
    return ((np.asarray(mu_idx) + (127 if half_down else 128)) >> 8) - 64


def classes(lat, M, half=WIN_HALF):
    """0 mode, 1 near (M +- 1), 2 window (the rest of M - half ... M + half + 2), 3 far."""
    o = np.asarray(lat, np.int64) - M
    return np.select([o == 0, np.abs(o) == 1, (o >= -half) & (o <= half + 2)], [0, 1, 2], 3)


def _de_bruijn(k, n):
    a, seq = [0] * (k * n), []

    def db(t, p):
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)

    db(1, 1)
    return seq


# offsets -1 / 0 / +1: B(3, 3) starts with 000, so one more 0 in front keeps every window of the cycle; period 28 is prime
# to the 3 symbols of a round, so every alignment of rounds meets all 27 sequences
DB28 = np.array([0] + _de_bruijn(3, 3)) - 1


# ---- crafting --------------------------------------------------------------------------------------------------
def _seed_header():
    from coolchic_b200 import synth

    return synth.parse_single_image(open(synth.SEED_STREAM, "rb").read())[2]


def _overrides(hdr, shape=None):
    q = copy.deepcopy(hdr.get_value("nn_q_step"))
    q.set_value(2.0 ** -8, "arm", "weight")
    q.set_value(2.0 ** -8, "arm", "bias")
    ov = {"nn_q_step": q}
    if shape is not None:
        ov.update(spatial_context_arm=shape[0], output_feature_ifce=shape[1])
    return ov


def craft_nn(d, m: Model):
    from coolchic_b200 import synth

    assert d.qshift[0] == d.qshift[1] == -8 and d.arm_stab and d.arm_hidden >= 1
    sec = {key: {name: np.zeros(shape, np.int64) for name, shape in items} for key, items in synth.nn_sections(d).items()}
    last = sec["arm.bias"][f"mlp.{2 * d.arm_hidden}"]
    last[0] = m.mu - 16384
    last[1] = m.sc - 1280 + 1024  # subtract_last takes 4 << 8 units off o1
    stab = sec["arm.weight"]["stab"]
    stab[0, 0] = m.qm
    stab[1, 1] = m.qs
    if m.qi:
        assert (d.qshift[2], d.qshift[3]) == (-6, -5) and d.n_ifce_out > 0
        stab[0, d.n_ctx] = m.qi
        for name in sec["ifce.weight"]:
            sec["ifce.weight"][name][0, 0] = IFCE_W
            sec["ifce.bias"][name][0] = IFCE_B
    if m.big:
        sec["arm.weight"]["mlp.0"][0, 0] = 1 << 24  # W = 2^32: no int32 operand; |acc| < 2^55 in every layer
    ints, _ = synth.join_nn(d, sec)
    return ints


def pattern_code(name, n, rng):
    """(kind, value) per coding-order position: kind 0 = offset from M, 1 = absolute symbol, 2 = far offset whose
    sign keeps M + value inside [-64, 63]."""
    j = np.arange(n)
    kind, val = np.zeros(n, np.int64), np.zeros(n, np.int64)
    if name in ("P1", "P2"):
        val = DB28[j % 28].copy()
        if name == "P2":
            sel = rng.random(n) < 0.2
            val[sel] = rng.choice([-WIN_HALF, WIN_HALF + 2, -WIN_HALF - 1, WIN_HALF + 3], size=int(sel.sum()))
    elif name == "P3":
        kind[:], val = 1, rng.choice([-64, 63], size=n)
    elif name == "P4":
        kind[:], val = 1, rng.integers(-64, 64, size=n)
    elif name == "P5":
        p, k = 0, 0
        while p < n:
            p += int(rng.integers(1, 7))  # a mode run
            run = k % 12 + 1
            kind[p:p + run] = 2
            val[p:p + run] = WIN_HALF + 3 + rng.integers(0, 24, size=len(kind[p:p + run]))
            p += run
            k += 1
    return kind, val


def _values(kind, val, M):
    far = np.where(M < 32, val, -val)
    return np.where(kind == 1, val, np.clip(M + np.where(kind == 2, far, val), -64, 63))


def craft_latents(d, m: Model, pattern, seed=0):
    """(latents, mu_idx, sc_idx) in decode order: the pattern's symbols, placed in coding order under the model."""
    n = d.n_symbols()
    pos = np.empty(n, np.int64)
    pos[_coding_order(d)] = np.arange(n)
    kind, val = pattern_code(pattern, n, np.random.default_rng(seed))
    offs = _latent_offsets(d)
    lat, mu, sc = (np.zeros(n, np.int64) for _ in range(3))
    grids = {}
    for g in range(d.n_grids - 1, -1, -1):
        h, w = d.grid_h[g], d.grid_w[g]
        sl = slice(offs[g], offs[g] + h * w)
        P = pos[sl].reshape(h, w)
        feat = np.zeros((h, w), np.int64)
        if m.qi and d.flag_ifce and d.grid_ifce_in[g] > 0:
            v = np.zeros((h, w), np.int64)
            if g < d.n_grids - 1:
                v = grids[g + 1][(np.arange(h) >> 1)[:, None], (np.arange(w) >> 1)[None, :]]
            f = (IFCE_B * (1 << (32 + d.qshift[3])) + v * IFCE_W * (1 << (32 + d.qshift[2]))) >> 24
            feat = (m.qi * f) >> 8
        G, Mu = np.zeros((h, w), np.int64), np.zeros((h, w), np.int64)
        for x in range(w):
            left = G[:, x - 1] if x else 0
            Mu[:, x] = np.clip(m.mu + m.qm * left + feat[:, x], 0, 32767)
            G[:, x] = _values(kind[P[:, x]], val[P[:, x]], mode_of(Mu[:, x]))
        above = np.vstack([np.zeros((1, w), np.int64), G[:-1]])
        grids[g] = G
        lat[sl], mu[sl], sc[sl] = G.ravel(), Mu.ravel(), np.clip(m.sc + m.qs * above, 0, 2560).ravel()
    return lat, mu, sc


class Stream(NamedTuple):
    label: str
    desc: object
    nn: np.ndarray
    nb: bytes
    lb: bytes
    lat: np.ndarray
    mu: np.ndarray
    sc: np.ndarray

    @property
    def n_far(self):
        return int((classes(self.lat, mode_of(self.mu)) == 3).sum())


def build_header(geom, shape=None, hw=None, lr=None):
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    hdr = _seed_header()
    g_hw, g_lr, g_hr = GEOMS[geom] if geom else (hw, lr, None)
    ov = _overrides(hdr, shape)
    d = desc_from_header(synth.make_coolchic_header(hdr, g_hw, g_lr, g_hr, None, ov))
    return hdr, (g_hw, g_lr, g_hr), ov, d


def build_stream(backend, geom, model: Model, pattern, seed=0, shape=None, latents=None, hw=None, lr=None):
    """A crafted Cool-chic through synth.make_coolchic (header, exp-Golomb NN payload, range encoder of `backend`).
    The model of every symbol is checked against model_indices unless the latents are given."""
    import torch

    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    hdr, (g_hw, g_lr, g_hr), ov, d0 = build_header(geom, shape, hw, lr)
    nn = craft_nn(d0, model)
    if latents is None:
        lat, mu, sc = craft_latents(d0, model, pattern, seed)
    else:
        lat, mu, sc = latents
    cc, h, _ = synth.make_coolchic(backend, types.SimpleNamespace(header=hdr), g_hw, g_lr, g_hr, overrides=ov,
                                   latents=torch.from_numpy(lat.astype(np.int8)), nn=nn)
    h2 = type(h)()
    rest = h2.read_header(cc)
    d = desc_from_header(h2)
    n_nn, n_lat = h2.get_value("nn_n_bytes"), h2.get_value("n_bytes_latent")
    s = Stream(f"{geom}/{model}/{pattern}/{shape}", d, nn, bytes(rest[:n_nn]), bytes(rest[n_nn:n_nn + n_lat]), lat,
               mu, sc)
    if latents is None:
        mi, si = model_indices(d, nn, lat)
        assert np.array_equal(mi, mu) and np.array_equal(si, sc), s.label
    return s


def _oracle_backend():
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    from pipeline import OracleBackend

    return OracleBackend()


# ---- CPU -------------------------------------------------------------------------------------------------------
def test_crafted_models_hit_their_indices():
    """Every C pair of both axes, D / D2 / DI / G: model_indices agrees with the closed form (build_stream asserts
    it), and the clamps and the half-way tie land where they are meant to."""
    backend = _oracle_backend()
    for mu in MU_AXIS:
        for sc in SC_AXIS:
            s = build_stream(backend, "17x33", Model(mu, sc), "P2", seed=abs(mu) + sc + 100)
            assert (s.mu == min(max(mu, 0), 32767)).all() and (s.sc == min(max(sc, 0), 2560)).all()
    assert mode_of(16256) == 0 and mode_of(16256, half_down=True) == -1  # mu = -0.5: a tie between two modes
    assert mode_of(32640) == 64 and mode_of(127) == -64 and mode_of(128) == -63
    for name, m in {**MODELS, **EXTRA_MODELS}.items():
        s = build_stream(backend, "64x96", m, "P4", seed=1)
        if m.qm or m.qi:
            assert len(np.unique(s.mu)) > 20, name
        if m.qm == 512:
            assert s.mu.min() == 0 and s.mu.max() == 32767  # both clamps reached
        if m.qs:
            assert s.sc.min() == 0 and s.sc.max() == 2560, name


def test_patterns_have_their_design():
    """Class and run-length counts of each pattern under a model whose window lies inside the support."""
    backend = _oracle_backend()
    for pattern in PATTERNS:
        s = build_stream(backend, "64x96", MODELS["smax"], pattern, seed=2)
        order = _coding_order(s.desc)
        M = mode_of(s.mu)
        cls = classes(s.lat, M)[order]
        off = (s.lat - M)[order]
        n = len(order)
        if pattern == "P0":
            assert (cls == 0).all()
        elif pattern == "P1":
            assert set(cls) == {0, 1}
            for a in range(3):  # every round alignment meets all 27 hypotheses
                t = off[a:a + 3 * ((n - a) // 3)].reshape(-1, 3) + 1
                assert len(set((t[:, 0] * 9 + t[:, 1] * 3 + t[:, 2]).tolist())) == 27
        elif pattern == "P2":
            special = np.isin(off, [-14, 16, -15, 17])
            assert abs(special.mean() - 0.2) < 0.02
            assert all((off == o).sum() > 0.03 * n for o in (-14, 16, -15, 17))
            assert (cls == 3).sum() == np.isin(off, [-15, 17]).sum() and (cls[np.isin(off, [-14, 16])] == 2).all()
        elif pattern == "P3":
            assert set(s.lat.tolist()) == {-64, 63}
        elif pattern == "P4":
            assert set(s.lat.tolist()) == set(range(-64, 64))
        elif pattern == "P5":
            far = np.concatenate([[0], (cls == 3).astype(np.int8), [0]])
            starts, ends = np.flatnonzero(np.diff(far) == 1), np.flatnonzero(np.diff(far) == -1)
            runs = ends - starts
            assert set(cls) == {0, 3} and set(runs.tolist()) == set(range(1, 13))
            assert np.array_equal(runs[:24], np.tile(np.arange(1, 13), 2))


@pytest.mark.parametrize("geom", ["64x96", "129x7"])
def test_oracle_round_trip(oracle, geom):
    """Oracle encode -> oracle decode gives the crafted latents back, and its checker model decodes the payload."""
    backend = _oracle_backend()
    for mname, m in {**MODELS, **EXTRA_MODELS}.items():
        for pattern in PATTERNS:
            s = build_stream(backend, geom, m, pattern, seed=3)
            lat, _ = oracle.decode_latents(s.desc, s.nn, s.lb)
            assert np.array_equal(lat, s.lat), s.label
            if pattern == "P2":
                order = _coding_order(s.desc)
                mu = ((s.mu - 16384) / 256.0).astype(np.float32)
                dec = _oracle_range_decode(oracle, s.lb, mu[order], _oracle_scales()[s.sc][order])
                assert np.array_equal(dec, s.lat[order]), s.label


def test_worst_case_payload_fits(oracle):
    """sigma min, every symbol far: freq = 1 of 2^24, at least 24 bits a symbol -- more than 16 bits a symbol."""
    backend = _oracle_backend()
    s = build_stream(backend, "64x96", MODELS["smin"], "P0")  # checks the model
    n = s.desc.n_symbols()
    far = (s.lat * 0 + 20, s.mu, s.sc)  # M = 0: 20 is far
    s = build_stream(backend, "64x96", MODELS["smin"], None, latents=far)
    freq = model_freq(oracle, s.lat, s.mu, s.sc)
    assert (freq == 1).all()
    assert 8 * len(s.lb) >= 24 * n and len(s.lb) <= oracle.payload_cap_bytes(n)
    lat, _ = oracle.decode_latents(s.desc, s.nn, s.lb)
    assert np.array_equal(lat, s.lat)


@pytest.mark.parametrize("bad", [-65, 64])
def test_oracle_refuses_latent_out_of_range(oracle, bad):
    backend = _oracle_backend()
    s = build_stream(backend, "17x33", MODELS["D"], "P2", seed=5)
    lat = s.lat.astype(np.int8)
    lat[321] = bad
    with pytest.raises(oracle.OracleError, match=r"latent 321 is outside \[-64, 63\]"):
        oracle.encode_latents(s.desc, s.nn, lat)


def test_negative_controls_change_the_far_count():
    """The device check (slow count == #far) is sensitive to an off-by-one: restating the classification with a window
    half of 13 or 15, or with M rounded half-down, changes the expected far count of P2 streams."""
    backend = _oracle_backend()
    streams = [build_stream(backend, "64x96", m, "P2", seed=6) for m in (MODELS["smax"], MODELS["D"], Model(16256, 2000))]
    for half in (13, 15):
        for s in streams:
            assert (classes(s.lat, mode_of(s.mu), half) == 3).sum() != s.n_far, (half, s.label)
    tie = streams[-1]
    assert (classes(tie.lat, mode_of(tie.mu, half_down=True)) == 3).sum() != tie.n_far


def test_cdf_table_index_identity(oracle):
    """Entry [sc][f][t] of the cumulative table is lo[-n] (n <= 0) or hi[n] (n > 0) of oracle.laplace_domain at
    n = 256 t - f - 3584: left(s) - (s + 64) of the symbol s = M - 14 + t of any mu_idx with (mu_idx + 128) & 255 = f."""
    rng = np.random.default_rng(7)
    scales = _oracle_scales()
    L = oracle.lib()
    for sc in rng.integers(0, 2561, size=40).tolist() + [0, 2560]:
        lo, hi = oracle.laplace_domain(sc, sc + 1)
        for _ in range(50):
            f, t = int(rng.integers(0, 256)), int(rng.integers(0, 32))
            M = int(rng.integers(-49, 47))  # s = M - 14 + t stays inside (-64, 63]
            mu_idx = 256 * (M + 64) + f - 128
            assert mode_of(mu_idx) == M and (mu_idx + 128) & 255 == f
            s = M - WIN_HALF + t
            n = 256 * t - f - 3584
            want = lo[-n] if n <= 0 else hi[n]
            got = L.cco_laplace_left(s, np.float32((mu_idx - 16384) / 256.0), scales[sc]) - (s + 64)
            assert got == want, (sc, f, t)


# ---- GPU -------------------------------------------------------------------------------------------------------
@pytest.fixture
def masks(ctx):
    """Sets producer masks through the exported debug entry; restores the library default afterwards."""
    try:
        yield ctx.set_producer_mask
    finally:
        ctx.set_producer_mask(DEFAULT_MASK)


def _check_stream(ctx, oracle, masks, s, mask_list=(DEFAULT_MASK, 0x0001, 0x3FFF)):
    import torch

    _, payload, slow = ctx.encode_latents(s.desc, s.nn, latents=torch.from_numpy(s.lat.astype(np.int8)))
    assert payload == s.lb == oracle.encode_latents(s.desc, s.nn, s.lat), s.label
    assert slow == s.n_far, s.label
    lat_o, stats = oracle.decode_latents(s.desc, s.nn, s.lb)
    assert np.array_equal(lat_o, s.lat), s.label
    for mask in mask_list:
        masks(mask)
        _, lats = ctx.decode_many([s.desc], [s.nb], [s.lb], want_latents=True)
        st = ctx.last_status()
        assert np.array_equal(lats[0].cpu().numpy(), s.lat), (s.label, hex(mask))
        assert st[:4] == [0, int(stats[0]), s.n_far, 0], (s.label, hex(mask), st[:4], int(stats[0]), s.n_far)
    masks(DEFAULT_MASK)


@pytest.mark.gpu
def test_status_words_count_like_the_oracle(ctx, oracle, kodim14):
    """Status word [1] (words consumed) and the oracle's stats[0] count the same way, over-read word included."""
    from test_rate import _coolchics, _golden
    from coolchic_b200._desc import desc_from_header

    for name in ["kodim14", "img_48x64_rgb_arm8_1hidden", "arch_129x7", "gop5_64x96_yuv420"]:
        for h, nb, lb in _coolchics(_golden(name)):
            d = desc_from_header(h)
            ctx.decode_many([d], [nb], [lb], want_latents=True)
            _, stats = oracle.decode_latents(d, oracle.decode_nn(d, nb), lb)
            assert ctx.last_status()[:2] == [0, int(stats[0])], name
    assert int(oracle.decode_latents(kodim14["desc"], oracle.decode_nn(kodim14["desc"], kodim14["nn_bytes"]),
                                     kodim14["lat_bytes"])[1][0]) == 7739


@pytest.mark.gpu
@pytest.mark.parametrize("model", list(MODELS))
@pytest.mark.parametrize("geom", list(GEOMS))
def test_adversarial_streams(ctx, oracle, masks, geom, model):
    """Every pattern under the model: device encode == oracle encode, slow count == #far; the decode gives the crafted
    latents with status [0, oracle words consumed, #far, 0] under the default, a one-warp and an all-warp producer
    mask."""
    for pattern in PATTERNS:
        _check_stream(ctx, oracle, masks, build_stream(ctx, geom, MODELS[model], pattern, seed=11))


@pytest.mark.gpu
def test_constant_models_every_index_pair(ctx, oracle, masks):
    """C at every (mu_idx, sc_idx) pair of both axes (clamped and beyond), P2 and P4 latents."""
    for mu in MU_AXIS:
        for sc in SC_AXIS:
            for pattern in ("P2", "P4"):
                _check_stream(ctx, oracle, masks, build_stream(ctx, "17x33", Model(mu, sc), pattern, seed=abs(mu) + sc + 100),
                              mask_list=(DEFAULT_MASK, 0x0001))


@pytest.mark.gpu
def test_worst_case_encode_on_device(ctx, oracle, masks):
    """sigma min, every symbol far: the device encoder's buffer holds 24+ bits a symbol, and the payload decodes."""
    proto = build_stream(ctx, "64x96", MODELS["smin"], "P0")
    s = build_stream(ctx, "64x96", MODELS["smin"], None, latents=(proto.lat * 0 + 20, proto.mu, proto.sc))
    assert 8 * len(s.lb) >= 24 * s.desc.n_symbols() and s.n_far == s.desc.n_symbols()
    _check_stream(ctx, oracle, masks, s)


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [-65, 64])
def test_device_encoder_refuses_latent_out_of_range(ctx, bad):
    import torch

    from coolchic_b200 import _native

    s = build_stream(ctx, "17x33", MODELS["D"], "P2", seed=5)
    lat = torch.from_numpy(s.lat.astype(np.int8))
    lat[321] = bad
    with pytest.raises(_native.CcdError) as e:
        ctx.encode_latents(s.desc, s.nn, latents=lat)
    assert e.value.code == -1 and "latent 321 is outside [-64, 63]" in str(e.value)


@pytest.mark.gpu
@pytest.mark.parametrize("model", ["D2", "DI", "G"])
def test_extra_models(ctx, oracle, masks, model):
    for geom in ("64x96", "40x250", "256x384"):
        for pattern in PATTERNS:
            _check_stream(ctx, oracle, masks, build_stream(ctx, geom, EXTRA_MODELS[model], pattern, seed=12))


@pytest.mark.gpu
def test_result_tags_wrap(ctx, oracle):
    """One constant-model stream of more than 2^22 + 1024 symbols, dense in non-mode symbols around coding index
    2^22, where the helper's 22-bit result tags wrap.  Its classes come from the model's constants."""
    import torch

    hdr, _, _, d = build_header(None, hw=(2048, 2056), lr=(0, 1))
    n = d.n_symbols()
    assert n > (1 << 22) + 1024
    m = Model(16384, 1280)
    kind, val = pattern_code("P2", n, np.random.default_rng(13))
    j = np.arange(n)
    keep = np.abs(j - (1 << 22)) > 40000
    kind[keep], val[keep] = 0, 0
    order = _coding_order(d)
    lat = np.zeros(n, np.int64)
    lat[order] = _values(kind, val, np.zeros(n, np.int64))
    mu, sc = np.full(n, 16384), np.full(n, 1280)
    s = build_stream(ctx, None, m, None, latents=(lat, mu, sc), hw=(2048, 2056), lr=(0, 1))
    n_far = s.n_far
    assert n_far > 1000 and (classes(lat, 0)[order][(1 << 22) - 8:(1 << 22) + 8] != 0).any()
    _, payload, slow = ctx.encode_latents(s.desc, s.nn, latents=torch.from_numpy(lat.astype(np.int8)))
    assert payload == s.lb and slow == n_far
    assert payload == oracle.encode_latents(s.desc, s.nn, lat)
    _, lats = ctx.decode_many([s.desc], [s.nb], [s.lb], want_latents=True)
    st = ctx.last_status()
    lat_o, stats = oracle.decode_latents(s.desc, s.nn, s.lb)
    assert np.array_equal(lat_o, lat) and np.array_equal(lats[0].cpu().numpy(), lat)
    assert st[:3] == [0, int(stats[0]), n_far]


def _batch_streams(ctx, n):
    names = list(MODELS) + ["D2", "DI"]
    allm = {**MODELS, **EXTRA_MODELS}
    return [build_stream(ctx, "17x33", allm[names[i % len(names)]], PATTERNS[i % len(PATTERNS)], seed=100 + i)
            for i in range(n)]


@pytest.mark.gpu
def test_batch_more_streams_than_sms(ctx, masks):
    """2 x SM + 5 adversarial streams of one kernel key in one call (8-warp CTAs), default and one-warp producer
    masks: every stream's latents are its crafted ones, and its output equals its decode alone."""
    import torch

    n = 2 * torch.cuda.get_device_properties(ctx.device).multi_processor_count + 5
    streams = _batch_streams(ctx, n)
    alone = {}
    for i in range(12):
        alone[i] = ctx.decode_many([streams[i].desc], [streams[i].nb], [streams[i].lb])[0][0]
    for mask in (DEFAULT_MASK, 0x0001):
        masks(mask)
        outs, lats = ctx.decode_many([s.desc for s in streams], [s.nb for s in streams], [s.lb for s in streams],
                                     want_latents=True)
        for i, s in enumerate(streams):
            assert np.array_equal(lats[i].cpu().numpy(), s.lat), (i, hex(mask))
        for i, out in alone.items():
            assert torch.equal(outs[i], out), (i, hex(mask))
        st = ctx.last_status()  # the last job's
        assert st[0] == 0 and st[2] == streams[-1].n_far


INSTANCES = [((6, 2), False), ((10, 2), False), ((10, 4), False), ((14, 6), False), ((20, 6), False), ((8, 6), False),
             ((14, 6), True)]


def _instance_stream(ctx, shape, big, pattern="P2"):
    m = EXTRA_MODELS["G"] if big else MODELS["D"]
    return build_stream(ctx, "64x96", m, pattern, seed=14, shape=shape)


def _traced_instances():
    """Run in a fresh process: the k_entropy names of one decode per kernel instance, in a torch.profiler trace."""
    import json
    import time

    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    ctx = _native.get_context(0)
    out = []
    for shape, big in INSTANCES:
        s = _instance_stream(ctx, shape, big)
        ctx.decode_many([s.desc], [s.nb], [s.lb])
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            time.sleep(0.05)
            ctx.decode_many([s.desc], [s.nb], [s.lb])
            torch.cuda.synchronize()
            time.sleep(0.05)
        out.append(sorted({m.group(0) for m in (re.search(r"k_entropy<[^>]*>", e.name) for e in prof.events()) if m}))
    print(json.dumps(out))


@pytest.mark.gpu
def test_every_kernel_instance(ctx, oracle, masks):
    """The five fast instances, generic by shape (8 contexts) and generic by weights (G on the 14 + 6 shape), each on
    P2 and P5 streams; the instance is confirmed from the template arguments of the k_entropy name in a trace."""
    import json

    for shape, big in INSTANCES:
        for pattern in ("P2", "P5"):
            _check_stream(ctx, oracle, masks, _instance_stream(ctx, shape, big, pattern))
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.join(ROOT, 'oracle')!r}, {ROOT!r}]; "
            "import test_entropy_edges; test_entropy_edges._traced_instances()")
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True, cwd=here).stdout
    names = json.loads(r.strip().splitlines()[-1])
    want = [f"k_entropy<{a}, {b}, true>" for (a, b), big in INSTANCES[:5]] + ["k_entropy<0, 0, false>"] * 2
    assert names == [[w] for w in want]


@pytest.mark.gpu
def test_progressive_adversarial(ctx):
    """P2 and P5 streams stopped and resumed at every grid boundary; a stage decodes from its payload prefix."""
    import torch

    from coolchic_b200 import _native
    from coolchic_b200.bitstream.progressive import ProgressiveCoolChic, stage_grid_ends

    for geom, mname in (("64x96", "D"), ("40x250", "smin"), ("17x33", "Mhi")):
        for pattern in ("P2", "P5"):
            s = build_stream(ctx, geom, MODELS[mname], pattern, seed=15)
            d = s.desc
            _check_staged(ctx, d, s.nb, s.lb, None, list(range(1, d.n_grids + 1)), s.label)
            _, offs = _native.latent_layout(d)
            full = ProgressiveCoolChic(ctx, d, s.nb, s.lb)
            for e in stage_grid_ends(d):
                full.decode_to(e)
                done = offs[d.n_grids - e] + d.grid_h[d.n_grids - e] * d.grid_w[d.n_grids - e]
                cut = ProgressiveCoolChic(ctx, d, s.nb, s.lb[:4 * full.words_consumed])
                cut.decode_to(e)
                assert torch.equal(cut.latents[:done], full.latents[:done]), (s.label, e)
                assert cut.words_consumed == full.words_consumed
            assert np.array_equal(full.latents.cpu().numpy(), s.lat)


@pytest.mark.gpu
def test_rate_on_adversarial_streams(ctx, oracle):
    """The rate pass against the checker where its exact f64 branch carries many symbols."""
    for geom, m, pattern in (("64x96", MODELS["D"], "P2"), ("40x250", MODELS["smin"], "P4"),
                             ("64x96", MODELS["Mhi"], "P2"), ("256x384", MODELS["smax"], "P4")):
        s = build_stream(ctx, geom, m, pattern, seed=16)
        r = _check_against_checker(ctx, oracle, s.desc, s.nb, s.lb)
        assert 0 <= 8 * len(s.lb) - sum(r["grid_bits"])


@pytest.mark.gpu
def test_sampling_at_the_edges(ctx, oracle):
    """Mode 2 on C (sigma max, M = -64 and M = 64) and on D: latents and bytes equal oracle.sample_latents, and the
    decode returns them with slow count = #far."""
    for geom, m in (("64x96", Model(0, 2560)), ("64x96", Model(32767, 2560)), ("40x250", MODELS["D"]),
                    ("129x7", MODELS["smax"])):
        _, _, _, d = build_header(geom)
        nn = craft_nn(d, m)
        lat, payload, slow = ctx.encode_latents(d, nn, seed=17)
        lat_o, payload_o = oracle.sample_latents(d, nn, 17)
        lat = lat.cpu().numpy()
        assert np.array_equal(lat, lat_o) and payload == payload_o, m
        mu, _ = model_indices(d, nn, lat)
        n_far = int((classes(lat, mode_of(mu)) == 3).sum())
        assert slow == n_far
        dec = ctx.decode_latents(d, nn, payload)
        assert np.array_equal(dec.cpu().numpy(), lat) and ctx.last_status()[2] == n_far
        if m.sc == 2560:
            assert n_far > 0.25 * lat.size  # sigma max: the slow path carries a large share of the draws


@pytest.mark.gpu
def test_cdf_table_equals_host(ctx, oracle):
    """k_cdf_table, read back through ccd_debug_cdf_table, equals the host image on all 2561 x 256 x 32 entries."""
    f = np.arange(256)[:, None]
    t = np.arange(32)[None, :]
    n = 256 * t - f - 3584
    bad = total = 0
    step = 128
    for sc in range(0, 2561, step):
        hi_sc = min(2561, sc + step)
        dev = ctx.cdf_table(sc, hi_sc)
        lo, hi = oracle.laplace_domain(sc, hi_sc)
        lo, hi = lo.reshape(-1, 32641), hi.reshape(-1, 32641)
        host = np.where(n <= 0, lo[:, np.clip(-n, 0, None)], hi[:, np.clip(n, 0, None)])
        bad += int((dev != host).sum())
        total += dev.size
    assert total == 2561 * 256 * 32 == 20979712 and bad == 0
