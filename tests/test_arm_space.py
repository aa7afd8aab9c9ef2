"""The entropy model over every ARM and IFCE the header allows: 0 ... 7 hidden layers (0: a linear ARM), 0 ... 40
spatial contexts, 0 ... 31 IFCE features, IFCE on any sub-range of the grids, hyperlatents below, among and above the
latent grids, 1 ... 31 grids, with and without the linear stabiliser.

Every architecture of ARCHS gets live weights (synth.liven_nn), scaled so that its hidden activations stay bounded
and its (mu_idx, sc_idx) spread over the whole table and past both clamps, and latents tiled from the sample stream
with noise.  The oracle encodes them; its decode, the checker of test_rate (model_indices, numpy int64 with every
partial sum proven below 2^62) driving the oracle's range decoder, and on the GPU the decoder, the encoder (mode 1 and
2), the rate pass, the model-edit pass and a batch of every stream in one call must all agree bit for bit.  Which
k_entropy instance a stream takes follows from a rule restated here (a fast (NCTX, CF) shape, at most 12 IFCE inputs
on every grid, the f64 bound of test_arm_f64) and is pinned against the plan's ARM blob size.

oracle/gen_golden_arm_space.py decoded six extreme architectures with the unmodified reference (tests/golden/
arch_space_*): the checker and the device must reproduce its latents, and four bugs put into the checker pass every
older fixture and fail on these."""
import copy
import glob
import os
import re
import subprocess
import sys
import time
from typing import NamedTuple, Optional, Tuple

import numpy as np
import pytest
from conftest import GOLDEN, ROOT
from test_arm_f64 import FAST_SHAPES, IFCE_FAST_MAX, _blob_bytes, arm_ints, fits_f64
from test_rate import (CHECKER_BUGS, CTX_DX, CTX_DY, _coding_order, _coolchics, _fixed_point, _latent_offsets,
                       _oracle_range_decode, _oracle_scales, model_indices)

SMEM_MAX = 227 * 1024
MU_SPAN, SC_SPAN = 18000, 1500  # index units the 5th / 95th percentiles of (mu, log-scale) are moved to (+-)


class Arch(NamedTuple):
    n_ctx: int
    hidden: int
    cf: int                                # output_feature_ifce
    hw: Tuple[int, int]
    lat: Tuple[int, int] = (0, 6)          # latent_resolution
    hyper: Optional[Tuple[int, int]] = None
    ifce: Optional[Tuple[int, int]] = (0, 2)  # ifce_resolution (cf > 0 only)
    stab: int = 1
    seed: int = 0

    @property
    def label(self):
        s = f"c{self.n_ctx}h{self.hidden}f{self.cf}_{self.hw[0]}x{self.hw[1]}_l{self.lat[0]}-{self.lat[1]}"
        if self.hyper:
            s += f"_y{self.hyper[0]}-{self.hyper[1]}"
        if self.cf:
            s += f"_i{self.ifce[0]}-{self.ifce[1]}"
        return s + ("" if self.stab else "_nostab") + f"_s{self.seed}"


# hand-picked edges of the space
EDGES = [
    Arch(40, 0, 0, (37, 61), (0, 4)),                 # linear, 40 contexts
    Arch(6, 0, 0, (29, 40), (0, 3), stab=0),          # linear without stabiliser: the last layer alone
    Arch(2, 0, 0, (19, 33), (0, 3)),                  # dim 2: the reference folds +I into the square last layer
    Arch(1, 1, 0, (17, 23), (0, 3)),                  # one context
    Arch(1, 0, 1, (23, 30), (0, 4), ifce=(0, 4)),     # dim 2 with an IFCE feature
    Arch(39, 3, 1, (40, 56), (0, 5), ifce=(0, 5)),
    Arch(40, 7, 31, (24, 35), (0, 4), ifce=(0, 4)),   # dim 71, the widest ARM
    Arch(24, 7, 2, (33, 47), (0, 5), stab=0),
    Arch(0, 2, 6, (48, 64), (0, 6), ifce=(0, 6)),     # IFCE only
    Arch(0, 0, 1, (31, 45), (0, 5), ifce=(0, 5)),     # IFCE only, linear, one feature: grid 5 has no context at all
    Arch(8, 1, 31, (40, 56), (0, 6), ifce=(0, 6)),
    Arch(14, 2, 6, (64, 96), (0, 15), ifce=(0, 15)),  # 16 grids, IFCE on all: 15 inputs on the finest, generic
    Arch(20, 2, 6, (64, 96), (0, 13), ifce=(0, 1)),   # 14 grids: 13 and 12 inputs
    Arch(10, 2, 4, (64, 96), (0, 10), ifce=(0, 10)),  # 11 grids, IFCE on all: at most 10 inputs, fast
    Arch(12, 1, 3, (64, 96), (0, 15), (1, 15), ifce=(0, 15)),  # 31 grids (the header's most), 30 IFCE inputs
    Arch(10, 2, 2, (45, 70), (2, 5), (0, 1), ifce=(0, 3)),     # hyperlatents below the latent range
    Arch(12, 2, 3, (50, 70), (0, 5), (1, 3), ifce=(0, 4)),     # hyperlatents among latent grids of the same size
    Arch(9, 3, 2, (40, 56), (0, 3), (4, 6), ifce=(0, 6)),      # hyperlatents above
    Arch(14, 2, 6, (1, 37), (0, 3), ifce=(0, 3)),     # 1 x k: every grid one row, IFCE ratio 0 on all of them
    Arch(25, 1, 0, (61, 1), (0, 3)),                  # k x 1
    Arch(30, 2, 5, (1, 1), (0, 2), ifce=(0, 2)),      # 1 x 1
    Arch(33, 2, 0, (60, 9), (0, 3)),                  # width 9: raster
    Arch(36, 1, 7, (60, 10), (0, 3), ifce=(0, 1)),    # width 10: wavefront
    Arch(40, 3, 0, (60, 11), (0, 3)),                 # width 11
    Arch(28, 2, 0, (20, 96), (0, 4)),                 # 96 wide: the 64-column row ring wraps under dx = +-4
    Arch(5, 4, 4, (33, 41), (0, 4), stab=0),
    Arch(20, 5, 12, (36, 52), (0, 5), ifce=(1, 3)),
    Arch(16, 6, 9, (27, 39), (0, 4), ifce=(2, 4)),
]
# every fast shape with 0, 1, 3 and 7 hidden layers
FAST = [Arch(nc, h, cf, hw, (0, 5), ifce=(0, 3), seed=h)
        for (nc, cf), hw in zip(sorted(FAST_SHAPES), [(40, 56), (9, 64), (64, 96), (33, 47), (50, 61)])
        for h in (0, 1, 3, 7)]


def _random_archs(n, seed=20261017):
    rng = np.random.default_rng(seed)
    out = []
    while len(out) < n:
        n_ctx = int(rng.choice([0, int(rng.integers(1, 6)), int(rng.integers(6, 25)), int(rng.integers(25, 41))]))
        cf = int(rng.choice([0, int(rng.integers(1, 7)), int(rng.integers(7, 32))]))
        if n_ctx + cf == 0:
            continue
        h = int(rng.integers(1, 65))
        w = int(rng.choice([9, 10, 11, int(rng.integers(1, 97))]))
        lo = int(rng.integers(0, 3))
        hi = lo + int(rng.integers(0, 8))
        hyper = None
        if rng.random() < 0.3:  # touching or overlapping the latent range (test_resolution_gap_is_refused)
            a = int(rng.integers(max(0, lo - 3), hi + 2))
            hyper = (a, max(a, lo - 1) + int(rng.integers(0, 4)))
        ifce = None
        if cf:
            top = hi if hyper is None else max(hi, hyper[1])
            a = int(rng.integers(0, top + 1))
            ifce = (a, int(rng.integers(a, top + 1)))
        out.append(Arch(n_ctx, int(rng.integers(0, 8)), cf, (h, w), (lo, hi), hyper, ifce, int(rng.random() < 0.8),
                        seed=len(out) + 100))
    return out


RANDOM = _random_archs(40)
# decoded by the unmodified reference (oracle/gen_golden_arm_space.py -> tests/golden/arch_space_<name>.*)
GOLDEN_ARCHS = {
    "linear_6_2": Arch(6, 0, 2, (40, 56), (0, 5), ifce=(0, 3)),          # the fast 6 + 2 kernel, no hidden layer
    "deep7": Arch(16, 7, 4, (33, 47), (0, 5), ifce=(0, 2)),
    "ctx40": Arch(40, 2, 0, (37, 61), (0, 4)),
    "ifce31": Arch(8, 1, 31, (40, 56), (0, 6), ifce=(0, 6)),
    # up to 15 IFCE inputs beside one spatial context (the reference cannot decode an ARM without spatial context:
    # latent.py:148 reshapes its empty context to [-1, 0])
    "ifce_16grids": Arch(1, 1, 5, (48, 64), (0, 15), ifce=(0, 15)),
    "hyper_interleaved": Arch(12, 2, 3, (50, 70), (0, 5), (1, 3), ifce=(0, 4)),
}
ARCHS = EDGES + FAST + RANDOM
ARCHS += [a for a in GOLDEN_ARCHS.values() if a not in ARCHS]
ARCH_IDS = [a.label for a in ARCHS]


# ---- building -----------------------------------------------------------------------------------------------------
def overrides(a: Arch, template):
    ov = {"spatial_context_arm": a.n_ctx, "n_hidden_layers_arm": a.hidden, "linear_stabiliser_arm": a.stab,
          "output_feature_ifce": a.cf, "ifce_resolution": list(a.ifce) if a.cf else None}
    if a.hidden * (a.n_ctx + a.cf) ** 2 > 8000:
        # the NN payload has 14 bits of byte count: the widest ARMs take the small weights of calibrate() at
        # exp-Golomb order 0
        eg = copy.deepcopy(template.get_value("nn_expgol_cnt"))
        eg.set_value(0, "arm", "weight")
        ov["nn_expgol_cnt"] = eg
    return ov


def arch_header(a: Arch, template):
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    fin = "nearest" if a.lat[0] > 0 else None
    h = synth.make_coolchic_header(template, a.hw, a.lat, a.hyper, fin, overrides(a, template))
    return h, desc_from_header(h)


def _scaled(q, f):
    """Integers q times f, rounded away from zero: no live entry dies."""
    q = np.asarray(q, np.int64)
    v = np.sign(q) * np.maximum(1, np.round(np.abs(q) * f)).astype(np.int64)
    return np.where(q == 0, 0, v)


def _last_inputs(d, sec, latents):
    """The hidden state entering the last layer and the stabiliser's input, [n, dim] each (decode order), as
    test_rate.model_indices computes them."""
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim, H = d.n_ctx + cf, d.arm_hidden
    s_w, s_b = int(d.qshift[0]), int(d.qshift[1])
    ifce_cols = np.arange(dim) >= dim - cf if cf else np.zeros(dim, dtype=bool)
    aw, ab = sec["arm.weight"], sec["arm.bias"]
    offs = _latent_offsets(d)
    lat = np.asarray(latents).astype(np.int64)
    grids = [lat[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]].reshape(d.grid_h[g], d.grid_w[g]) for g in range(d.n_grids)]
    xs, x0s = [], []
    for g in range(d.n_grids):
        h, w = grids[g].shape
        X = np.zeros((h, w, dim), np.int64)
        P = np.pad(grids[g], ((4, 0), (4, 4)))
        for t in range(d.n_ctx):
            X[:, :, t] = P[4 + CTX_DY[t]:4 + CTX_DY[t] + h, 4 + CTX_DX[t]:4 + CTX_DX[t] + w]
        n_in = int(d.grid_ifce_in[g]) if cf else 0
        if n_in:
            Wi, Bi = _fixed_point(sec["ifce.weight"][f"grid{g}"], sec["ifce.bias"][f"grid{g}"], int(d.qshift[2]),
                                  int(d.qshift[3]), np.zeros(n_in, dtype=bool), False)
            yy, xx = np.arange(h) >> 1, np.arange(w) >> 1
            V = np.zeros((h, w, n_in), np.int64)
            sh = 0
            for c in range(n_in if g < d.n_grids - 1 else 0):
                if c > 0 and (d.grid_h[g + c], d.grid_w[g + c]) != (d.grid_h[g + 1 + c], d.grid_w[g + 1 + c]):
                    sh += 1
                V[:, :, c] = grids[g + 1 + c][(yy >> sh)[:, None], (xx >> sh)[None, :]]
            X[:, :, d.n_ctx:] = ((Bi + (V << 16) @ Wi) >> 24).astype(np.float32).astype(np.int64)
        x = X.reshape(h * w, dim) << 16
        x0s.append(x)
        for l in range(H):
            W, B = _fixed_point(aw[f"mlp.{2 * l}"], ab[f"mlp.{2 * l}"], s_w, s_b,
                                ifce_cols if l == 0 else np.zeros(dim, dtype=bool), True)
            x = np.maximum(B + x @ W, 0) >> 16
        xs.append(x)
    return np.concatenate(xs), np.concatenate(x0s)


def calibrate(d, nn, latents):
    """Live weights made usable over the whole space: every hidden weight scaled to |w| <= 1 / dim in value (a hidden
    layer at most doubles its worst-case input, residual included), then each output's weights (last layer and
    stabiliser) scaled and its bias set so that the 5th / 95th percentiles of mu and of the log-scale index land at
    -+MU_SPAN and -+SC_SPAN: both clamps of both axes are reached."""
    from coolchic_b200 import synth

    sec = synth.split_nn(d, nn)
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim, H = d.n_ctx + cf, d.arm_hidden
    s_w, s_b = int(d.qshift[0]), int(d.qshift[1])
    q_max = max(1, (1 << -s_w) // dim)
    for l in range(H):
        w = sec["arm.weight"][f"mlp.{2 * l}"]
        m = np.abs(w).max(initial=0)
        if m > q_max:
            sec["arm.weight"][f"mlp.{2 * l}"] = _scaled(w, q_max / m)
    last, bl = sec["arm.weight"][f"mlp.{2 * H}"], sec["arm.bias"][f"mlp.{2 * H}"]
    x, x0 = _last_inputs(d, sec, latents)
    ifce_last = np.arange(dim) >= dim - cf if (cf and H == 0) else np.zeros(dim, dtype=bool)
    ifce_cols = np.arange(dim) >= dim - cf if cf else np.zeros(dim, dtype=bool)
    for o, span in ((0, MU_SPAN), (1, SC_SPAN)):
        for _ in range(3):  # rounding of the scaled integers: settle in a few passes
            Wl, _ = _fixed_point(last, np.zeros(2), s_w, s_b, ifce_last, True)
            r = (x @ Wl[:, o]).astype(np.float64)
            if d.arm_stab:
                Ws, _ = _fixed_point(sec["arm.weight"]["stab"], np.zeros(2), s_w, s_b, ifce_cols, False)
                r = r + (x0 @ Ws[:, o]).astype(np.float64)
            r /= 2.0**24
            p5, p95 = np.percentile(r, [5, 95]) if r.size else (0.0, 0.0)
            f = 2 * span / max(p95 - p5, 1e-9)
            if 0.8 < f < 1.25 or p95 - p5 < 1e-6:
                break
            f = min(f, 1e4)
            last[o] = _scaled(last[o], f)
            if d.arm_stab:
                sec["arm.weight"]["stab"][o] = _scaled(sec["arm.weight"]["stab"][o], f)
        unit = 2.0 ** (8 + s_b)  # index units of one bias integer
        centre = 0.5 * (p5 + p95) if r.size else 0.0
        b = -centre / unit + (4 << -s_b if o == 1 else 0)
        if d.arm_stab:
            sec["arm.bias"]["stab"][o] = 0
        bl[o] = int(round(b))
    ints, _ = synth.join_nn(d, sec)
    return ints


class Stream(NamedTuple):
    arch: Arch
    desc: object
    nn: np.ndarray
    nb: bytes
    lb: bytes
    lat: np.ndarray
    data: bytes  # the whole single-image bitstream


_CPU = {}


def cpu_seed():
    """(oracle backend, SeedStream decoded by the oracle): the CPU writer of every stream here."""
    if "ss" not in _CPU:
        sys.path.insert(0, os.path.join(ROOT, "oracle"))
        import coolchic_b200  # noqa: F401
        from coolchic_b200 import synth
        from pipeline import OracleBackend

        be = OracleBackend()
        _CPU["be"], _CPU["ss"] = be, synth.SeedStream(be)
    return _CPU["be"], _CPU["ss"]


def build(a: Arch) -> Stream:
    """The architecture's Cool-chic in a 1-frame rgb stream, range-encoded by the oracle (every call: the same bytes)."""
    import torch

    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header
    from coolchic_b200.bitstream.header import FrameHeader, VideoHeader

    if a in _CPU:
        return _CPU[a]
    be, ss = cpu_seed()
    hdr, d = arch_header(a, ss.header)
    rng = np.random.default_rng(a.seed + 7)
    lat = synth.tile_latents(ss.desc, ss.latents, d, a.seed).numpy().astype(np.int64)
    lat = np.clip(lat + rng.integers(-6, 7, size=lat.size), -64, 63)
    nn = calibrate(d, synth.liven_nn(ss.desc, ss.nn, d, a.seed), lat)
    fin = "nearest" if a.lat[0] > 0 else None
    cc, h, _ = synth.make_coolchic(be, ss, a.hw, a.lat, a.hyper, a.seed, fin, overrides=overrides(a, ss.header),
                                   latents=torch.from_numpy(lat.astype(np.int8)), nn=nn)
    h2 = type(h)()
    rest = h2.read_header(cc)
    d = desc_from_header(h2)
    n_nn, n_lat = h2.get_value("nn_n_bytes"), h2.get_value("n_bytes_latent")
    v = VideoHeader()
    v.set_header(1, [0], [])
    f = FrameHeader()
    f._values.update(display_index=0, frame_type="I", frame_data_type="rgb", bitdepth=8, index_references=[],
                     global_flow=[])
    s = Stream(a, d, nn, bytes(rest[:n_nn]), bytes(rest[n_nn:n_nn + n_lat]), lat, v.to_bytes() + f.to_bytes() + cc)
    _CPU[a] = s
    return s


def rule_fast(d, nn):
    """The kernel a stream takes: fast iff its (n_ctx, n_ifce_out) is a fast instance, no grid has more than 12 IFCE
    inputs, every IFCE layer has int32 weights and a bounded feature, and the f64 bound holds."""
    cf = d.n_ifce_out if d.flag_ifce else 0
    if (d.n_ctx, cf) not in FAST_SHAPES:
        return False
    if any(d.grid_ifce_in[g] > IFCE_FAST_MAX for g in range(d.n_grids) if cf):
        return False
    a = arm_ints(d, nn)
    return a["feat_bound"] is not None and fits_f64(a)


def _plan_layout(d, nn):
    """(bytes of the entropy plan beyond its window and row rings, total bytes)."""
    from coolchic_b200 import _native

    ring, rows, smem = _native.entropy_plan(d, nn)
    base = smem - ring * (16 + 32 * 4 + 16 + 4) - rows * 64
    return base, smem


# ---- CPU ----------------------------------------------------------------------------------------------------------
def test_table_covers_the_space():
    """Every hidden-layer count, every band of contexts and of IFCE features, every fast shape at 0 / 1 / 3 / 7 hidden
    layers, hyperlatents on every side of the latent range, both stabiliser settings, the widths around the
    raster / wavefront switch and the IFCE beyond the fast kernel's 12 inputs."""
    assert {a.hidden for a in ARCHS} == set(range(8))
    band = lambda v, edges: next(i for i, e in enumerate(edges) if v <= e)  # noqa: E731
    assert {band(a.n_ctx, (0, 5, 24, 40)) for a in ARCHS} == {0, 1, 2, 3}
    assert {band(a.cf, (0, 6, 31)) for a in ARCHS} == {0, 1, 2}
    assert {a.n_ctx for a in ARCHS} >= {0, 1, 39, 40} and {a.cf for a in ARCHS} >= {1, 31}
    assert {(a.n_ctx, a.cf, a.hidden) for a in FAST} == {(nc, cf, h) for nc, cf in FAST_SHAPES for h in (0, 1, 3, 7)}
    assert len(RANDOM) == 40 and len(set(ARCH_IDS)) == len(ARCHS)
    assert {a.stab for a in ARCHS} == {0, 1}
    assert {a.hw[1] for a in ARCHS} >= {1, 9, 10, 11} and any(a.hw[0] == 1 for a in ARCHS)
    _, ss = cpu_seed()
    sides = set()
    for a in ARCHS:
        if a.hyper:
            sides |= {"below" if a.hyper[0] < a.lat[0] else "", "above" if a.hyper[1] > a.lat[1] else "",
                      "among" if a.hyper[0] <= a.lat[1] and a.hyper[1] >= a.lat[0] else ""}
    assert {"below", "among", "above"} <= sides
    n_in = [max(arch_header(a, ss.header)[1].grid_ifce_in[:32]) for a in ARCHS if a.cf]
    assert max(n_in) == 30 and any(13 <= v <= 16 for v in n_in)


@pytest.mark.parametrize("arch", ARCHS, ids=ARCH_IDS)
def test_arch_on_cpu(oracle, arch):
    """The oracle decodes the stream; the checker's (mu, scale) drive the oracle's range decoder to the same latents;
    the model spans the table; the library plans it within the shared memory a CTA has, in the layout the rule says."""
    from coolchic_b200 import _native

    s = build(arch)
    d = s.desc
    assert np.array_equal(oracle.decode_nn(d, s.nb), s.nn)
    lat, _ = oracle.decode_latents(d, s.nn, s.lb)
    assert np.array_equal(lat, s.lat)
    mu_idx, sc_idx = model_indices(d, s.nn, s.lat)  # asserts that no sum can wrap
    order = _coding_order(d)
    mu = ((mu_idx - 16384) / 256.0).astype(np.float32)
    dec = _oracle_range_decode(oracle, s.lb, mu[order], _oracle_scales()[sc_idx][order])
    assert np.array_equal(dec, s.lat[order].astype(np.int32))
    if d.n_symbols() >= 400 and d.n_ctx > 0:
        assert mu_idx.min() == 0 and mu_idx.max() == 32767 and sc_idx.min() == 0 and sc_idx.max() == 2560
        assert len(np.unique(mu_idx)) > 4 and len(np.unique(sc_idx)) > 4
    if refused(d, s.nn):
        with pytest.raises(_native.CcdError) as e:
            _native.entropy_plan(d, s.nn)
        assert e.value.code == -4 and f"{SMEM_MAX} are available" in str(e.value)
        return
    base, smem = _plan_layout(d, s.nn)
    assert smem <= SMEM_MAX
    # beyond its rings, the plan holds a fixed part and the ARM / IFCE blobs of the layout it chose
    fast = rule_fast(d, s.nn)
    assert base - _blob_bytes(d, fast) == plan_fixed(), (arch.label, fast)
    # (where both layouts have the same size -- 6 + 2 and 10 + 2 -- the trace of test_instances_from_a_trace pins it)


def refused(d, nn):
    """Does the stream need more shared memory than a CTA has, with its ARM and IFCE blobs, the row ring its widest
    grid needs and the smallest (64-slot) window ring?"""
    from test_wide_frames import ROW_BYTES, SLOT_BYTES, _natural

    need = plan_fixed() + _blob_bytes(d, rule_fast(d, nn)) + 64 * SLOT_BYTES + _natural(d)[1] * ROW_BYTES
    return need > SMEM_MAX


def plan_fixed():
    """The plan's bytes beyond its rings and blobs (control words, grid record, spare line), from the sample
    stream's 14 + 6 ARM, which runs on the fast kernel (test_arm_f64)."""
    if "fixed" not in _CPU:
        _, ss = cpu_seed()
        assert rule_fast(ss.desc, ss.nn)
        _CPU["fixed"] = _plan_layout(ss.desc, ss.nn)[0] - _blob_bytes(ss.desc, True)
    return _CPU["fixed"]


def test_resolution_gap_is_refused(oracle):
    """Latent and hyperlatent resolutions with a gap between them (grids 0 and 3 ... 4 here): the IFCE would read the
    coarse grids outside their bounds (the reference cannot decode such a stream either).  With IFCE, the library and
    the oracle refuse it as an argument error; without IFCE nothing reads across grids and it plans."""
    from coolchic_b200 import _native, synth

    _, ss = cpu_seed()
    for cf in (2, 0):
        a = Arch(5, 1, cf, (43, 78), (0, 0), (3, 4), ifce=(2, 4))
        _, d = arch_header(a, ss.header)
        assert [(d.grid_h[g], d.grid_w[g]) for g in range(d.n_grids)] == [(43, 78), (6, 10), (3, 5)]
        nn = synth.liven_nn(ss.desc, ss.nn, d, 1)
        if cf:
            with pytest.raises(_native.CcdError) as e:
                _native.entropy_plan(d, nn)
            assert e.value.code == -1 and "less than half of grid 0" in str(e.value)
            with pytest.raises(oracle.OracleError):
                oracle.sample_latents(d, nn, 1)
        else:
            assert _native.entropy_plan(d, nn)[2] <= SMEM_MAX
            lat, payload = oracle.sample_latents(d, nn, 1)
            assert np.array_equal(oracle.decode_latents(d, nn, payload)[0], lat)


def _fixture(oracle, name):
    from coolchic_b200._desc import desc_from_header

    data = open(os.path.join(GOLDEN, f"arch_space_{name}.cool"), "rb").read()
    (h, nb, lb), = _coolchics(data)
    d = desc_from_header(h)
    return data, d, oracle.decode_nn(d, bytes(nb)), bytes(nb), bytes(lb), \
        np.load(os.path.join(GOLDEN, f"arch_space_{name}.npz"))["latents"]


def _payload_decodes(oracle, d, nn, lb, lat, bug=None):
    """Do the checker's (mu, scale), with ``bug``, drive the oracle's range decoder to ``lat``?"""
    mu_idx, sc_idx = model_indices(d, nn, lat, bug)
    order = _coding_order(d)
    mu = ((mu_idx - 16384) / 256.0).astype(np.float32)
    try:
        dec = _oracle_range_decode(oracle, lb, mu[order], _oracle_scales()[sc_idx][order])
    except AssertionError:  # the decoder met a quantile outside the model
        return False
    return np.array_equal(dec, np.asarray(lat)[order].astype(np.int32))


@pytest.mark.parametrize("name", list(GOLDEN_ARCHS))
def test_reference_fixtures(oracle, name):
    """The reference's latents of each extreme architecture: the oracle decodes them, the checker's model decodes
    the payload to them, and the fixture is what build() writes today."""
    data, d, nn, _, lb, ref = _fixture(oracle, name)
    assert build(GOLDEN_ARCHS[name]).data == data
    assert np.array_equal(oracle.decode_latents(d, nn, lb)[0], ref)
    assert _payload_decodes(oracle, d, nn, lb, ref)


# each bug of the checker (test_rate.CHECKER_BUGS) against the reference fixture that must catch it
BUG_FIXTURES = {"ctx_swap": "ctx40", "ifce_grid": "ifce_16grids", "linear_identity": "linear_6_2",
                "residual_drop": "deep7"}


@pytest.mark.parametrize("bug", CHECKER_BUGS)
def test_checker_negative_controls(oracle, bug):
    """A bug in the checker gives the same model on every older fixture (so it passes all of them) and fails on the
    reference's latents of one new fixture: that fixture is what catches it."""
    from coolchic_b200._desc import desc_from_header

    n_old = 0
    for path in sorted(glob.glob(os.path.join(GOLDEN, "*.cool"))):
        if os.path.basename(path).startswith("arch_space_"):
            continue
        for h, nb, lb in _coolchics(open(path, "rb").read()):
            d = desc_from_header(h)
            nn = oracle.decode_nn(d, bytes(nb))
            lat, _ = oracle.decode_latents(d, nn, bytes(lb))
            for got, want in zip(model_indices(d, nn, lat, bug), model_indices(d, nn, lat)):
                assert np.array_equal(got, want), (bug, path)
            n_old += 1
    assert n_old > 40
    _, d, nn, _, lb, ref = _fixture(oracle, BUG_FIXTURES[bug])
    assert _payload_decodes(oracle, d, nn, lb, ref) and not _payload_decodes(oracle, d, nn, lb, ref, bug)


# ---- GPU ----------------------------------------------------------------------------------------------------------
def _instance(d, nn):
    cf = d.n_ifce_out if d.flag_ifce else 0
    return f"k_entropy<{d.n_ctx}, {cf}, true>" if rule_fast(d, nn) else "k_entropy<0, 0, false>"


@pytest.mark.gpu
@pytest.mark.parametrize("arch", ARCHS, ids=ARCH_IDS)
def test_arch_on_device(ctx, oracle, arch):
    """Decoder, rate pass (mu_idx, sc_idx), encoder in mode 1 and 2 and the model edits of every single input, bit for
    bit against the oracle and the checker; an architecture the plan refuses is refused before any launch."""
    import torch

    from coolchic_b200 import _native
    from test_model import variant_indices

    s = build(arch)
    d, nn = s.desc, s.nn
    lat_t = torch.from_numpy(s.lat.astype(np.int8))
    if refused(d, nn):
        for call in (lambda: ctx.decode_many([d], [s.nb], [s.lb]), lambda: ctx.encode_latents(d, nn, latents=lat_t),
                     lambda: ctx.latent_rate([d], [nn], [lat_t.cuda()])):
            n0 = ctx.launch_count()
            with pytest.raises(_native.CcdError) as e:
                call()
            assert e.value.code == -4 and ctx.launch_count() == n0
        return
    _, lats = ctx.decode_many([d], [s.nb], [s.lb], want_latents=True)
    assert ctx.last_status()[0] == 0
    assert np.array_equal(lats[0].cpu().numpy(), s.lat)
    cf = d.n_ifce_out if d.flag_ifce else 0
    edits = [(0, 0, 0)] + [(1 << t, 0, 0) for t in range(d.n_ctx)] + [(0, 1 << c, 0) for c in range(cf)]
    res = ctx.latent_rate([d] * len(edits), [nn] * len(edits), [lats[0]] * len(edits), want_mu_sc=True, edits=edits)
    for e, r in zip(edits, res):
        mu, sc = model_indices(d, nn, s.lat) if e == (0, 0, 0) else variant_indices(d, nn, s.lat, *e)
        ms = r["mu_sc"].cpu().numpy().view(np.uint32)
        assert np.array_equal((ms & 0xFFFF).astype(np.int64), mu), e
        assert np.array_equal((ms >> 16).astype(np.int64), sc), e
    plain = ctx.latent_rate([d], [nn], [lats[0]], want_mu_sc=True)[0]
    assert torch.equal(plain["mu_sc"], res[0]["mu_sc"])
    _, payload, _ = ctx.encode_latents(d, nn, latents=lat_t)
    assert payload == s.lb
    lat2, pay2, _ = ctx.encode_latents(d, nn, seed=arch.seed + 1)
    lat_o, pay_o = oracle.sample_latents(d, nn, arch.seed + 1)
    assert np.array_equal(lat2.cpu().numpy(), lat_o) and pay2 == pay_o
    assert np.array_equal(ctx.decode_latents(d, nn, pay2).cpu().numpy(), lat_o)


@pytest.mark.gpu
def test_batch_of_every_stream(ctx):
    """Every stream the decoder takes, cycled to 2 x SM + 5 jobs, in one decode_many call (8-warp CTAs): every job's
    latents are its own and its output equals its decode alone."""
    import torch

    streams = [build(a) for a in ARCHS]
    streams = [s for s in streams if not refused(s.desc, s.nn)]
    n = 2 * torch.cuda.get_device_properties(ctx.device).multi_processor_count + 5
    items = [streams[i % len(streams)] for i in range(n)]
    outs, lats = ctx.decode_many([s.desc for s in items], [s.nb for s in items], [s.lb for s in items],
                                 want_latents=True)
    for i, s in enumerate(items):
        assert np.array_equal(lats[i].cpu().numpy(), s.lat), s.arch.label
    for i, s in enumerate(streams):
        alone = ctx.decode_many([s.desc], [s.nb], [s.lb])[0][0]
        assert torch.equal(outs[i], alone), s.arch.label


def _traced_instances():
    """Run in a fresh process: the k_entropy instance of one decode of every stream, in order, from one trace."""
    import json

    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    ctx = _native.get_context(0)
    streams = [s for s in (build(a) for a in ARCHS) if not refused(s.desc, s.nn)]
    ctx.decode_many([streams[0].desc], [streams[0].nb], [streams[0].lb])
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for s in streams:
            ctx.decode_many([s.desc], [s.nb], [s.lb])
            torch.cuda.synchronize()
    ev = sorted((e.time_range.start, m.group(0)) for e in prof.events()
                for m in [re.search(r"k_entropy<[^>]*>", e.name)] if m)
    print(json.dumps([name for _, name in ev]))


@pytest.mark.gpu
def test_instances_from_a_trace(ctx):
    """The k_entropy instance each stream launched, read from a kernel trace, is the one the rule gives; the set
    covers the generic kernel and all five fast instances."""
    import json

    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.join(ROOT, 'oracle')!r}, {ROOT!r}]; "
            "import test_arm_space; test_arm_space._traced_instances()")
    t0 = time.time()
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, check=True, cwd=here).stdout
    names = json.loads(r.strip().splitlines()[-1])
    want = [_instance(s.desc, s.nn) for s in (build(a) for a in ARCHS) if not refused(s.desc, s.nn)]
    assert names == want
    assert set(want) == {"k_entropy<0, 0, false>"} | {f"k_entropy<{a}, {b}, true>" for a, b in FAST_SHAPES}
    print(f"{len(names)} traced decodes in {time.time() - t0:.1f} s")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(GOLDEN_ARCHS))
def test_reference_fixtures_on_device(ctx, oracle, name):
    """The device decodes the reference's latents of every extreme architecture, and its rate pass gives the
    checker's (mu_idx, sc_idx) on them."""
    _, d, nn, nb, lb, ref = _fixture(oracle, name)
    _, lats = ctx.decode_many([d], [nb], [lb], want_latents=True)
    assert np.array_equal(lats[0].cpu().numpy(), ref)
    ms = ctx.latent_rate([d], [nn], [lats[0]], want_mu_sc=True)[0]["mu_sc"].cpu().numpy().view(np.uint32)
    mu, sc = model_indices(d, nn, ref)
    assert np.array_equal((ms & 0xFFFF).astype(np.int64), mu) and np.array_equal((ms >> 16).astype(np.int64), sc)
