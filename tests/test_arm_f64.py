"""The fast ARM on the FP64 tensor cores (DmmaArm in ccd_entropy.cu) and the bound that selects it (arm_fits_f64).

A numpy restatement of the host's fragment-order packing (pack_arm) and of the DMMA m8n8k4 evaluation -- each symbol a
row of the A fragment, lane t of its quad owning the inputs t, t + 4, ..., hidden units permuted so that accumulator
column 8j + 2t + e holds unit 4(2j + e) + t -- equals the int64 ARM (armint.py:180-203) on every ARM of the golden
streams, on random contexts and on contexts at the bound's edge.  The bound accepts the reference's preset shapes; an
ARM whose partial sum reaches 2^53 is refused and runs on the generic int64 kernel, where it decodes like the oracle."""
import glob
import os

import numpy as np
import pytest
from conftest import GOLDEN
from test_entropy_edges import Model, _check_stream, build_header, build_stream, masks  # noqa: F401
from test_rate import _coolchics, _fixed_point
from test_wide_frames import PRESET_ARMS, _arm_desc, seed  # noqa: F401

LIM = 1 << 53
FAST_SHAPES = {(6, 2), (10, 2), (10, 4), (14, 6), (20, 6)}  # ccd_entropy_has_fast
IFCE_FAST_MAX = 12


def arm_ints(d, nn):
    """The ARM integers build_arm makes (W [in][out], B per layer; stabiliser) and the IFCE feature bound (ifce_bound),
    or None for the bound when an IFCE layer is outside the fast path's int32 operands."""
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
    fb, fast_ifce = 0, True
    for name in sec.get("ifce.weight", {}):
        g = int(name[4:])
        n_in = int(d.grid_ifce_in[g])
        Wi, Bi = _fixed_point(sec["ifce.weight"][name], sec["ifce.bias"][name], int(d.qshift[2]), int(d.qshift[3]),
                              np.zeros(n_in, dtype=bool), False)
        Wi, Bi = Wi.astype(object), Bi.astype(object)
        if np.abs(Wi).max(initial=0) > 2**31 - 1 or n_in > IFCE_FAST_MAX:
            fast_ifce = False
            continue
        acc = np.abs(Bi) + (np.abs(Wi) * (64 << 16)).sum(axis=0)
        if max(acc) >= 1 << 62:
            fast_ifce = False
            continue
        f = [(int(a) >> 24) + 1 for a in acc]
        fb = max([fb] + [v + (v >> 22) + 1 for v in f])  # fp32 rounding
    return dict(n_ctx=d.n_ctx, dim=dim, layers=layers, Ws=Ws, Bs=Bs, feat_bound=fb if fast_ifce else None)


def input_bound(a):
    return np.array([64 << 16] * a["n_ctx"] + [a["feat_bound"] << 16] * (a["dim"] - a["n_ctx"]), dtype=object)


def fits_f64(a):
    """arm_fits_f64: every weight, bias and input, every product and partial sum below 2^53, for the worst input."""
    X = input_bound(a)
    if (X >= LIM).any():
        return False

    def layer(W, B, X):
        W, B = np.abs(W.astype(object)), np.abs(B.astype(object))
        if (W >= LIM).any() or (B >= LIM).any():
            return None
        s = B + (W * X[:, None]).sum(axis=0)
        return None if (s >= LIM).any() else s

    stab = layer(a["Ws"], a["Bs"], X)
    if stab is None:
        return False
    for W, B in a["layers"][:-1]:
        s = layer(W, B, X)
        if s is None:
            return False
        X = np.array([int(v) >> 16 for v in s], dtype=object)
    last = layer(*a["layers"][-1], X)
    return last is not None and all(int(v) < LIM for v in last + stab)


def _unit(j, c):
    """The hidden unit in accumulator column c of n-tile j."""
    return 8 * j + 4 * (c & 1) + (c >> 1)


def pack(a, bug=None):
    """pack_arm's fast layout, as arrays: Wh [l][s][j][lane], Bh [l][j][column], Wo [input][wl0, wl1, ws0, ws1].
    ``bug="tile3_perm"`` (a negative control): the fourth n-tile (units 24 ... 31) packed with its column pairs
    swapped."""
    dim, hidden = a["dim"], a["layers"][:-1]

    def unit(j, c):
        return _unit(j, c ^ 1 if bug == "tile3_perm" and j == 3 else c)

    ks = (dim + 3) // 4
    nt = (ks + 1) // 2
    Wh = np.zeros((len(hidden), ks, nt, 32))
    Bh = np.zeros((len(hidden), nt, 8))
    for l, (W, B) in enumerate(hidden):
        for s in range(ks):
            for j in range(nt):
                for lane in range(32):
                    i, o = 4 * s + (lane & 3), unit(j, lane >> 2)
                    Wh[l, s, j, lane] = W[i, o] if i < dim and o < dim else 0
        for j in range(nt):
            for c in range(8):
                Bh[l, j, c] = B[unit(j, c)] if unit(j, c) < dim else 0
    Wo = np.zeros((4 * ks, 4))
    Wo[:dim, :2] = a["layers"][-1][0]
    Wo[:dim, 2:] = a["Ws"]
    return Wh, Bh, Wo


def eval_f64(a, P, X):
    """DmmaArm::run on 8-symbol warps: X [n][dim] int64 inputs (contexts, IFCE features) -> (o0, o1) int64."""
    Wh, Bh, Wo = P
    dim = a["dim"]
    ks, nt = Wh.shape[1], Wh.shape[2]
    n = X.shape[0]
    xin = np.zeros((n, 4 * ks))
    xin[:, :dim] = (X << 16).astype(np.float64)
    x0 = xin.reshape(n, ks, 4)  # A operand of k-step s on lane t: input 4s + t
    xo = x0
    for l in range(Wh.shape[0]):
        acc = np.broadcast_to(Bh[l], (n, nt, 8)).copy()  # C fragment: column c of tile j
        for s in range(ks):
            for j in range(nt):
                B = Wh[l, s, j].reshape(8, 4).T  # B fragment: lane L = 4 column + row
                acc[:, j, :] = xo[:, s, :] @ B + acc[:, j, :]
        h = np.floor(np.maximum(acc, 0.0) * (1.0 / 65536.0))
        # column 2t + e of tile j lands on lane t as its operand of k-step 2j + e
        xo = h.reshape(n, nt, 4, 2).transpose(0, 1, 3, 2).reshape(n, 2 * nt, 4)[:, :ks]
    Wq = Wo.reshape(ks, 4, 4)
    t = [(Wq[None, :, :, o] * xo).sum(axis=1) + (Wq[None, :, :, 2 + o] * x0).sum(axis=1) for o in (0, 1)]
    out = []
    for o in (0, 1):
        p = t[o]
        p = p + p[:, [1, 0, 3, 2]]  # quad butterfly: lane ^ 1, then lane ^ 2
        p = p + p[:, [2, 3, 0, 1]]
        assert (p == p[:, :1]).all()
        Bl, Bs = int(a["layers"][-1][1][o]), int(a["Bs"][o])
        out.append((p[:, 0].astype(np.int64) + Bl + Bs) >> 24)
    return out


def eval_int64(a, X):
    x = X << 16
    s = a["Bs"] + x @ a["Ws"]
    for W, B in a["layers"][:-1]:
        x = np.maximum(B + x @ W, 0) >> 16
    o = (a["layers"][-1][1] + x @ a["layers"][-1][0] + s) >> 24
    return o[:, 0], o[:, 1]


def contexts(a, rng, n=4096):
    """Random inputs, half of them at the bound's edge (every context -64 or 64, every feature +-bound)."""
    nc, nf, fb = a["n_ctx"], a["dim"] - a["n_ctx"], a["feat_bound"]
    C = rng.integers(-64, 64, size=(n, nc))
    F = rng.integers(-fb, fb + 1, size=(n, nf))
    edge = rng.random(n) < 0.5
    C[edge] = rng.choice([-64, 64], size=(int(edge.sum()), nc))
    F[edge] = rng.choice([-fb, fb], size=(int(edge.sum()), nf))
    return np.concatenate([C, F], axis=1).astype(np.int64)


def golden_arms():
    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native
    from coolchic_b200._desc import desc_from_header

    for path in sorted(glob.glob(os.path.join(GOLDEN, "*.cool"))):
        for k, (h, nb, _) in enumerate(_coolchics(open(path, "rb").read())):
            d = desc_from_header(h)
            yield f"{os.path.basename(path)}#{k}", d, _native.decode_nn(d, bytes(nb))


def test_f64_evaluation_equals_int64_on_golden_arms():
    rng = np.random.default_rng(0)
    n_fast = 0
    for label, d, nn in golden_arms():
        a = arm_ints(d, nn)
        cf = d.n_ifce_out if d.flag_ifce else 0
        if (d.n_ctx, cf) not in FAST_SHAPES or a["feat_bound"] is None:
            continue
        assert fits_f64(a), label
        n_fast += 1
        X = contexts(a, rng)
        got, want = eval_f64(a, pack(a), X), eval_int64(a, X)
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), label
    assert n_fast >= 10


@pytest.mark.parametrize("arm", PRESET_ARMS, ids=[f"arm{a}-{b}-ifce{c}" for a, b, c in PRESET_ARMS])
def test_preset_shapes_fit(seed, arm):  # noqa: F811
    d, nn = _arm_desc(seed, arm, 64, 96)
    a = arm_ints(d, nn)
    assert fits_f64(a)
    X = contexts(a, np.random.default_rng(1))
    got, want = eval_f64(a, pack(a), X), eval_int64(a, X)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])


def _stab_arm(q, shape=(14, 6)):
    """A zero ARM but one stabiliser weight q on context 0: its only product reaches q * 2^8 * 64 * 2^16 = q * 2^30."""
    from test_entropy_edges import craft_nn

    d = build_header(None, shape, (64, 96), (0, 6))[3]
    return d, craft_nn(d, Model(qm=q))


def _blob_bytes(d, fast):
    """align16 of the ARM blob plus align16 of the largest IFCE blob, in the fast or the generic layout."""
    a16 = lambda v: (v + 15) & ~15  # noqa: E731
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim, H = d.n_ctx + cf, d.arm_hidden
    if fast:
        ks = (dim + 3) // 4
        nt = (ks + 1) // 2
        arm = 8 * (H * ks * nt * 32 + H * nt * 8 + 16 * ks) + 32
    else:
        arm = 8 * (H * dim * dim + 4 * dim + H * dim) + 32
    ifce = 0
    for g in range(d.n_grids):
        n_in = int(d.grid_ifce_in[g]) if cf else 0
        if n_in:
            w = ((n_in * ((cf + 3) & ~3) * 4 + 7) & ~7) if fast else n_in * cf * 8
            ifce = max(ifce, a16(w + cf * 8))
    return a16(arm) + ifce


def test_bound_refuses_a_partial_sum_of_2_53():
    """q = 2^23: the stabiliser's partial sum is exactly 2^53, the generic layout is planned; one less fits."""
    from coolchic_b200 import _native

    base = {}
    for q in (2**23 - 1, 2**23):
        d, nn = _stab_arm(q)
        a = arm_ints(d, nn)
        assert fits_f64(a) == (q < 2**23)
        ring, rows, smem = _native.entropy_plan(d, nn)
        base[q] = smem - ring * (16 + 32 * 4 + 16 + 4) - rows * 64
    assert base[2**23] - base[2**23 - 1] == _blob_bytes(d, False) - _blob_bytes(d, True)


@pytest.mark.gpu
@pytest.mark.parametrize("q", [2**23 - 1, 2**23])
def test_bound_edge_decodes(ctx, oracle, masks, q):  # noqa: F811
    """Both sides of the bound (the fast kernel, then the generic one) encode and decode like the oracle."""
    from test_entropy_edges import _oracle_backend

    s = build_stream(_oracle_backend(), None, Model(qm=q), "P4", seed=8, shape=(14, 6), hw=(64, 96), lr=(0, 6))
    _check_stream(ctx, oracle, masks, s)
