"""The float side (upsampling cascade, synthesis, common randomness, final resize, frame tail, P/B warp and blend)
against an independent float64 restatement of the reference, at every architecture and edge shape the decoder
accepts.

The oracle and the kernels follow one canonical fp32 order, and the rest of the suite checks them against each
other bit for bit.  This file checks that the order computes the reference's function.  The restatement below is
written from the reference's PyTorch modules (file:line cited at each step), in float64 with CPU torch ops; it uses
neither the oracle's float code nor the kernels.

Each step runs three passes at once (class ``T``): the value; the magnitude pass (|weights|, |biases|, |inputs|, ReLU
as the identity, no clamp), which gives per sample A = sum |w x| propagated through the network; and the absolute
error of coefficients computed in fp32 from a coordinate (resize and grid-sample taps), propagated the same way.
``T.k`` counts the fp32 roundings along the longest accumulation path, stage by stage, so an fp32 implementation of
the same function is within ``k * 2^-24 * A + e`` of the float64 value to first order.  The negative controls show
the bound is tight enough to catch an off-by-one.

Integer samples after the frame tail must equal the rounding of the float64 value, except where that value is within
the bound of a rounding tie; those are counted and printed.
"""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from conftest import GOLDEN

U = 2.0**-24
MODULES = ("arm", "ifce", "upsampling", "synthesis")  # core/types.py:98-101, the bitstream order
KINDS = ("weight", "bias")                            # core/types.py:18-19


# ------------------------------------------------------------------------------------------------------------------
# value, magnitude and coefficient-error passes
class T:
    """A float64 tensor ``v`` with its magnitude pass ``m``, the absolute coefficient error ``e`` propagated to it,
    and ``k``, the fp32 roundings along the longest accumulation path that produced it."""

    def __init__(self, v, m=None, e=None, k=0):
        self.v = v
        self.m = v.abs() if m is None else m
        self.e = torch.zeros_like(v) if e is None else e
        self.k = k

    def map(self, f):  # a structural step (crop, pad, reshape): no rounding
        return T(f(self.v), f(self.m), f(self.e), self.k)

    def bound(self):
        return self.k * U * self.m + self.e


def _cat(a, b):
    return T(torch.cat([a.v, b.v], 1), torch.cat([a.m, b.m], 1), torch.cat([a.e, b.e], 1), max(a.k, b.k))


def _add(a, b):
    return T(a.v + b.v, a.m + b.m, a.e + b.e, max(a.k, b.k) + 1)


def _lin(x, f, w, b, n):
    """A linear step y = f(x, w, b) of n terms per output: the value, then |w| on the magnitude and error passes."""
    return T(f(x.v, w, b), f(x.m, w.abs(), None if b is None else b.abs()), f(x.e, w.abs(), None), x.k + n)


# ------------------------------------------------------------------------------------------------------------------
# NN parameters
def nn_layout(p):
    """[(module, kind, name, shape)] in the reference's get_param order: module order, then weights / biases, then
    named parameters (bitstream/neuralnet/neuralnet.py:121-148, 155-201)."""
    mods = {m: [] for m in MODULES}
    dim, cf = p.total_context_arm, p.output_feature_ifce
    # arm.py:176-195: n hidden ArmLinear(dim, dim) + ReLU, ArmLinear(dim, 2), the stabiliser ArmLinear(dim, 2)
    for i in range(p.n_hidden_layers_arm):
        mods["arm"].append((f"mlp.{2 * i}", (dim, dim), (dim,)))
    mods["arm"].append((f"mlp.{2 * p.n_hidden_layers_arm}", (2, dim), (2,)))
    if p.linear_stabiliser_arm:
        mods["arm"].append(("stabiliser_branch", (2, dim), (2,)))
    # arm.py:336-350: one Arm(nin, 0 hidden layers, cf outputs, no stabiliser) per grid with an IFCE
    if p.flag_ifce:
        j = 0
        for nin in p.input_features_ifce:
            if nin:
                mods["ifce"].append((f"arms.{j}.mlp.0", (cf, nin), (cf,)))
                j += 1
    # coolchic.py:1081-1089, upsampling.py:451-461: latent_resolution[1] kernels of each kind; the parametrised weight
    # is the (k + 1) // 2 vector of upsampling.py:66-85
    n = p.latent_resolution[1]
    mods["upsampling"] = ([(f"conv_transpose2ds.{i}", ((p.ups_k_size + 1) // 2,), (1,)) for i in range(n)]
                          + [(f"conv2ds.{i}", ((p.ups_preconcat_k_size + 1) // 2,), (1,)) for i in range(n)])
    # synthesis.py:197-241: output_transform, stabiliser_branch, then main_branch (a layer every other module)
    layers = p.parsed_synthesis_layers()
    C, cin = layers[-1][0], p.input_feature_synthesis
    mods["synthesis"].append(("output_transform", (C, C, 1, 1), (C,)))
    if p.linear_stabiliser_synth:
        ns = cin // 2 if p.flag_common_randomness else cin
        mods["synthesis"].append(("stabiliser_branch", (C, ns, 1, 1), (C,)))
    for i, (o, k, _, _) in enumerate(layers):
        mods["synthesis"].append((f"main_branch.{2 * i}", (o, cin, k, k), (o,)))
        cin = o
    return [(m, kind, name, ws if kind == "weight" else bs) for m in MODULES for kind in KINDS
            for name, ws, bs in mods[m]]


def dequantise(header, ints):
    """{(module, name, kind): float64 tensor}: int * q_step (neuralnet.py:184-188)."""
    p = header.get_coolchic_parameter()
    q = header.get_value("nn_q_step")
    out, pos = {}, 0
    for m, kind, name, shape in nn_layout(p):
        n = int(np.prod(shape))
        out[(m, name, kind)] = torch.from_numpy(np.asarray(ints[pos:pos + n], dtype=np.float64)).view(shape) * float(
            q.get_value(m, kind))
        pos += n
    assert pos == len(ints), (pos, len(ints))
    return out


# ------------------------------------------------------------------------------------------------------------------
# upsampling (upsampling.py)
def _sym(par, k, bug=None):
    """upsampling.py:53-64: a b c -> a b c b a (odd k) or a b c c b a (even k)."""
    if bug == "even_preconcat" and k % 2:
        return torch.cat([par, par.flip(0)])
    return torch.cat([par, par.flip(0)[k % 2:]])


def _per_channel(t, f):
    c = t.shape[1]
    y = f(t.reshape(-1, 1, *t.shape[-2:]))
    return y.reshape(1, c, *y.shape[-2:])


def _convt(x, w1):
    """upsampling.py:306-325 (train mode): kron 2-D kernel, replicate padding by k // 2, stride-2 transposed conv,
    crop of C on each side.  (k / 2)^2 products of fp32 kernel entries per output."""
    k = w1.numel()
    p0 = k // 2
    c = 2 * p0 - 1 + k // 2
    ker = torch.kron(w1.view(1, -1), w1.view(-1, 1)).view(1, 1, k, k)

    def f(t, w, b):
        def g(z):
            y = F.conv_transpose2d(F.pad(z, (p0, p0, p0, p0), mode="replicate"), w, stride=2)
            return y[..., c:y.shape[-2] - c, c:y.shape[-1] - c]
        return _per_channel(t, g)

    return _lin(x, f, ker, None, (k // 2) ** 2 + 2)


def _preconcat(x, w1):
    """upsampling.py:180-196 (train mode): kron 2-D kernel, zero padding by k // 2, plus the input."""
    k = w1.numel()
    ker = torch.kron(w1.view(1, -1), w1.view(-1, 1)).view(1, 1, k, k)
    h, w = x.v.shape[-2:]

    def f(t, wt, b):
        return _per_channel(t, lambda z: F.conv2d(z, wt, padding=k // 2)[..., :h, :w])

    return _add(_lin(x, f, ker, None, k * k + 1), x)


def upsampling(p, P, coded, bug=None):
    """upsampling.py:463-500: from the coarsest grid, upsample, crop to the next grid, filter that grid, concatenate."""
    n = p.latent_resolution[1]
    rev = [T(t) for t in reversed(coded)]
    up = rev[0]
    for idx, tgt in enumerate(rev[1:]):
        if tgt.v.shape[1] == 0:
            break
        x = _convt(up, _sym(P[("upsampling", f"conv_transpose2ds.{idx % n}", "weight")], p.ups_k_size))
        th, tw = tgt.v.shape[-2:]
        if bug == "crop_shift" and idx == len(rev) - 2:
            x = x.map(lambda t: F.pad(t, (0, 1, 0, 1), mode="replicate")[..., 1:th + 1, 1:tw + 1])
        else:
            x = x.map(lambda t: t[..., :th, :tw])
        hb = _preconcat(tgt, _sym(P[("upsampling", f"conv2ds.{idx % n}", "weight")], p.ups_preconcat_k_size, bug))
        up = _cat(hb, x)
    return up


# ------------------------------------------------------------------------------------------------------------------
# F.interpolate(align_corners=False) along one axis, with the fp32 coefficient and coordinate errors
A_CUBIC = -0.75


def _cc1(x):
    return ((A_CUBIC + 2) * x - (A_CUBIC + 3)) * x * x + 1


def _cc2(x):
    return ((A_CUBIC * x - 5 * A_CUBIC) * x + 8 * A_CUBIC) * x - 4 * A_CUBIC


def _dcc1(x):
    return 3 * (A_CUBIC + 2) * x * x - 2 * (A_CUBIC + 3) * x


def _dcc2(x):
    return 3 * A_CUBIC * x * x - 10 * A_CUBIC * x + 8 * A_CUBIC


def _cubic_taps(t):
    """Keys coefficients of the four taps at floor(x) - 1 .. + 2 for the fraction t, and |d coefficient / dt|."""
    c = [_cc2(t + 1), _cc1(t), _cc1(1 - t), _cc2(2 - t)]
    d = [abs(_dcc2(t + 1)), abs(_dcc1(t)), abs(_dcc1(1 - t)), abs(_dcc2(2 - t))]
    return c, d


# |fp32 error of one coefficient| / 2^-24.  Resize and grid-sample coefficients are polynomials of the fraction; a sinc
# tap rounds its argument s - k and pi (s - k) before sin / cos, which leaves an absolute error even where the exact
# coefficient is 0 (an integer flow: torch.sinc(-k) in fp32 is about 2.8e-8, not 0)
KAPPA = {"bilinear": 4, "bicubic": 64, "sinc": 8}


def _axis(n_in, n_out, mode, scale):
    """Coefficient matrix R, |derivative| matrix D, tap-count matrix N and the source coordinate of every output."""
    R, D, N = (np.zeros((n_out, n_in)) for _ in range(3))
    src = np.zeros(n_out)
    for o in range(n_out):
        real = scale * (o + 0.5) - 0.5
        if mode == "bilinear":
            real = max(real, 0.0)
            x0 = int(real)
            l1 = real - x0
            x1 = x0 + (1 if x0 < n_in - 1 else 0)
            for i, c in ((x0, 1 - l1), (x1, l1)):
                R[o, i] += c
                D[o, i] += 1
                N[o, i] += 1
        else:
            x0 = math.floor(real)
            c, d = _cubic_taps(real - x0)
            for j in range(4):
                i = min(max(x0 - 1 + j, 0), n_in - 1)
                R[o, i] += c[j]
                D[o, i] += d[j]
                N[o, i] += 1
        src[o] = abs(real)
    return [torch.from_numpy(a) for a in (R, D, N, src)]


def _resize_axis(x, n_out, mode, axis, scale):
    n_in = x.v.shape[axis]
    R, D, N, src = _axis(n_in, n_out, mode, n_in / n_out if scale is None else scale)
    eq = "oi,bcix->bcox" if axis == 2 else "oi,bcxi->bcxo"
    ap = lambda M, t: torch.einsum(eq, M, t)  # noqa: E731
    # coefficient error: kappa per coefficient, plus the coordinate's own fp32 error (4 roundings of |src| + 1) times
    # the coefficient's derivative
    sh = (1, 1, -1, 1) if axis == 2 else (1, 1, 1, -1)
    e = ap(R.abs(), x.e) + U * (KAPPA[mode] * ap(N, x.m) + (4 * (src + 1)).view(sh) * ap(D, x.m))
    return T(ap(R, x.v), ap(R.abs(), x.m), e, x.k + (2 if mode == "bilinear" else 4) + 2)


def resize(x, size=None, mode="bicubic", scale_factor=None):
    """F.interpolate(x, size | scale_factor, mode, align_corners=False) restated (UpSample.h: source index
    scale * (dst + 0.5) - 0.5, clamped at 0 for bilinear; Keys cubic, A = -0.75, taps clamped to the border)."""
    if mode == "nearest":
        f = lambda t: F.interpolate(t, size=size, mode="nearest")  # noqa: E731  (an index gather: exact)
        return x.map(f)
    H, W = (x.v.shape[-2] * 2, x.v.shape[-1] * 2) if scale_factor else size
    s = 1.0 / scale_factor if scale_factor else None
    y = _resize_axis(_resize_axis(x, W, mode, 3, s), H, mode, 2, s)
    want = F.interpolate(x.v, scale_factor=scale_factor, mode=mode) if scale_factor else F.interpolate(
        x.v, size=size, mode=mode)
    assert torch.allclose(y.v, want, rtol=0, atol=1e-12 * (1 + float(x.m.max())))  # the restatement, checked
    return y


# ------------------------------------------------------------------------------------------------------------------
# synthesis (synthesis.py) and the intra path (bitstream/component/coolchic.py:174-192)
def _syn_conv(x, w, b):
    """synthesis.py:61-76 without the residual: replicate padding by (k - 1) / 2, conv2d with bias."""
    k = w.shape[-1]
    pd = (k - 1) // 2

    def f(t, wt, bt):
        return F.conv2d(F.pad(t, (pd, pd, pd, pd), mode="replicate"), wt, bt)

    return _lin(x, f, w, b, w.shape[1] * k * k + 2)


def synthesis(p, P, x, bug=None):
    """synthesis.py:272-294."""
    h = x
    for i, (_, _, res, relu) in enumerate(p.parsed_synthesis_layers()):
        y = _syn_conv(h, P[("synthesis", f"main_branch.{2 * i}", "weight")],
                      P[("synthesis", f"main_branch.{2 * i}", "bias")])
        if res:
            y = _add(y, h)  # synthesis.py:73-74: the residual adds the layer's input, before the non-linearity
        if relu:
            y = T(torch.relu(y.v), y.m, y.e, y.k)
        h = y
    if p.linear_stabiliser_synth:
        ws = P[("synthesis", "stabiliser_branch", "weight")]
        ns = ws.shape[1]  # n_input_ft_stabiliser: half the inputs under common randomness (synthesis.py:205-208)
        if bug == "stab_all":
            ws, ns = torch.cat([ws] * (x.v.shape[1] // ns), 1), x.v.shape[1]
        s = _syn_conv(x.map(lambda t: t[:, :ns]), ws, P[("synthesis", "stabiliser_branch", "bias")])
        h = _add(h, s)
    return _syn_conv(h, P[("synthesis", "output_transform", "weight")], P[("synthesis", "output_transform", "bias")])


def cr_noise(p):
    """noise.py:18-55 (Park-Miller LCG, Box-Muller with pi = 3.14159265359, kept in fp32 by the reference), one grid
    per latent resolution (coolchic.py:187-191), then fixed_upsampling (upsampling.py:556-595) and the bicubic resize
    to the image size (bitstream/component/coolchic.py:179-183)."""
    seed, m, grids = 18101995, 2**31 - 1, []
    for i in range(p.latent_resolution[0], p.latent_resolution[1] + 1):
        h, w = [int(math.ceil(s / 2**i)) for s in p.img_size]
        vals = []
        for _ in range(h * w):
            seed = (16807 * seed) % m
            u1 = seed / m
            seed = (16807 * seed) % m
            u2 = seed / m
            vals.append(math.sqrt(-2 * math.log(u1)) * math.cos(2 * 3.14159265359 * u2))
        grids.append(torch.tensor(vals, dtype=torch.float32).to(torch.float64).view(1, 1, h, w))
    rev = [T(g) for g in reversed(grids)]
    up = rev[0]
    for tgt in rev[1:]:
        if up.v.shape[2:] != tgt.v.shape[2:]:
            th, tw = tgt.v.shape[-2:]
            x = resize(up, mode="bicubic", scale_factor=2.0).map(lambda t: t[..., :th, :tw])
        else:
            x = up
        up = _cat(tgt, x)
    if tuple(up.v.shape[-2:]) != tuple(p.img_size):
        up = resize(up, size=tuple(p.img_size), mode="bicubic")
    return up


def latent_grids(p, lat):
    """The decoded latents, grid n - 1 first (coolchic.py:89), as [1, 1, h, w] float64 grids, grid 0 first."""
    grids, off = [None] * p.n_latent_grids, 0
    for g in range(p.n_latent_grids - 1, -1, -1):
        h, w = p.size_per_latent[g][-2:]
        grids[g] = torch.from_numpy(np.asarray(lat[off:off + h * w], dtype=np.float64)).view(1, 1, h, w)
        off += h * w
    assert off == len(lat)
    return grids


def intra(header, ints, lat, bug=None):
    """encode_decode_coolchic's float side (bitstream/component/coolchic.py:174-192): [C, H, W] as T."""
    p = header.get_coolchic_parameter()
    P = dequantise(header, ints)
    grids = latent_grids(p, lat)
    coded = [g for g, hyp in zip(grids, p.flag_is_hyperlatent) if not hyp]
    x = upsampling(p, P, coded, bug)
    if p.flag_common_randomness:
        x = _cat(x, cr_noise(p))
    y = synthesis(p, P, x, bug)
    H, W = p.img_size
    if tuple(y.v.shape[-2:]) != (H, W):
        y = resize(y, size=(H, W), mode=p.final_upsampling_type)
    return y.map(lambda t: t[0, :, :H, :W])


# ------------------------------------------------------------------------------------------------------------------
# P / B prediction (bitstream/decode.py:156-189)
def global_shift(ref, g):
    """globalmotion.py:151-160: vanilla_warp_fn nearest / border with a constant integer flow (g[0] horizontal)."""
    _, h, w = ref.shape
    ys = torch.clamp(torch.arange(h) + int(g[1]), 0, h - 1)
    xs = torch.clamp(torch.arange(w) + int(g[0]), 0, w - 1)
    return ref[:, ys][:, :, xs]


def _warp_axis(q, n, pos, fs, bug=None):
    """Taps of one axis: (index, coefficient, absolute fp32 coefficient error / 2^-24) per tap, each [H, W]."""
    taps = []
    if fs > 4:  # warp.py:346-397 and 226-243: integer part by clamped gathers, windowed sinc of the fraction
        fl = torch.floor(q)
        s = q - fl
        for kk in range(-fs // 2 + 1, fs // 2 + 1):
            win = kk + 1 if bug == "sinc_shift" else kk
            c = torch.cos(math.pi * (s - win) / fs) * torch.sinc(s - kk)
            taps.append((torch.clamp(pos + fl + kk, 0, n - 1).long(), c, c.abs() + KAPPA["sinc"]))
        return taps
    # warp.py:324-343: grid_sample(align_corners=True, border) on the exact coordinate pos + q.  The reference's fp32
    # coordinate ((linspace + q / ((n - 1) / 2)) + 1) / 2 * (n - 1) is off by delta / 2^-24: the linspace entry's and
    # the three operations' roundings, scaled by (n - 1) / 2, and the product's own
    ix = pos + q
    delta = 2 * (n - 1) + 2 * q.abs() + ix.abs() + 2
    if fs == 2:  # bilinear: the coordinate is clipped first (GridSampler: compute_source_index)
        ix = torch.clamp(ix, 0, n - 1)
        x0 = torch.floor(ix)
        t = ix - x0
        for j, c in ((0, 1 - t), (1, t)):
            taps.append((torch.clamp(x0 + j, 0, n - 1).long(), c, KAPPA["bilinear"] + delta))
        # an integer coordinate rounded down in fp32 interpolates from the tap before with a weight of up to delta:
        # the hat function's slope is 1 on both sides of a tap
        taps.append((torch.clamp(x0 - 1, 0, n - 1).long(), torch.zeros_like(t), delta))
        return taps
    x0 = torch.floor(ix)  # bicubic: every tap is clamped (get_value_bounded)
    c, d = _cubic_taps(ix - x0)
    for j in range(4):
        taps.append((torch.clamp(x0 - 1 + j, 0, n - 1).long(), c[j], KAPPA["bicubic"] + delta * d[j]))
    return taps


def warp(ref, flow, fs, bug=None):
    """Warper.forward in the reference's decode (a fresh module: training mode, so the flow is not quantised):
    horizontal taps with flow[0], then vertical taps with flow[1]."""
    _, h, w = ref.shape
    yy, xx = torch.meshgrid(torch.arange(h, dtype=torch.float64), torch.arange(w, dtype=torch.float64), indexing="ij")
    tx = _warp_axis(flow[0], w, xx, fs, bug)
    ty = _warp_axis(flow[1], h, yy, fs, bug)
    v = torch.zeros_like(ref)
    m = torch.zeros_like(ref)
    e = torch.zeros_like(ref)
    a = ref.abs()
    for iy, cy, ey in ty:
        for ix, cx, ex in tx:
            g, ga = ref[:, iy, ix], a[:, iy, ix]
            v += cy * cx * g
            m += (cy * cx).abs() * ga
            e += U * (ey * cx.abs() + cy.abs() * ex) * ga
    nt = fs  # taps with a coefficient
    return T(v, m, e, 2 * (nt + 2))


def inter(residue, motion, refs, gf, fs, bug=None):
    """decode.py:168-189 on float64 copies of fp32 inputs: global shift, warp, alpha / beta blend, residue."""
    r = torch.from_numpy(np.asarray(residue, dtype=np.float64))
    mo = torch.from_numpy(np.asarray(motion, dtype=np.float64))
    is_b = len(refs) == 2
    g = [list(gf[0:2]), list(gf[2:4])]
    if bug == "neg_gf1":
        g[1] = [-x for x in g[1]]
    shifted = [global_shift(torch.from_numpy(np.asarray(rf, dtype=np.float64)), g[i]) for i, rf in enumerate(refs)]
    alpha = torch.clamp(r[3] + 0.5, 0, 1)
    pred = warp(shifted[0], mo[0:2], fs, bug)
    if is_b:
        beta = torch.clamp(r[4] + 0.5, 0, 1)
        bm = r[4].abs() + 0.5
        p2 = warp(shifted[1], mo[2:4], fs, bug)
        pred = T(beta * pred.v + (1 - beta) * p2.v, bm * pred.m + (1 + bm) * p2.m, bm * pred.e + (1 + bm) * p2.e,
                 max(pred.k, p2.k) + 4)
    am = r[3].abs() + 0.5
    return T(alpha * pred.v + r[0:3], am * pred.m + r[0:3].abs(), am * pred.e, pred.k + 3)


# ------------------------------------------------------------------------------------------------------------------
# frame tail (decode.py:191-206) and the comparisons
def tail_levels(x, bd, fmt, window=None):
    """Integer levels of decode_frame's tail on the float64 value, the samples within ``window`` (by default the bound)
    of a tie, and the chroma samples whose exact 2x2 average of rounded samples is itself a tie."""
    M = 2**bd - 1
    # plus the tail's own fp32 product M * x (one rounding, and one to spare)
    z, zb = x.v * M, ((x.bound() if window is None else window) + 2 * U * x.v.abs()) * M
    k = torch.round(z)
    tie = (z - torch.floor(z) - 0.5).abs() <= zb
    if fmt != "yuv420":
        return {"rgb": (torch.clamp(k, 0, M), tie, torch.zeros_like(tie))}
    out = {"y": (torch.clamp(k[0], 0, M), tie[0], torch.zeros_like(tie[0]))}
    h, w = k.shape[-2:]
    for c, name in ((1, "u"), (2, "v")):  # yuv.py:274-299: 2x2 average of the rounded samples, clamp, round
        kk = k[c, :h // 2 * 2, :w // 2 * 2]
        tt = tie[c, :h // 2 * 2, :w // 2 * 2]
        s = kk[0::2, 0::2] + kk[1::2, 0::2] + kk[0::2, 1::2] + kk[1::2, 1::2]
        anyt = tt[0::2, 0::2] | tt[1::2, 0::2] | tt[0::2, 1::2] | tt[1::2, 1::2]
        out[name] = (torch.clamp(torch.round(s / 4), 0, M), anyt, torch.remainder(s, 4) == 2)
    return out


def ratio(got, x):
    """max |got - value| / bound over all samples (0 where both are 0)."""
    err = (torch.as_tensor(np.asarray(got)).to(torch.float64) - x.v).abs()
    b = x.bound()
    r = torch.where(b > 0, err / torch.where(b > 0, b, torch.ones_like(b)),
                    torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))
    return float(r.max())


def check_levels(got, x, bd, fmt, what, window=None):
    """got: finished frame (float k / M: [3, H, W], or the y / u / v dict).  Returns (ties, differing ties).

    Where the raw fp32 output that went into the tail is known, ``window`` is its measured distance from the float64
    value, sample by sample: a sample further than that from a tie has one correct rounding, whatever the bound.
    At most 5 % of the samples (or 4) may be within the window of a tie, so that the check cannot pass by excusing
    every sample (a 4:2:0 chroma sample is near a tie when any of its four luma-grid samples is)."""
    M = 2**bd - 1
    n_tie = n_diff = n_all = n_win = 0
    for key, (want, win, avg) in tail_levels(x, bd, fmt, window).items():
        g = np.asarray(got[key] if fmt == "yuv420" else got, dtype=np.float64)
        lv = torch.from_numpy(np.round(g * M))
        diff = lv != want
        tie = win | avg
        assert not bool((diff & ~tie).any()), f"{what} {key}: {int((diff & ~tie).sum())} samples off a tie differ"
        n_tie += int(tie.sum())
        n_diff += int((diff & tie).sum())
        n_win += int(win.sum())
        n_all += win.numel()
    assert n_win <= max(4, n_all // 20), f"{what}: {n_win} of {n_all} samples within the window of a tie"
    return n_tie, n_diff


def assert_within(got, x, what):
    """Asserts |got - value| <= bound everywhere; returns |got - value| per sample (the tie window of the tail)."""
    r = ratio(got, x)
    err = (torch.as_tensor(np.asarray(got)).to(torch.float64) - x.v).abs()
    print(f"{what}: max |err| / bound = {r:.3g} (K = {x.k}, max |err| = {float(err.max()):.3g})")
    assert r <= 1.0, f"{what}: max |err| / bound = {r}"
    return err


# ------------------------------------------------------------------------------------------------------------------
# the case matrix, shared by the CPU and GPU tests
def _syn(*layers, **fields):
    """Cool-chic header overrides: these synthesis layers, then any other header fields."""
    ov = {"n_layer_synthesis": len(layers), **{f"syn_layer_{i}": lay for i, lay in enumerate(layers)}}
    ov.update(fields)
    return ov


_FIVE = _syn("48-1-linear-relu", "3-1-linear-none", "3-3-residual-relu", "3-3-residual-relu", "3-3-residual-none")

# id -> (size, latent_resolution, hyperlatent_resolution, final upsampling, header overrides, frame tail, seed)
INTRA = {
    # the rows of test_gpu_decode.py::test_synthesis_paths_vs_oracle
    "hop_3ch_two_3x3": ((131, 203), (0, 6), None, None, None, None, 2),
    "residue_4ch": ((70, 50), (0, 3), None, None, _syn("16-1-linear-relu", "4-1-linear-none", "4-3-residual-relu",
                                                       "4-3-residual-none"), None, 2),
    "residue_5ch_one_3x3": ((64, 96), (0, 4), None, None, _syn("16-1-linear-relu", "5-1-linear-none",
                                                               "5-3-residual-relu"), None, 2),
    "motion_2ch_no_3x3_resize": ((48, 80), (2, 5), None, "nearest", _syn("16-1-linear-relu", "2-1-linear-none"), None,
                                 2),
    "smaller_than_one_tile": ((17, 9), (0, 2), None, None, None, None, 2),
    "resized_finish_rgb": ((50, 70), (1, 5), None, "bicubic", None, (8, "rgb"), 2),
    "resized_finish_yuv420": ((44, 60), (1, 5), None, "bilinear", None, (10, "yuv420"), 2),
    "common_randomness": ((40, 56), (0, 3), None, None, {"flag_common_randomness": 1}, None, 2),
    "ups_6_5": ((37, 61), (0, 3), None, None, {"ups_k_size": 6, "ups_preconcat_k_size": 5}, None, 2),
    "five_layers": ((40, 56), (0, 3), None, None, _FIVE, None, 2),
    "3x3_first_layer": ((40, 56), (0, 3), None, None, _syn("8-3-linear-relu", "3-1-linear-none",
                                                           linear_stabiliser_synth=0), None, 2),
    "single_grid": ((40, 56), (0, 0), None, None, None, None, 2),
    "five_layers_finish_yuv420": ((40, 56), (0, 3), None, None, _FIVE, (8, "yuv420"), 2),
    # the sizes of test_gpu_decode.py::CASES with a float tail
    "64x96_hyper": ((64, 96), (0, 6), (4, 6), None, None, (8, "rgb"), 3),
    "17x33": ((17, 33), (0, 4), None, None, None, (8, "rgb"), 3),
    "129x7": ((129, 7), (0, 3), None, None, None, (10, "yuv444"), 3),
    "40x250_hyper": ((40, 250), (0, 6), (4, 6), None, None, (8, "yuv420"), 3),
    "96x64": ((96, 64), (0, 2), None, None, None, (8, "rgb"), 3),
    "1x1": ((1, 1), (0, 1), None, None, None, (8, "rgb"), 3),
    "72x88_nearest_2_5": ((72, 88), (2, 5), None, "nearest", None, (8, "rgb"), 3),
    # the finest grid's row pitch: 100 bytes (plain loads) and 128 bytes (TMA staging)
    "48x100_pitch": ((48, 100), (0, 4), None, None, None, (8, "rgb"), 4),
    "48x128_pitch": ((48, 128), (0, 4), None, None, None, (8, "yuv420"), 4),
}
# the 32 x 16 tile of k_tail_syn: one column / row short, exact, one over, and twice that
for _w in (31, 32, 33, 63, 65):
    for _h in (15, 16, 17):
        INTRA[f"tile_{_h}x{_w}"] = ((_h, _w), (0, 4), None, None, None, (8, "rgb"), 5)

FULL_HD = ((1080, 1920), (0, 6), None, None, None, (8, "rgb"), 1)  # GPU only


def _stream(backend, ss, case):
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    size, lat, hyp, fin, ov, _, seed = case
    cc, h, lat_t = synth.make_coolchic(backend, ss, size, lat, hyp, seed=seed, final_upsampling_type=fin,
                                       overrides=dict(ov) if ov else None)
    h2 = type(h)()
    rest = h2.read_header(cc)
    n_nn, n_lat = h2.get_value("nn_n_bytes"), h2.get_value("n_bytes_latent")
    return h2, desc_from_header(h2), rest[:n_nn], rest[n_nn:n_nn + n_lat], lat_t.cpu().numpy()


@pytest.fixture(scope="session")
def cpu_seed(oracle):
    import pipeline

    from coolchic_b200 import synth

    be = pipeline.OracleBackend()
    return be, synth.SeedStream(be)


# P / B: (size, filter size, B frame, global flows, motion seed)
INTER = {}
for _hw in ((45, 70), (3, 5), (2, 97), (97, 2)):
    for _fs in (2, 4, 6, 8, 10, 12, 14):
        for _b in (False, True):
            _gf = [3, -2, -5, 4] if _b else [-4, 1]
            if _hw == (3, 5):
                _gf = [-1, 2, 2, -1] if _b else [1, -1]
            INTER[f"{_hw[0]}x{_hw[1]}-{'B' if _b else 'P'}-fs{_fs}"] = (_hw, _fs, _b, _gf, _fs * 7 + _b)


def inter_inputs(hw, is_b, seed):
    """Residue, motion and references: flows zero, integer, exactly half-pel, +-500 (border clamp) and fractional,
    mixed pixel by pixel; alpha / beta below 0, inside and above 1."""
    rng = np.random.default_rng(seed)
    h, w = hw
    residue = rng.normal(0, 0.3, size=(5 if is_b else 4, h, w)).astype(np.float32)
    residue[3:] = rng.normal(0, 0.6, size=residue[3:].shape)
    nm = 4 if is_b else 2
    kind = rng.integers(0, 5, size=(nm, h, w))
    frac = rng.normal(0, 3.0, size=(nm, h, w))
    ints = rng.integers(-5, 6, size=(nm, h, w)).astype(np.float64)
    far = np.where(rng.integers(0, 2, size=(nm, h, w)) == 1, 500.0, -500.0)
    motion = np.select([kind == 0, kind == 1, kind == 2, kind == 3], [0.0 * frac, ints, ints + 0.5, far],
                       frac).astype(np.float32)
    refs = [rng.uniform(0, 1, size=(3, h, w)).astype(np.float32) for _ in range(2 if is_b else 1)]
    return residue, motion, refs


# ------------------------------------------------------------------------------------------------------------------
# CPU: layout, the oracle against the restatement, negative controls, reference fixtures
@pytest.mark.parametrize("name", list(INTRA))
def test_nn_layout_matches_split_nn(oracle, cpu_seed, name):
    """The reference's get_param layout, restated here, against synth.split_nn (shared by the writer and decoder)."""
    from coolchic_b200 import synth

    h, d, nnb, _, _ = _stream(*cpu_seed, INTRA[name])
    ints = oracle.decode_nn(d, nnb)
    p = h.get_coolchic_parameter()
    mine = {}
    pos = 0
    for m, kind, nm, shape in nn_layout(p):
        n = int(np.prod(shape))
        mine.setdefault(f"{m}.{kind}", []).append(ints[pos:pos + n])
        pos += n
    assert pos == len(ints)
    theirs = synth.split_nn(d, ints)
    for key, tensors in theirs.items():
        a = [t.reshape(-1) for t in tensors.values()]
        b = mine.get(key, [])
        assert [x.size for x in a] == [x.size for x in b], key
        assert all(np.array_equal(x, y) for x, y in zip(a, b)), key


@pytest.mark.parametrize("name", list(INTRA))
def test_intra_oracle_vs_restatement(oracle, cpu_seed, name):
    h, d, nnb, _, lat = _stream(*cpu_seed, INTRA[name])
    ints = oracle.decode_nn(d, nnb)
    x = intra(h, ints, lat)
    raw = oracle.synthesize(d, ints, lat)
    err = assert_within(raw, x, f"{name} oracle raw")
    fin = INTRA[name][5]
    if fin is not None:
        n_tie, n_diff = check_levels(oracle.finish_frame(raw, *fin), x, *fin, f"{name} oracle", window=err)
        print(f"{name}: {n_tie} samples within the bound of a rounding tie, {n_diff} of them differ")


def _inter_case(name):
    hw, fs, is_b, gf, seed = INTER[name]
    residue, motion, refs = inter_inputs(hw, is_b, seed)
    return residue, motion, refs, gf, fs


@pytest.mark.parametrize("name", list(INTER))
def test_inter_oracle_vs_restatement(oracle, name):
    residue, motion, refs, gf, fs = _inter_case(name)
    got = oracle.inter_predict(residue, motion, refs[0], refs[1] if len(refs) == 2 else None, gf, fs)
    assert_within(got, inter(residue, motion, refs, gf, fs), f"{name} oracle")


# reconstruct_frame: 4:2:0 references are upsampled by repetition (yuv.py:302-316, decode.py:159-160)
RECON = [("rgb", 8, False, 2), ("rgb", 8, True, 14), ("yuv444", 10, True, 4), ("yuv444", 10, False, 10),
         ("yuv420", 8, True, 8), ("yuv420", 10, False, 6), ("yuv420", 8, True, 12), ("yuv420", 8, False, 2)]


def recon_inputs(fmt, bd, is_b, fs):
    rng = np.random.default_rng(100 + fs + 50 * is_b)
    h, w = 46, 72
    M = 2**bd - 1
    residue, motion, _ = inter_inputs((h, w), is_b, fs + 3)

    def make_ref():
        if fmt == "yuv420":
            return {"y": (rng.integers(0, M + 1, size=(h, w)) / M).astype(np.float32),
                    "u": (rng.integers(0, M + 1, size=(h // 2, w // 2)) / M).astype(np.float32),
                    "v": (rng.integers(0, M + 1, size=(h // 2, w // 2)) / M).astype(np.float32)}
        return (rng.integers(0, M + 1, size=(3, h, w)) / M).astype(np.float32)

    refs = [make_ref() for _ in range(2 if is_b else 1)]
    gf = [2, -3, -1, 4] if is_b else [-4, 1]
    return residue, motion, refs, gf


def to444(r):
    if not isinstance(r, dict):
        return r
    up = lambda p: np.repeat(np.repeat(p, 2, axis=0), 2, axis=1)  # noqa: E731
    return np.stack([r["y"], up(r["u"]), up(r["v"])])


@pytest.mark.parametrize("fmt,bd,is_b,fs", RECON)
def test_reconstruct_oracle_vs_restatement(oracle, fmt, bd, is_b, fs):
    residue, motion, refs, gf = recon_inputs(fmt, bd, is_b, fs)
    r444 = [to444(r) for r in refs]
    x = inter(residue, motion, r444, gf, fs)
    pre = oracle.inter_predict(residue, motion, r444[0], r444[1] if is_b else None, gf, fs)
    err = assert_within(pre, x, f"{fmt} {'B' if is_b else 'P'} fs{fs} oracle")
    n_tie, n_diff = check_levels(oracle.finish_frame(pre, bd, fmt), x, bd, fmt, "oracle", window=err)
    print(f"{n_tie} samples within the bound of a rounding tie, {n_diff} of them differ")


# each deliberate change must fail the comparison with the oracle on at least one of its cases
CONTROLS = {
    "crop_shift": ["17x33", "hop_3ch_two_3x3", "ups_6_5"],
    "even_preconcat": ["17x33", "ups_6_5"],
    "stab_all": ["common_randomness"],
    "sinc_shift": ["45x70-P-fs8", "3x5-B-fs14"],
    "neg_gf1": ["45x70-B-fs6", "45x70-B-fs2"],
}


@pytest.mark.parametrize("bug", list(CONTROLS))
def test_negative_controls_are_detected(oracle, cpu_seed, bug):
    worst = 0.0
    for name in CONTROLS[bug]:
        if name in INTRA:
            h, d, nnb, _, lat = _stream(*cpu_seed, INTRA[name])
            ints = oracle.decode_nn(d, nnb)
            got, x = oracle.synthesize(d, ints, lat), intra(h, ints, lat, bug)
        else:
            residue, motion, refs, gf, fs = _inter_case(name)
            got = oracle.inter_predict(residue, motion, refs[0], refs[1] if len(refs) == 2 else None, gf, fs)
            x = inter(residue, motion, refs, gf, fs, bug)
        r = ratio(got, x)
        print(f"negative control {bug} on {name}: max |err| / bound = {r:.3g}")
        worst = max(worst, r)
    assert worst > 1.0, f"negative control {bug} was not detected"
    print(f"negative control {bug}: detected")


def _coolchics(rest, n):
    """Parse n Cool-chic sections: [(header, nn_bytes, latent_bytes)] and the rest."""
    from coolchic_b200.bitstream.header import CoolChicHeader

    out = []
    for _ in range(n):
        c = CoolChicHeader()
        rest = c.read_header(rest)
        n_nn, n_lat = c.get_value("nn_n_bytes"), c.get_value("n_bytes_latent")
        out.append((c, rest[:n_nn], rest[n_nn:n_nn + n_lat]))
        rest = rest[n_nn + n_lat:]
    return out, rest


def _restate_coolchic(oracle, c, nnb, lb, bug=None):
    from coolchic_b200._desc import desc_from_header

    d = desc_from_header(c)
    ints = oracle.decode_nn(d, nnb)
    lat, _ = oracle.decode_latents(d, ints, lb)  # the entropy side, pinned to constriction's output elsewhere
    return intra(c, ints, lat, bug)


def test_kodim14_reference_raw_rows_vs_restatement(oracle, kodim14):
    """The reference's raw synthesis rows (fp32, its own PyTorch order) within the bound of the float64 value."""
    ints = oracle.decode_nn(kodim14["desc"], kodim14["nn_bytes"])
    x = intra(kodim14["header"], ints, kodim14["latents"])
    g = kodim14["raw_rows"]
    rows = torch.as_tensor(g["rows"]).long()
    assert_within(g["data"], x.map(lambda t: t[:, rows, :]), "kodim14 reference rows")
    assert_within(g["left"], x.map(lambda t: t[:, :, :8]), "kodim14 reference left columns")
    assert_within(g["right"], x.map(lambda t: t[:, :, -8:]), "kodim14 reference right columns")
    ref = kodim14["image"].transpose(2, 0, 1).astype(np.float64) / 255
    # within the rows' measured error of a tie, and nowhere else, may a row of the reference's image differ
    # (the image and the rows come from two runs of the reference, which may round a tie apart: the rows' largest
    # error is the window, not their error sample by sample)
    err = float((torch.from_numpy(g["data"]).to(torch.float64) - x.v[:, rows, :]).abs().max())
    xr = x.map(lambda t: t[:, rows, :])
    n_tie, n_diff = check_levels(ref[:, g["rows"], :], xr, 8, "rgb", "kodim14 reference rows", window=err)
    print(f"kodim14: {n_tie} samples within the bound of a rounding tie, {n_diff} of them differ")


# every stream decoded by the unmodified reference, with its integer samples and the raw output of each of its
# Cool-chics (oracle/gen_golden_modes.py, gen_golden_gop.py, gen_golden_archs.py)
REF_FIXTURES = ["img_48x72_rgb_common_randomness", "img_50x70_rgb_final_bicubic", "img_44x60_yuv420_final_bilinear",
                "img_48x64_rgb_arm8_1hidden", "img_40x56_yuv444_10bit_arm24",
                "gop5_64x96_yuv420", "gop3_40x56_rgb", "gop3_48x72_yuv420_bilinear", "gop3_40x56_rgb_bicubic",
                "gop3_48x72_yuv420_sinc6", "gop4_40x56_rgb_sinc12",
                "arch_37x61_ups_6_5", "arch_40x56_five_layers", "arch_40x56_3x3_first_layer", "arch_40x56_single_grid",
                "arch_17x33", "arch_129x7", "arch_1x1", "arch_45x70_nearest_2_5", "arch_gop3_7x9_sinc10",
                "arch_gop3_7x9_sinc14"]


def reference_fixture(oracle, name, bug=None):
    """Each Cool-chic of the stream restated and compared with the reference's raw output under the bound; each frame's
    integer samples against the reference's, within the measured error of the raw output of a tie (I frames), or
    within the prediction's bound (P / B frames, predicted from the reference's own residue, motion and decoded
    references).  Returns the largest max |err| / bound; with ``bug`` nothing is asserted, and a frame whose
    integer samples differ off a tie counts as infinitely far."""
    from coolchic_b200.bitstream.header import FrameHeader, VideoHeader

    data = open(os.path.join(GOLDEN, name + ".cool"), "rb").read()
    gold = np.load(os.path.join(GOLDEN, name + ("_frames.npz" if "gop" in name else ".npz")))
    raw = np.load(os.path.join(GOLDEN, name + "_raw.npz"))
    v = VideoHeader()
    rest = v.read_header(data)
    worst, n_tie, n_diff, i = 0.0, 0, 0, 0
    for _ in range(v.get_coding_structure().get_max_coding_order() + 1):
        f = FrameHeader()
        rest = f.read_header(rest)
        ftype, fmt, bd = f.get_value("frame_type"), f.get_value("frame_data_type"), f.get_value("bitdepth")
        ccs, rest = _coolchics(rest, 1 if ftype == "I" else 2)
        outs = []
        for cc in ccs:
            x, r = _restate_coolchic(oracle, *cc, bug=bug), raw[f"c{i}"]
            worst = max(worst, ratio(r, x))
            err = (torch.from_numpy(r).to(torch.float64) - x.v).abs() if bug else assert_within(
                r, x, f"{name} Cool-chic {i}")
            outs.append((x, r, err))
            i += 1
        M = 2**bd - 1

        def frame(idx):
            if name.startswith("img"):  # gen_golden_modes.py names the planes only
                return {k: gold[k] / M for k in "yuv"} if fmt == "yuv420" else gold["rgb"] / M
            return {k: gold[f"{idx}_{k}"] / M for k in "yuv"} if fmt == "yuv420" else gold[str(idx)] / M

        if ftype == "I":
            x, _, window = outs[0]
        else:
            refs = [to444(frame(j)) for j in f.get_value("index_references")]
            x = inter(outs[0][1], outs[1][1], refs, f.get_value("global_flow"), f.get_value("warp_filter_size"), bug)
            window = None
        try:
            t, d = check_levels(frame(f.get_value("display_index")), x, bd, fmt,
                                f"{name} frame {f.get_value('display_index')}", window=window)
        except AssertionError:
            if bug is None:
                raise
            worst = math.inf
            continue
        n_tie += t
        n_diff += d
    assert i == len(raw.files)
    if bug is None:
        print(f"{name}: {n_tie} samples within the bound of a rounding tie, {n_diff} of them differ")
    return worst


@pytest.mark.parametrize("name", REF_FIXTURES)
def test_reference_fixtures_vs_restatement(oracle, name):
    reference_fixture(oracle, name)


# each deliberate change must fail against every reference fixture listed for it
REF_CONTROLS = {
    "crop_shift": ["img_50x70_rgb_final_bicubic", "arch_17x33", "arch_37x61_ups_6_5"],
    "even_preconcat": ["img_40x56_yuv444_10bit_arm24", "arch_37x61_ups_6_5", "arch_129x7"],
    "stab_all": ["img_48x72_rgb_common_randomness"],
    "sinc_shift": ["gop4_40x56_rgb_sinc12", "arch_gop3_7x9_sinc10", "arch_gop3_7x9_sinc14"],
    "neg_gf1": ["gop5_64x96_yuv420"],
}


@pytest.mark.parametrize("bug", list(REF_CONTROLS))
def test_negative_controls_fail_against_the_reference(oracle, bug):
    for name in REF_CONTROLS[bug]:
        r = reference_fixture(oracle, name, bug)
        print(f"negative control {bug} on the reference's {name}: max |err| / bound = {r:.3g}")
        assert r > 1.0, f"negative control {bug} passes against the reference's {name}"


# ------------------------------------------------------------------------------------------------------------------
# GPU: the device against the restatement
def _device_intra(ctx, d, nnb, lb, fin):
    out, _ = ctx.decode_many([d], [nnb], [lb], finish=[fin])
    o = out[0]
    if isinstance(o, dict):
        return {k: o[k][0, 0].cpu().numpy() for k in "yuv"}
    return o[0].cpu().numpy()


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(INTRA))
def test_intra_device_vs_restatement(ctx, oracle, cpu_seed, name):
    h, d, nnb, lb, lat = _stream(*cpu_seed, INTRA[name])
    x = intra(h, oracle.decode_nn(d, nnb), lat)
    err = assert_within(_device_intra(ctx, d, nnb, lb, None), x, f"{name} device raw")
    fin = INTRA[name][5]
    if fin is not None:
        n_tie, n_diff = check_levels(_device_intra(ctx, d, nnb, lb, fin), x, *fin, f"{name} device", window=err)
        print(f"{name}: {n_tie} samples within the bound of a rounding tie, {n_diff} of them differ")


MIXED = ["64x96_hyper", "17x33", "129x7", "1x1", "40x250_hyper", "tile_15x31", "48x128_pitch", "resized_finish_rgb",
         "residue_4ch", "common_randomness", "ups_6_5"]


@pytest.mark.gpu
def test_mixed_batch_device_vs_restatement(ctx, oracle, cpu_seed):
    """One decode_many call for Cool-chics of different sizes and architectures, raw and then with their frame
    tails: the jobs share the cascade and tail launches, so every job's offsets and indexing are checked."""
    items = [_stream(*cpu_seed, INTRA[n]) for n in MIXED]
    fins = [INTRA[n][5] for n in MIXED]
    args = ([it[1] for it in items], [it[2] for it in items], [it[3] for it in items])
    raws, _ = ctx.decode_many(*args)
    fin_outs, _ = ctx.decode_many(*args, finish=fins)
    for name, (h, d, nnb, _, lat), raw, out, fin in zip(MIXED, items, raws, fin_outs, fins):
        x = intra(h, oracle.decode_nn(d, nnb), lat)
        err = assert_within(raw[0].cpu().numpy(), x, f"{name} in a batch, raw")
        if fin is not None:
            got = {k: out[k][0, 0].cpu().numpy() for k in "yuv"} if fin[1] == "yuv420" else out[0].cpu().numpy()
            check_levels(got, x, *fin, f"{name} in a batch", window=err)


@pytest.mark.gpu
def test_full_hd_device_vs_restatement(ctx, oracle, seed_stream):
    """One whole 1080p 7-grid frame: raw output and the fused frame tail."""
    h, d, nnb, lb, lat = _stream(ctx, seed_stream, FULL_HD)
    x = intra(h, oracle.decode_nn(d, nnb), lat)
    err = assert_within(_device_intra(ctx, d, nnb, lb, None), x, "1080p device raw")
    n_tie, n_diff = check_levels(_device_intra(ctx, d, nnb, lb, FULL_HD[5]), x, *FULL_HD[5], "1080p device",
                                 window=err)
    print(f"1080p: {n_tie} samples within the bound of a rounding tie, {n_diff} of them differ")


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(INTER))
def test_inter_device_vs_restatement(ctx, name):
    from coolchic_b200.io import FrameData

    residue, motion, refs, gf, fs = _inter_case(name)
    is_b = len(refs) == 2
    fds = [FrameData(8, "rgb", torch.from_numpy(r[None]).cuda()) for r in refs]
    got = ctx.inter_predict(torch.from_numpy(residue[None]).cuda(), torch.from_numpy(motion[None]).cuda(), fds, is_b,
                            "rgb", gf, fs)
    assert_within(got[0].cpu().numpy(), inter(residue, motion, refs, gf, fs), f"{name} device")


@pytest.mark.gpu
@pytest.mark.parametrize("fmt,bd,is_b,fs", RECON)
def test_reconstruct_device_vs_restatement(ctx, fmt, bd, is_b, fs):
    from coolchic_b200.io import FrameData

    residue, motion, refs, gf = recon_inputs(fmt, bd, is_b, fs)
    x = inter(residue, motion, [to444(r) for r in refs], gf, fs)

    def to_fd(r):
        if fmt == "yuv420":
            return FrameData(bd, fmt, {k: torch.from_numpy(v[None, None]).cuda() for k, v in r.items()})
        return FrameData(bd, fmt, torch.from_numpy(r[None]).cuda())

    res_d, mot_d = torch.from_numpy(residue[None]).cuda(), torch.from_numpy(motion[None]).cuda()
    # the prediction before the tail, from the same references in 4:4:4
    pre = ctx.inter_predict(res_d, mot_d, [FrameData(bd, "rgb", torch.from_numpy(to444(r)[None]).cuda()) for r in refs],
                            is_b, "rgb", gf, fs)
    err = assert_within(pre[0].cpu().numpy(), x, f"{fmt} {'B' if is_b else 'P'} fs{fs} device prediction")
    got = ctx.reconstruct_frame(res_d, mot_d, [to_fd(r) for r in refs], is_b, fmt, bd, gf, fs)
    got = {k: got[k][0, 0].cpu().numpy() for k in "yuv"} if fmt == "yuv420" else got[0].cpu().numpy()
    n_tie, n_diff = check_levels(got, x, bd, fmt, "device", window=err)
    print(f"{fmt} {'B' if is_b else 'P'} fs{fs}: {n_tie} samples within the bound of a rounding tie, {n_diff} differ")
