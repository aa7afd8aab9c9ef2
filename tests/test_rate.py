"""Rate analysis (coolchic_b200.bitstream.rate, ccd_latent_rate): exact bits per latent symbol under the model the
range coder used, per grid and per pixel, and the exp-Golomb length of the network.

The checker is a numpy restatement of the integer ARM + IFCE (armint.py:30-203, component/coolchic.py:72-146,
latent.py:142-173), evaluated on all symbols of a grid at once (the latents are known: no wavefront).  Its
cumulatives come from the oracle's exported Laplace tables (``cco_laplace_domain``), and the CPU tests prove its
(mu, scale) right by driving the oracle's range decoder with them over a real payload: the golden latents come back
bit for bit.  The GPU tests compare the rate kernel with the checker symbol for symbol."""
import ctypes
import glob
import os
import re

import numpy as np
import pytest
from conftest import GOLDEN, ROOT

GENERIC_ARM = ["img_48x64_rgb_arm8_1hidden", "img_40x56_yuv444_10bit_arm24"]

# causal context of the ARM in priority order over the 9x9 mask (core/arm.py:496-562)
CTX_DY = [0, -1, -1, -1, 0, -2, -3, 0, -1, -2, -2, -1, -2, -1, -2, -3, 0, -1, -2, -2, -3, -3, -3, -4, -1, -4, -1, -2,
          -3, -3, -4, -4, -2, -3, -3, -4, -4, -4, -4, -4]
CTX_DX = [-1, 0, -1, 1, -2, 0, 0, -3, -2, 1, -1, 2, -2, -3, 2, 1, -4, 3, -3, 3, -1, -2, 2, 0, -4, -1, 4, 4, -3, 3, -2,
          1, -4, -4, 4, -3, 2, 3, -4, 4]


def _latent_offsets(d):
    """Decode-order offset of every grid (coarsest grid first)."""
    offs, p = [0] * d.n_grids, 0
    for g in range(d.n_grids - 1, -1, -1):
        offs[g] = p
        p += d.grid_h[g] * d.grid_w[g]
    return offs


def _fixed_point(q, b, s_w, s_b, ifce_cols, residual, subtract_last=False):
    """armint.py:30-170 for one linear layer: q [out][in], b [out] -> int64 W [in][out], B [out]."""
    q = np.asarray(q, dtype=np.int64)
    shift = np.where(ifce_cols, 16 + s_w - 8, 16 + s_w).astype(np.int64)
    W = (q * np.left_shift(np.int64(1), shift)[None, :]).T.copy()
    if residual and q.shape[0] == q.shape[1]:
        i = np.arange(q.shape[0])
        W[i, i] += np.where(ifce_cols, 1 << 8, 1 << 16)
    B = np.asarray(b, dtype=np.int64).copy()
    if subtract_last:
        B[1] -= 4 << (-s_b)
    return W, B * (1 << (32 + s_b))


def mac(B, x, W):
    """B + x @ W in int64, after proving that no partial sum can wrap: |B| + |x| @ |W| in float64 (relative error
    below 2^-40 at these sizes) stays under 2^62.  A wrap would go unnoticed, on the device as here."""
    bound = np.abs(B).astype(np.float64) + np.abs(x).astype(np.float64) @ np.abs(W).astype(np.float64)
    assert bound.size == 0 or bound.max() < 2.0**62, f"an ARM / IFCE sum reaches {bound.max():.3g}"
    return B + x @ W


# negative controls of the checker (tests/test_arm_space.py), each outside the ARMs the older fixtures have:
#   ctx_swap         spatial contexts 24 and 25 read each other's neighbour
#   ifce_grid        IFCE channels 12 and up read the grid one finer than theirs
#   linear_identity  an ARM without hidden layer evaluated through one identity layer (a ReLU of its inputs)
#   residual_drop    hidden layers from the third on lose their residual connection
CHECKER_BUGS = ("ctx_swap", "ifce_grid", "linear_identity", "residual_drop")


def model_indices(d, nn, latents, bug=None):
    """(mu_idx, sc_idx) of every symbol (decode order) after the clamp of latent.py:165 / rangecoder.py:89-91.
    ``bug``: one of CHECKER_BUGS (a negative control), or None."""
    from coolchic_b200 import synth

    sec = synth.split_nn(d, nn)
    cf = d.n_ifce_out if d.flag_ifce else 0
    dim, H = d.n_ctx + cf, d.arm_hidden
    s_w, s_b = int(d.qshift[0]), int(d.qshift[1])
    ifce_cols = np.arange(dim) >= dim - cf if cf else np.zeros(dim, dtype=bool)
    aw, ab = sec["arm.weight"], sec["arm.bias"]
    layers = [_fixed_point(aw[f"mlp.{2 * l}"], ab[f"mlp.{2 * l}"], s_w, s_b,
                           ifce_cols if l == 0 else np.zeros(dim, dtype=bool), not (bug == "residual_drop" and l >= 2),
                           l == H) for l in range(H + 1)]
    if bug == "linear_identity" and H == 0:
        layers.insert(0, (np.eye(dim, dtype=np.int64) << 16, np.zeros(dim, np.int64)))
    dy, dx = list(CTX_DY), list(CTX_DX)
    if bug == "ctx_swap":
        dy[24], dy[25], dx[24], dx[25] = dy[25], dy[24], dx[25], dx[24]
    if d.arm_stab:
        Ws, Bs = _fixed_point(aw["stab"], ab["stab"], s_w, s_b, ifce_cols, False)
    else:
        Ws, Bs = np.zeros((dim, 2), np.int64), np.zeros(2, np.int64)
    offs = _latent_offsets(d)
    lat = np.asarray(latents).astype(np.int64)
    grids = [lat[offs[g]:offs[g] + d.grid_h[g] * d.grid_w[g]].reshape(d.grid_h[g], d.grid_w[g]) for g in range(d.n_grids)]
    mu_idx, sc_idx = np.zeros(lat.size, np.int64), np.zeros(lat.size, np.int64)
    for g in range(d.n_grids):
        h, w = grids[g].shape
        X = np.zeros((h, w, dim), np.int64)
        P = np.pad(grids[g], ((4, 0), (4, 4)))
        for t in range(d.n_ctx):
            X[:, :, t] = P[4 + dy[t]:4 + dy[t] + h, 4 + dx[t]:4 + dx[t] + w]
        n_in = int(d.grid_ifce_in[g]) if cf else 0
        if n_in:
            # IFCE features at (y >> 1, x >> 1) from the coarser grids g+1+c, each read at >> sh[c] (coolchic.py:95-146)
            Wi, Bi = _fixed_point(sec["ifce.weight"][f"grid{g}"], sec["ifce.bias"][f"grid{g}"], int(d.qshift[2]),
                                  int(d.qshift[3]), np.zeros(n_in, dtype=bool), False)
            yy, xx = np.arange(h) >> 1, np.arange(w) >> 1
            V = np.zeros((h, w, n_in), np.int64)
            if g < d.n_grids - 1:  # the first grid decoded has one all-zero input
                sh = 0
                for c in range(n_in):
                    if c > 0 and (d.grid_h[g + c], d.grid_w[g + c]) != (d.grid_h[g + 1 + c], d.grid_w[g + 1 + c]):
                        sh += 1
                    if bug == "ifce_grid" and c >= 12:
                        G = grids[g + c]
                        V[:, :, c] = G[(yy >> sh)[:, None] % G.shape[0], (xx >> sh)[None, :] % G.shape[1]]
                        continue
                    V[:, :, c] = grids[g + 1 + c][(yy >> sh)[:, None], (xx >> sh)[None, :]]
            acc = mac(Bi, V << 16, Wi)
            X[:, :, d.n_ctx:] = (acc >> 24).astype(np.float32).astype(np.int64)  # fp32 round trip
        x = X.reshape(h * w, dim) << 16
        s = mac(Bs, x, Ws)
        for W, B in layers[:-1]:
            x = np.maximum(mac(B, x, W), 0) >> 16
        o = (mac(layers[-1][1], x, layers[-1][0]) + s) >> 24
        sl = slice(offs[g], offs[g] + h * w)
        mu_idx[sl] = np.clip(o[:, 0] + 16384, 0, 32767)
        sc_idx[sl] = np.clip(o[:, 1] + 1280, 0, 2560)
    return mu_idx, sc_idx


def model_freq(oracle, latents, mu_idx, sc_idx):
    """freq = left(s+1) - left(s) of the leaky quantised Laplace (SURVEY Appendix C.1), from the oracle's tables
    trunc(FW * 0.5 exp(-|d|/b)) / trunc(FW * (1 - 0.5 exp(-|d|/b))) at |d| = n / 256 of each scale used."""
    s = np.asarray(latents).astype(np.int64)
    freq = np.zeros(s.size, np.int64)
    order = np.argsort(sc_idx, kind="stable")
    uniq, first = np.unique(sc_idx[order], return_index=True)
    bounds = list(first) + [s.size]
    for j, sc in enumerate(uniq):
        idx = order[bounds[j]:bounds[j + 1]]
        lo, hi = oracle.laplace_domain(int(sc), int(sc) + 1)

        def left(v):
            n = 256 * v - 128 - mu_idx[idx] + 16384  # 256 * ((v - 0.5) - mu), an exact integer
            l = np.where(n <= 0, lo[np.clip(-n, 0, 32640)], hi[np.clip(n, 0, 32640)]).astype(np.int64) + (v + 64)
            return np.where(v <= -64, 0, np.where(v > 63, 1 << 24, l))

        freq[idx] = left(s[idx] + 1) - left(s[idx])
    return freq


def _coding_order(d):
    """Decode-order indices in the order the range coder visits the symbols: grids coarsest first, each along its
    wavefront (diagonal k = x + 10 y, rising y; latent.py:63-122), or in raster order when w <= 9."""
    offs, out = _latent_offsets(d), []
    for g in range(d.n_grids - 1, -1, -1):
        h, w = d.grid_h[g], d.grid_w[g]
        y, x = np.divmod(np.arange(h * w), w)
        out.append(offs[g] + (np.arange(h * w) if w <= 9 else np.lexsort((y, x + 10 * y))))
    return np.concatenate(out)


def _oracle_range_decode(oracle, latent_bytes, mu, scale):
    """The oracle's constriction stand-in decoder driven by per-symbol (mu, scale) in coding order."""
    L = oracle.lib()
    L.cco_rc_dec_new.restype = ctypes.c_void_p
    L.cco_rc_dec_new.argtypes = [ctypes.c_void_p, ctypes.c_size_t]
    L.cco_rc_dec_free.argtypes = [ctypes.c_void_p]
    L.cco_rc_decode_block.restype = ctypes.c_int
    L.cco_rc_decode_block.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p]
    words = np.frombuffer(latent_bytes[:len(latent_bytes) // 4 * 4], dtype="<u4").copy()
    mu, scale = np.ascontiguousarray(mu, np.float32), np.ascontiguousarray(scale, np.float32)
    out = np.zeros(mu.size, np.int32)
    h = L.cco_rc_dec_new(words.ctypes.data, words.size)
    try:
        rc = L.cco_rc_decode_block(h, mu.ctypes.data, scale.ctypes.data, mu.size, out.ctypes.data)
    finally:
        L.cco_rc_dec_free(h)
    assert rc == 0
    return out


def _oracle_scales():
    words = re.findall(r"0x([0-9a-fA-F]{8})u", open(os.path.join(ROOT, "oracle", "scale_table.inc")).read())
    return np.array([int(v, 16) for v in words], dtype=np.uint32).view(np.float32)


def _coolchics(data: bytes):
    """(header, nn_bytes, latent_bytes) of every Cool-chic of a bitstream, in coding order."""
    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream import rate
    from coolchic_b200.bitstream.header import FrameHeader, VideoHeader

    buf = memoryview(data)
    v = VideoHeader()
    buf = v.read_header(buf)
    out = []
    for _ in range(v.get_coding_structure().get_max_coding_order() + 1):
        f = FrameHeader()
        buf = f.read_header(buf)
        for _ in range(2 if f.get_value("frame_type") in ("P", "B") else 1):
            h, nb, lb, buf = rate._split_coolchic(buf)
            out.append((h, nb, lb))
    assert len(buf) == 0
    return out


def _golden(name):
    return open(os.path.join(GOLDEN, name + ".cool"), "rb").read()


def spatial_canonical(bit_maps, H, W):
    """Canonical restatement of the spatial map: finest grid first, acc = 0; acc += bits / fp32((H*W)/(h*w)),
    nearest index floor(fp32(y) * fp32(h / H)) clamped to h - 1, everything in fp32."""
    acc = np.zeros((H, W), dtype=np.float32)
    for b in bit_maps:
        h, w = b.shape
        ratio = np.float32((H * W) / (h * w))
        sy, sx = np.float32(h) / np.float32(H), np.float32(w) / np.float32(W)
        yi = np.minimum(np.floor(np.arange(H, dtype=np.float32) * sy).astype(np.int64), h - 1)
        xi = np.minimum(np.floor(np.arange(W, dtype=np.float32) * sx).astype(np.int64), w - 1)
        acc = acc + (b.astype(np.float32) / ratio)[yi][:, xi]
    return acc


def _grid_maps(desc, flat):
    """Decode-order array -> per-grid [h, w] arrays, finest first."""
    out, off = [None] * desc.n_grids, 0
    for g in range(desc.n_grids - 1, -1, -1):
        h, w = desc.grid_h[g], desc.grid_w[g]
        out[g] = flat[off:off + h * w].reshape(h, w)
        off += h * w
    return out


# ---------------------------------------------------------------------------------------------- CPU
@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "*.cool"))), ids=os.path.basename)
def test_checker_model_decodes_the_payload(path, oracle):
    """The checker's (mu, scale) of every symbol, fed to the oracle's range decoder in coding order, decode the
    latent payload of every golden Cool-chic back to its latents: the checker's model is the coder's."""
    from coolchic_b200._desc import desc_from_header

    for h, nb, lb in _coolchics(open(path, "rb").read()):
        d = desc_from_header(h)
        nn = oracle.decode_nn(d, nb)
        lat, _ = oracle.decode_latents(d, nn, lb)
        mu_idx, sc_idx = model_indices(d, nn, lat)
        order = _coding_order(d)
        mu = ((mu_idx - 16384) / 256.0).astype(np.float32)
        dec = _oracle_range_decode(oracle, lb, mu[order], _oracle_scales()[sc_idx][order])
        assert np.array_equal(dec, lat[order].astype(np.int32))
        freq = model_freq(oracle, lat, mu_idx, sc_idx)
        assert freq.min() >= 1 and freq.max() <= 1 << 24
        assert 0 <= 8 * len(lb) - np.sum(24.0 - np.log2(freq.astype(np.float64))) < 3 * 32


def test_checker_rate_kodim14(kodim14, oracle):
    """The information content of kodim14's latents is below the latent payload by the range coder's seal and
    its scale truncation: 75.7 bits, between two and three 32-bit words."""
    d = kodim14["desc"]
    nn = oracle.decode_nn(d, kodim14["nn_bytes"])
    mu_idx, sc_idx = model_indices(d, nn, kodim14["latents"])
    freq = model_freq(oracle, kodim14["latents"], mu_idx, sc_idx)
    assert freq.min() >= 1 and freq.max() <= 1 << 24
    assert mu_idx.min() >= 0 and mu_idx.max() <= 32767 and sc_idx.min() >= 0 and sc_idx.max() <= 2560
    model = float(np.sum(24.0 - np.log2(freq.astype(np.float64))))
    payload = 8 * len(kodim14["lat_bytes"])
    assert payload == 247616
    assert model == pytest.approx(247540.28993988558, abs=1e-6)
    assert 0 < payload - model < 3 * 32


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "*.cool"))), ids=os.path.basename)
def test_nn_bits_fill_the_nn_payload(path, oracle):
    """Codeword lengths per section + the padding bits = 8 * nn_n_bytes exactly, for every Cool-chic."""
    from coolchic_b200._desc import desc_from_header
    from coolchic_b200.bitstream import rate

    for h, nb, _ in _coolchics(open(path, "rb").read()):
        d = desc_from_header(h)
        nn = oracle.decode_nn(d, nb)
        counts = rate.nn_section_counts(d)
        _, oc = oracle.nn_counts(d)
        assert [counts[m][k] for m in ("arm", "ifce", "upsampling", "synthesis") for k in ("weight", "bias")] == oc.tolist()
        bits = rate.nn_bits(d, nn)
        assert sum(sum(v.values()) for v in bits.values()) + h.get_value("nn_n_bit_pad") == 8 * h.get_value("nn_n_bytes")


def test_spatial_canonical_matches_reference_formula(kodim14):
    """The canonical fp32 order agrees with training/test.py:217-235 (divide, F.interpolate nearest, cat, sum)
    to 1e-6 relative, on kodim14's grid sizes and on a non-dyadic image size."""
    import torch
    import torch.nn.functional as F

    rng = np.random.default_rng(0)
    d = kodim14["desc"]
    cases = [((d.img_h, d.img_w), d.grid_sizes()), ((75, 101), [(75, 101), (38, 51), (19, 26), (10, 13), (5, 7)])]
    for (H, W), sizes in cases:
        maps = [rng.exponential(2.0, size=s).astype(np.float32) for s in sizes]
        ours = spatial_canonical(maps, H, W)
        up = []
        for m in maps:
            rate = torch.from_numpy(m.copy())[None, None]
            cur_h, cur_w = rate.shape[-2:]
            rate /= (H * W) / (cur_h * cur_w)
            up.append(F.interpolate(rate, size=(H, W), mode="nearest"))
        ref = torch.cat(up, dim=1).sum(dim=1, keepdim=True)[0, 0].numpy()
        np.testing.assert_allclose(ours, ref, rtol=1e-6, atol=0)


# ---------------------------------------------------------------------------------------------- GPU
def _device_rate(ctx, desc, nn_bytes, lat_bytes, **kw):
    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native

    _, lats = ctx.decode_many([desc], [nn_bytes], [lat_bytes], want_latents=True)
    nn = _native.decode_nn(desc, nn_bytes)
    return nn, lats[0], ctx.latent_rate([desc], [nn], [lats[0]], **kw)[0]


def _check_against_checker(ctx, oracle, desc, nn_bytes, lat_bytes):
    nn, lat, r = _device_rate(ctx, desc, nn_bytes, lat_bytes, want_freq=True, want_mu_sc=True, want_spatial=True)
    lat_h = lat.cpu().numpy()
    mu_idx, sc_idx = model_indices(desc, nn, lat_h)
    freq = model_freq(oracle, lat_h, mu_idx, sc_idx)
    f = r["freq"].cpu().numpy().view(np.uint32)
    ms = r["mu_sc"].cpu().numpy().view(np.uint32)
    assert np.array_equal(f, freq)
    assert np.array_equal((ms & 0xFFFF).astype(np.int32), mu_idx)
    assert np.array_equal((ms >> 16).astype(np.int32), sc_idx)
    # bits = fp32(24 - log2(f64(freq))) to one ulp
    bits = r["bits"].cpu().numpy()
    want = (24.0 - np.log2(freq.astype(np.float64))).astype(np.float32)
    assert np.all(np.abs(bits.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64)) <= 1)
    # grid sums: f64, against a host sum, identical on a second run
    exact = 24.0 - np.log2(freq.astype(np.float64))
    host = [float(m.sum()) for m in _grid_maps(desc, exact)]
    np.testing.assert_allclose(r["grid_bits"], host, rtol=1e-12, atol=1e-9)
    r2 = ctx.latent_rate([desc], [nn], [lat], want_spatial=True)[0]
    assert r2["grid_bits"] == r["grid_bits"]
    # spatial map: bit-equal to the canonical restatement
    sp = spatial_canonical(_grid_maps(desc, bits), desc.img_h, desc.img_w)
    assert np.array_equal(r["spatial"][0, 0].cpu().numpy(), sp)
    assert np.array_equal(r2["spatial"].cpu().numpy(), r["spatial"].cpu().numpy())
    return r


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["kodim14"] + GENERIC_ARM)
def test_rate_equals_checker(ctx, oracle, name):
    from coolchic_b200._desc import desc_from_header

    (h, nb, lb), = _coolchics(_golden(name))[:1]
    d = desc_from_header(h)
    r = _check_against_checker(ctx, oracle, d, nb, lb)
    assert sum(r["grid_bits"]) <= 8 * len(lb)


@pytest.mark.gpu
def test_rate_1080p_seven_grids(ctx, oracle, seed_stream):
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    data = synth.make_image_stream(ctx, seed_stream, 1080, 1920)
    (h, nb, lb), = _coolchics(data)
    d = desc_from_header(h)
    assert d.n_grids == 7
    r = _check_against_checker(ctx, oracle, d, nb, lb)
    assert 0 <= 8 * len(lb) - sum(r["grid_bits"]) < 0.001 * 8 * len(lb)


@pytest.mark.gpu
def test_rate_batch_one_launch(ctx):
    """2 x SM + 5 Cool-chics of different ARM variants in one call: one rate launch (plus one for the spatial
    maps), and every job's result equals the job run alone."""
    from coolchic_b200 import _native
    from coolchic_b200._desc import desc_from_header

    pool = [c for n in ["kodim14"] + GENERIC_ARM + ["gop5_64x96_yuv420"] for c in _coolchics(_golden(n))]
    import torch

    n_sm = torch.cuda.get_device_properties(ctx.device).multi_processor_count
    items = [pool[i % len(pool)] for i in range(2 * n_sm + 5)]
    descs = [desc_from_header(h) for h, _, _ in items]
    _, lats = ctx.decode_many(descs, [nb for _, nb, _ in items], [lb for _, _, lb in items], want_latents=True)
    nns = [_native.decode_nn(d, nb) for d, (_, nb, _) in zip(descs, items)]
    n0 = ctx.launch_count()
    res = ctx.latent_rate(descs, nns, lats, want_freq=True)
    assert ctx.launch_count() - n0 == 1
    n0 = ctx.launch_count()
    res_sp = ctx.latent_rate(descs, nns, lats, want_spatial=True)
    assert ctx.launch_count() - n0 == 2
    for i in range(len(pool)):
        alone = ctx.latent_rate([descs[i]], [nns[i]], [lats[i]], want_freq=True, want_spatial=True)[0]
        assert np.array_equal(alone["freq"].cpu().numpy(), res[i]["freq"].cpu().numpy())
        assert alone["grid_bits"] == res[i]["grid_bits"] == res_sp[i]["grid_bits"]
        assert np.array_equal(alone["spatial"].cpu().numpy(), res_sp[i]["spatial"].cpu().numpy())


@pytest.mark.gpu
def test_video_rate_gop(ctx, oracle):
    """Residue and motion Cool-chics of a GOP: frame header + Cool-chic totals = 8 x the frame's bytes, and the
    frames (plus the video header) make the whole file."""
    from coolchic_b200.bitstream import rate
    from coolchic_b200.bitstream.header import VideoHeader

    from coolchic_b200._desc import desc_from_header

    data = _golden("gop5_64x96_yuv420")
    ccs = _coolchics(data)
    n0 = ctx.launch_count()
    ctx.decode_many([desc_from_header(h) for h, _, _ in ccs], [nb for _, nb, _ in ccs], [lb for _, _, lb in ccs],
                    want_latents=True)
    n_decode = ctx.launch_count() - n0
    n0 = ctx.launch_count()
    fr = rate.video_rate(data)
    assert ctx.launch_count() - n0 == n_decode + 2  # one decode of every Cool-chic, one rate + one spatial launch
    assert list(fr) == [str(i) for i in range(5)]
    total = 0
    for f in fr.values():
        assert f.total_bits == 8 * f.n_bytes
        assert set(f.coolchics) == ({"residue"} if f.frame_type == "I" else {"residue", "motion"})
        for c in f.coolchics.values():
            assert sum(sum(v.values()) for v in c.nn_bits.values()) + c.nn_pad_bits == c.nn_payload_bits
            assert 0 <= c.latent_payload_bits - c.latent_model_bits < 3 * 32
            assert c.spatial_rate_bit.shape == (1, 1) + c.img_size
            assert [tuple(m.shape[-2:]) for m in c.rate_bit] == c.grid_sizes
        total += f.n_bytes
    v = VideoHeader()
    v.read_header(data)
    assert total + v.get_value("n_bytes_header") == len(data)


@pytest.mark.gpu
def test_coolchic_rate_maps(ctx, kodim14):
    """coolchic_rate: per-grid maps, the mu / scale the coder used, NN bits, header and payload bits."""
    import torch

    from coolchic_b200.bitstream import rate

    r = rate.coolchic_rate(kodim14["header"], kodim14["nn_bytes"], kodim14["lat_bytes"])
    d = kodim14["desc"]
    assert len(r.rate_bit) == len(r.mu) == len(r.scale) == d.n_grids
    assert r.latent_payload_bits == 247616
    assert sum(r.grid_bits) == pytest.approx(247540.28993988558, rel=1e-12)
    for g in range(d.n_grids):
        assert float(r.rate_bit[g].double().sum()) == pytest.approx(r.grid_bits[g], rel=1e-6)
    tab = torch.from_numpy(rate.scale_table())
    assert bool(torch.isin(r.scale[0].cpu().flatten(), tab).all())
    assert bool(((r.mu[0] * 256).round() == r.mu[0] * 256).all())
    assert r.header_bits == 8 * kodim14["header"].get_value("n_bytes_header")


@pytest.mark.gpu
@pytest.mark.parametrize("bad", [-65, 64])
def test_latent_out_of_range_is_an_argument_error(ctx, kodim14, bad):
    from coolchic_b200 import _native

    d = kodim14["desc"]
    nn = _native.decode_nn(d, kodim14["nn_bytes"])
    lat = __import__("torch").from_numpy(kodim14["latents"].copy()).cuda()
    idx = 123457
    lat[idx] = bad
    with pytest.raises(_native.CcdError) as e:
        ctx.latent_rate([d], [nn], [lat])
    assert e.value.code == -1 and e.value.bad_index == [idx]
    assert "outside [-64, 63]" in str(e.value)
