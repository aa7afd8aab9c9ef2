"""Frames wider than 5070 pixels on the device: the entropy kernel's window ring shrinks (1024 -> 512 slots) so that
it fits beside the row ring those widths need, and past width 10236 the row ring has 2048 rows, whose byte index
needs 17 bits of the meta word.  Every stream here is at least that wide; each is checked against the oracle."""
import os
import sys

import numpy as np
import pytest
from conftest import ROOT

pytestmark = pytest.mark.gpu


def _stream(ctx, seed_stream, hw, lr, seed, overrides=None):
    """-> (desc, nn bytes, latent payload, device latents) of one synthetic Cool-chic."""
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    cc, h, lat_dev = synth.make_coolchic(ctx, seed_stream, hw, lr, None, seed=seed, overrides=overrides)
    h2 = type(h)()
    rest = h2.read_header(cc)
    n_nn, n_lat = h2.get_value("nn_n_bytes"), h2.get_value("n_bytes_latent")
    return desc_from_header(h2), rest[:n_nn], rest[n_nn:n_nn + n_lat], lat_dev


def _longest_diagonal(d):
    return max(1 if d.grid_w[g] <= 9 else min(d.grid_h[g], -(-d.grid_w[g] // 10)) for g in range(d.n_grids))


@pytest.mark.parametrize("hw,lr,fmt,plan", [((2880, 5120), (0, 7), "rgb", (512, 1024)),
                                            ((4320, 7680), (0, 8), "yuv420", (512, 1024))],
                         ids=["5k-8grids-rgb", "8k-9grids-yuv420"])
def test_wide_full_size_parity(ctx, oracle, seed_stream, hw, lr, fmt, plan):
    """As test_full_size_parity at 5K and 8K: every word consumed, round trip, payload idempotence; latents, raw
    synthesis output and finished frame identical to the oracle's, whole frame.  At 8K the 768-symbol diagonals of
    the finest grid run through a 512-slot ring."""
    import torch

    from coolchic_b200 import _native

    d, nn_bytes, payload, lat_dev = _stream(ctx, seed_stream, hw, lr, seed=1)
    nn = oracle.decode_nn(d, nn_bytes)
    assert _native.entropy_plan(d, nn)[:2] == plan
    if hw[1] == 7680:
        assert _longest_diagonal(d) == 768 > plan[0]
    out, lat = ctx.decode_coolchic(d, nn_bytes, payload, want_latents=True)
    torch.cuda.synchronize()
    st = ctx.last_status()
    assert st[0] == 0 and st[1] == len(payload) // 4 + 1  # every word consumed, one over-read
    assert torch.equal(lat, lat_dev)                       # encode -> decode round trip
    _, payload2, _ = ctx.encode_latents(d, nn, latents=lat)
    assert payload2 == payload                             # re-encoding reproduces the payload
    oracle.set_threads(0)
    lat_o, _ = oracle.decode_latents(d, nn, payload)
    assert np.array_equal(lat.cpu().numpy(), lat_o)
    raw_o = oracle.synthesize(d, nn, lat_o)
    assert np.array_equal(out[0].cpu().numpy(), raw_o)
    del out
    want = oracle.finish_frame(raw_o, 8, fmt)
    del raw_o
    fin, _ = ctx.decode_many([d], [nn_bytes], [payload], finish=[(8, fmt)])
    if fmt == "yuv420":
        for k in "yuv":
            assert np.array_equal(fin[0][k][0, 0].cpu().numpy(), want[k]), k
    else:
        assert np.array_equal(fin[0][0].cpu().numpy(), want)


def test_widest_frame_latents(ctx, oracle, seed_stream):
    """16383 x 1040, the widest frame the header can describe: a 2048-row ring, rows past index 1024 (the meta word's
    24-bit row index)."""
    import torch

    from coolchic_b200 import _native

    d, nn_bytes, payload, lat_dev = _stream(ctx, seed_stream, (1040, 16383), (0, 6), seed=4)
    nn = oracle.decode_nn(d, nn_bytes)
    assert _native.entropy_plan(d, nn)[:2] == (512, 2048)
    lat = ctx.decode_latents(d, nn, payload)
    torch.cuda.synchronize()
    assert ctx.last_status()[0] == 0
    assert torch.equal(lat, lat_dev)
    oracle.set_threads(0)
    lat_o, _ = oracle.decode_latents(d, nn, payload)
    assert np.array_equal(lat.cpu().numpy(), lat_o)


def test_wide_generic_arm(ctx, oracle, seed_stream):
    """The all-int64 kernel (8 contexts, 1 hidden layer, as img_48x64_rgb_arm8_1hidden) at 5200 x 240."""
    import torch

    from coolchic_b200 import _native

    ov = {"spatial_context_arm": 8, "n_hidden_layers_arm": 1}
    d, nn_bytes, payload, lat_dev = _stream(ctx, seed_stream, (240, 5200), (0, 4), seed=6, overrides=ov)
    nn = oracle.decode_nn(d, nn_bytes)
    assert _native.entropy_plan(d, nn)[:2] == (512, 1024)
    fin, lats = ctx.decode_many([d], [nn_bytes], [payload], want_latents=True, finish=[(8, "rgb")])
    torch.cuda.synchronize()
    assert torch.equal(lats[0], lat_dev)
    lat_o, _ = oracle.decode_latents(d, nn, payload)
    assert np.array_equal(lats[0].cpu().numpy(), lat_o)
    want = oracle.finish_frame(oracle.synthesize(d, nn, lat_o), 8, "rgb")
    assert np.array_equal(fin[0][0].cpu().numpy(), want)


def test_wide_gop_decode_rate_quality(ctx, oracle, seed_stream, tmp_path, monkeypatch):
    """A 5120 x 240 yuv420 I-B-P GOP: decode_video_bytes equals the oracle's chain frame by frame; video_rate and
    video_quality run on it with their invariants (model bits <= payload bits, exact SSE)."""
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    import pipeline  # the oracle's whole-stream decode (test infrastructure)

    from coolchic_b200 import synth
    from coolchic_b200.bitstream.decode import decode_video_bytes
    from coolchic_b200.bitstream.quality import video_quality
    from coolchic_b200.bitstream.rate import video_rate

    n, h, w = 3, 240, 5120
    data = synth.make_video_stream(ctx, seed_stream, h, w, n, "yuv420", 8, 8, seed=7)
    frames = decode_video_bytes(data)
    oracle.set_threads(0)
    want = pipeline.decode_video(data)
    dec = []
    for i in range(n):
        fmt, bd, planes = want[i]
        assert (fmt, bd) == ("yuv420", 8)
        for c in "yuv":
            assert np.array_equal(frames[str(i)].data[c][0, 0].numpy(), planes[c]), (i, c)
        dec.append([np.rint(planes[c].astype(np.float32) * np.float32(255)).astype(np.int64) for c in "yuv"])

    fr = video_rate(data)
    assert sorted(fr, key=int) == [str(i) for i in range(n)]
    for f in fr.values():
        assert f.total_bits == 8 * f.n_bytes
        for c in f.coolchics.values():
            # the range coder's truncation costs a fraction of a bit per thousand symbols
            assert 0 <= c.latent_payload_bits - c.latent_model_bits < 0.001 * c.latent_payload_bits
            assert c.spatial_rate_bit.shape == (1, 1) + c.img_size

    rng = np.random.default_rng(11)
    src = [[np.clip(p + rng.integers(-3, 4, size=p.shape), 0, 255) for p in fr_] for fr_ in dec]
    monkeypatch.chdir(tmp_path)  # bare names: the naming rules (_8b, 444) read the whole path
    path = f"src_{w}x{h}_30p_yuv420_8b.yuv"
    np.concatenate([np.concatenate([p.reshape(-1) for p in fr_]) for fr_ in src]).astype(np.uint8).tofile(path)
    q = video_quality(data, path)
    assert sorted(q, key=int) == [str(i) for i in range(n)]
    for k, fq in q.items():
        d_ = [a - b for a, b in zip(dec[int(k)], src[int(k)])]
        assert fq.sse == [int((x * x).sum()) for x in d_]
        assert fq.max_abs == [int(np.abs(x).max()) for x in d_]


def test_wide_stream_in_a_full_batch(ctx, seed_stream):
    """One decode_many call with 133 Kodak-size streams and one 6000 x 400 stream of the same architecture: more
    streams than SMs, but the wide stream's shared memory keeps the group at one CTA per SM.  Every output equals
    its single-stream decode."""
    import torch

    from coolchic_b200 import _native

    small = [_stream(ctx, seed_stream, (512, 768), (0, 6), seed=20 + i) for i in range(12)]
    wide = _stream(ctx, seed_stream, (400, 6000), (0, 6), seed=40)
    assert _native.entropy_plan(wide[0], _native.decode_nn(wide[0], wide[1]))[:2] == (512, 1024)
    items = [small[i % len(small)] for i in range(133)]
    items.insert(67, wide)
    outs, lats = ctx.decode_many([x[0] for x in items], [x[1] for x in items], [x[2] for x in items],
                                 want_latents=True, finish=[(8, "rgb")] * len(items))
    torch.cuda.synchronize()
    alone = {}
    for i, (d, nnb, lb, lat_in) in enumerate(items):
        key = id(items[i])
        if key not in alone:
            o, l_ = ctx.decode_many([d], [nnb], [lb], want_latents=True, finish=[(8, "rgb")])
            alone[key] = (o[0], l_[0])
        assert torch.equal(lats[i], lat_in), i
        assert torch.equal(lats[i], alone[key][1]), i
        assert torch.equal(outs[i], alone[key][0]), i
