"""Synthetic Cool-chic bitstreams (SURVEY 8d / 8f2): no encoder can be trained here, so the
benchmark inputs are fabricated from the shipped 768x512 sample stream:

  * latents: the sample's decoded latent grids, TILED to the target grid sizes level by level
    (periods 512/2^i x 768/2^i keep the cross-level alignment), rolled by a per-seed offset;
    they keep natural-image statistics, so the ARM sees realistic contexts and rates
    (sampling the ARM free-running diverges: mean |x| ~ 45 instead of 0.3);
  * networks: the sample's integers, re-shaped where the target architecture differs
    (IFCE inputs truncated / zero-padded, upsampling kernels cycled, synthesis input widened);
  * payload: range-ENcoded on the device by libccdec (``ccd_encode_latents``), NN integers
    exp-Golomb coded, headers written with the host header classes.

Writer side of the reference: ``coolchic/bitstream/encode.py:24-95``,
``neuralnet/neuralnet.py:26-89``, ``neuralnet/expgolomb.py:15-71``, ``header/header.py:90-105``.
"""
import os
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from ._desc import CcdCoolChicDesc, desc_from_header
from .bitstream.expgolomb import encode_exp_golomb
from .bitstream.header import (NN_KINDS, NN_MODULES, CoolChicHeader, DescriptorCoolChic, FrameHeader, VideoHeader)

SEED_STREAM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "seed_768x512.cool")


def parse_single_image(data: bytes):
    """-> (VideoHeader, FrameHeader, CoolChicHeader, nn_bytes, latent_bytes) of a 1-frame intra stream."""
    v = VideoHeader()
    rest = v.read_header(data)
    f = FrameHeader()
    rest = f.read_header(rest)
    c = CoolChicHeader()
    rest = c.read_header(rest)
    n_nn, n_lat = c.get_value("nn_n_bytes"), c.get_value("n_bytes_latent")
    return v, f, c, rest[:n_nn], rest[n_nn:n_nn + n_lat]


# ---- NN integer layout (module order arm, ifce, upsampling, synthesis; weights then biases) ----
def nn_sections(d: CcdCoolChicDesc) -> Dict[str, List[Tuple[str, Tuple[int, ...]]]]:
    """Named tensors with shapes, per (module, kind), in bitstream order (SURVEY 3.2)."""
    dim = d.n_ctx + d.n_ifce_out
    cf = d.n_ifce_out
    sec: Dict[str, List[Tuple[str, Tuple[int, ...]]]] = {f"{m}.{k}": [] for m in NN_MODULES for k in NN_KINDS}
    for l in range(d.arm_hidden):
        sec["arm.weight"].append((f"mlp.{2 * l}", (dim, dim)))
        sec["arm.bias"].append((f"mlp.{2 * l}", (dim,)))
    sec["arm.weight"].append((f"mlp.{2 * d.arm_hidden}", (2, dim)))
    sec["arm.bias"].append((f"mlp.{2 * d.arm_hidden}", (2,)))
    if d.arm_stab:
        sec["arm.weight"].append(("stab", (2, dim)))
        sec["arm.bias"].append(("stab", (2,)))
    if d.flag_ifce:
        for g in range(d.n_grids):
            if d.grid_ifce_in[g] > 0:
                sec["ifce.weight"].append((f"grid{g}", (cf, d.grid_ifce_in[g])))
                sec["ifce.bias"].append((f"grid{g}", (cf,)))
    kt, kc = (d.ups_k + 1) // 2, (d.ups_pre_k + 1) // 2
    for i in range(d.n_ups):
        sec["upsampling.weight"].append((f"convt{i}", (kt,)))
    for i in range(d.n_ups):
        sec["upsampling.weight"].append((f"conv{i}", (kc,)))
    for i in range(2 * d.n_ups):
        sec["upsampling.bias"].append((f"b{i}", (1,)))
    C = d.syn_out[d.n_syn_layers - 1]
    stab_in = d.syn_in // 2 if d.common_randomness else d.syn_in
    sec["synthesis.weight"].append(("out", (C, C)))
    sec["synthesis.bias"].append(("out", (C,)))
    if d.syn_stab:
        sec["synthesis.weight"].append(("stab", (C, stab_in)))
        sec["synthesis.bias"].append(("stab", (C,)))
    cin = d.syn_in
    for l in range(d.n_syn_layers):
        sec["synthesis.weight"].append((f"l{l}", (d.syn_out[l], cin, d.syn_k[l], d.syn_k[l])))
        sec["synthesis.bias"].append((f"l{l}", (d.syn_out[l],)))
        cin = d.syn_out[l]
    return sec


def split_nn(d: CcdCoolChicDesc, ints: np.ndarray) -> Dict[str, Dict[str, np.ndarray]]:
    out, p = {}, 0
    for key, items in nn_sections(d).items():
        out[key] = {}
        for name, shape in items:
            n = int(np.prod(shape))
            out[key][name] = np.asarray(ints[p:p + n], dtype=np.int64).reshape(shape)
            p += n
    assert p == len(ints), (p, len(ints))
    return out


def join_nn(d: CcdCoolChicDesc, tensors: Dict[str, Dict[str, np.ndarray]]) -> Tuple[np.ndarray, List[int]]:
    vals, counts = [], []
    j = 0
    for m in NN_MODULES:
        for k in NN_KINDS:
            for name, shape in nn_sections(d)[f"{m}.{k}"]:
                t = np.asarray(tensors[f"{m}.{k}"][name], dtype=np.int64)
                assert t.shape == tuple(shape), (m, k, name, t.shape, shape)
                vals.append(t.reshape(-1))
                counts += [int(d.expgol[j])] * t.size
            j += 1
    return np.concatenate(vals), counts


def _fit(src: np.ndarray, shape: Sequence[int]) -> np.ndarray:
    """Copy the overlapping block of src into a zero tensor of the requested shape."""
    out = np.zeros(shape, dtype=np.int64)
    sl = tuple(slice(0, min(a, b)) for a, b in zip(src.shape, shape))
    out[sl] = src[sl]
    return out


def _source(src: Dict[str, Dict[str, np.ndarray]], key: str, idx: int, name: str) -> Optional[np.ndarray]:
    """The sample's tensor that adapt_nn copies into tensor ``name`` (position ``idx`` of section ``key``), or None."""
    src_names = list(src[key].keys())
    if name in src[key]:
        return src[key][name]
    if key.startswith("ifce") and src_names:
        return src[key][src_names[min(idx, len(src_names) - 1)]]
    if key.startswith("upsampling") and src_names:
        kind = [n for n in src_names if n.rstrip("0123456789") == name.rstrip("0123456789")] or src_names
        return src[key][kind[idx % len(kind)]]
    return None


def adapt_nn(src_d: CcdCoolChicDesc, src_ints: np.ndarray, dst_d: CcdCoolChicDesc) -> np.ndarray:
    """Re-shape the sample's network integers for another architecture of the same family.  Every entry the sample
    does not have is zero (liven_nn fills them)."""
    src = split_nn(src_d, src_ints)
    dst: Dict[str, Dict[str, np.ndarray]] = {}
    for key, items in nn_sections(dst_d).items():
        dst[key] = {}
        for idx, (name, shape) in enumerate(items):
            cand = _source(src, key, idx, name)
            if cand is None:
                cand = np.zeros(shape, dtype=np.int64)
            dst[key][name] = _fit(cand, shape) if cand.shape != tuple(shape) else cand.copy()
    if dst_d.common_randomness and not src_d.common_randomness:
        # the noise half of the synthesis input gets (attenuated) copies of the latent half's weights
        w0 = dst["synthesis.weight"]["l0"]
        half = dst_d.syn_in // 2
        w0[:, half:] = w0[:, :half] // 3 + 1
    ints, _ = join_nn(dst_d, dst)
    return ints


def liven_nn(src_d: CcdCoolChicDesc, src_ints: np.ndarray, dst_d: CcdCoolChicDesc, seed: int) -> np.ndarray:
    """adapt_nn with every entry it padded made live: residue channels 3 and 4, the second flow, synthesis units past
    the sample's width, latent grids past its count and ARM units past its 14 + 6 otherwise only ever meet zero
    weights.  A padded entry gets a value drawn from the nonzero values of the same tensor (of its section, when the
    tensor has none) with a random sign; the sample's own zeros stay zero."""
    src = split_nn(src_d, src_ints)
    dst = split_nn(dst_d, adapt_nn(src_d, src_ints, dst_d))
    rng = np.random.default_rng(seed)
    for key, items in nn_sections(dst_d).items():
        for idx, (name, shape) in enumerate(items):
            t = dst[key][name]
            cand = _source(src, key, idx, name)
            pad = np.ones(t.shape, dtype=bool)
            if cand is not None:
                pad[tuple(slice(0, min(a, b)) for a, b in zip(cand.shape, t.shape))] = False
            if key == "synthesis.weight" and name == "l0" and dst_d.common_randomness and not src_d.common_randomness:
                pad[:, dst_d.syn_in // 2:] = pad[:, :dst_d.syn_in // 2]  # adapt_nn's copies of the latent half
            if not pad.any():
                continue
            pool = np.abs(t[t != 0])
            if pool.size == 0:
                pool = np.abs(np.concatenate([v[v != 0] for v in dst[key].values()] + [np.ones(1, np.int64)]))
            n = int(pad.sum())
            t[pad] = rng.choice(pool, size=n) * rng.choice(np.array([-1, 1]), size=n)
    ints, _ = join_nn(dst_d, dst)
    return ints


# 5th / 95th percentiles the output channels are moved to by scale_outputs, per kind of Cool-chic; channels 3 / 4 of a
# residue are alpha / beta - 0.5, so that alpha and beta have samples below 0, inside (0, 1) and above 1; a motion
# Cool-chic's outputs are flows in pixels
OUTPUT_TARGETS = {"intra": [(-0.06, 1.06)] * 3,
                  "residue": [(-0.45, 0.45)] * 3 + [(-0.8, 0.8)] * 2,
                  "motion": [(-3.5, 3.5)] * 4}


def scale_outputs(desc: CcdCoolChicDesc, ints: np.ndarray, raw: np.ndarray, kind: str) -> np.ndarray:
    """The network integers with every output channel c mapped affinely so that its 5th / 95th percentiles (on ``raw``,
    the unmodified output [C, H, W]) go to about OUTPUT_TARGETS[kind][c]: rows of the output transform scaled, its
    biases shifted."""
    t = split_nn(desc, ints)
    w, b = t["synthesis.weight"]["out"], t["synthesis.bias"]["out"]
    qb = 2.0 ** desc.qshift[NN_MODULES.index("synthesis") * len(NN_KINDS) + NN_KINDS.index("bias")]
    for c in range(w.shape[0]):
        lo, hi = OUTPUT_TARGETS[kind][c]
        p5, p95 = np.percentile(raw[c].astype(np.float64), [5, 95])
        a = (hi - lo) / max(p95 - p5, 1e-3)
        w[c] = np.round(a * w[c])
        b[c] = int(round(a * b[c] + (lo - a * p5) / qb))
    out, _ = join_nn(desc, t)
    return out


# ---- latents ---------------------------------------------------------------------------------
def _level_of(d: CcdCoolChicDesc, g: int) -> int:
    return int(round(np.log2(max(1.0, d.img_h / d.grid_h[g])))) if d.grid_h[g] < d.img_h else 0


def tile_latents(src_d: CcdCoolChicDesc, src_lat: torch.Tensor, dst_d: CcdCoolChicDesc, seed: int = 0) -> torch.Tensor:
    """Tile the sample's latent grids (int8, decode order) to the target's grid sizes."""
    def offsets(d):
        off, p = {}, 0
        for g in range(d.n_grids - 1, -1, -1):
            off[g] = p
            p += d.grid_h[g] * d.grid_w[g]
        return off, p

    s_off, _ = offsets(src_d)
    d_off, d_total = offsets(dst_d)
    # source grids by (level, is_hyper); level = position among the distinct resolutions
    def levels(d):
        lv, cur, prev = {}, -1, None
        for g in range(d.n_grids):
            size = (d.grid_h[g], d.grid_w[g])
            if size != prev:
                cur += 1
                prev = size
            lv[g] = cur + d.latent_res_lo if not d.grid_is_hyper[g] or True else cur
        return lv
    s_lv, d_lv = levels(src_d), levels(dst_d)
    by_key = {}
    for g in range(src_d.n_grids):
        by_key[(s_lv[g], bool(src_d.grid_is_hyper[g]))] = g
    max_lv = max(s_lv.values())
    rng = np.random.default_rng(1234 + seed)
    roll_y, roll_x = (int(rng.integers(0, 8)) * 64, int(rng.integers(0, 12)) * 64) if seed else (0, 0)
    out = torch.empty((d_total,), dtype=torch.int8, device=src_lat.device)
    for g in range(dst_d.n_grids):
        lv = min(d_lv[g], max_lv)
        key = (lv, bool(dst_d.grid_is_hyper[g]))
        sg = by_key.get(key, by_key.get((lv, False), src_d.n_grids - 1))
        hs, ws = src_d.grid_h[sg], src_d.grid_w[sg]
        src = src_lat[s_off[sg]: s_off[sg] + hs * ws].view(hs, ws)
        hd, wd = dst_d.grid_h[g], dst_d.grid_w[g]
        ys = (torch.arange(hd, device=src.device) + (roll_y >> lv)) % hs
        xs = (torch.arange(wd, device=src.device) + (roll_x >> lv)) % ws
        out[d_off[g]: d_off[g] + hd * wd] = src[ys][:, xs].reshape(-1)
    return out


# ---- stream assembly -------------------------------------------------------------------------
def make_coolchic_header(template: CoolChicHeader, img_size: Tuple[int, int], latent_resolution: Tuple[int, int],
                         hyperlatent_resolution: Optional[Tuple[int, int]], final_upsampling_type: Optional[str] = None,
                         overrides: Optional[dict] = None) -> CoolChicHeader:
    h = CoolChicHeader()
    for f in template._all_fields():
        if f[1] in template._values:
            h._values[f[1]] = template._values[f[1]]
    h._values["img_size"] = list(img_size)
    h._values["latent_resolution"] = list(latent_resolution)
    h._values["flag_hyperlatent"] = int(hyperlatent_resolution is not None)
    if hyperlatent_resolution is not None:
        h._values["hyperlatent_resolution"] = list(hyperlatent_resolution)
    else:
        h._values.pop("hyperlatent_resolution", None)
    if final_upsampling_type is not None:
        h._values["final_upsampling_type"] = final_upsampling_type
    for k, v in (overrides or {}).items():
        h._values[k] = v
    if h._values.get("output_feature_ifce", 0) > 0 and "ifce_resolution" not in h._values:
        h._values["ifce_resolution"] = [0, 2]
    p = h.get_coolchic_parameter()
    h._values["n_latent_grids"] = p.n_latent_grids
    h._values["nn_n_bytes"] = 0
    h._values["nn_n_bit_pad"] = 0
    h._values["n_bytes_latent"] = 0
    return h


class SeedStream:
    """The shipped 768x512 sample, decoded once (latents + network integers).

    ``ctx`` is a ``_native.Context`` (device) -- or any object with the same three methods
    ``decode_nn(desc, bytes)``, ``decode_latents(desc, nn, bytes)``, ``encode_latents(desc, nn, latents=)``
    (the CPU tests pass an oracle-backed one)."""

    def __init__(self, ctx, path: str = SEED_STREAM):
        with open(path, "rb") as f:
            data = f.read()
        self.video, self.frame, self.header, nn_bytes, lat_bytes = parse_single_image(data)
        self.desc = desc_from_header(self.header)
        if hasattr(ctx, "decode_nn"):
            self.nn = ctx.decode_nn(self.desc, nn_bytes)
        else:
            from . import _native

            self.nn = _native.decode_nn(self.desc, nn_bytes)
        self.latents = ctx.decode_latents(self.desc, self.nn, lat_bytes)


def make_coolchic(ctx, seed_stream: SeedStream, img_size, latent_resolution=(0, 6), hyperlatent_resolution=None,
                  seed: int = 0, final_upsampling_type=None, overrides=None, latents: Optional[torch.Tensor] = None,
                  nn: Optional[np.ndarray] = None,
                  live: Optional[str] = None) -> Tuple[bytes, CoolChicHeader, torch.Tensor]:
    """One Cool-chic section (header + NN payload + latent payload) for an image of ``img_size``.  ``nn``: the
    network integers to write (in bitstream order, for the header's architecture) instead of the sample's.
    ``live`` ("intra", "residue" or "motion"): the sample's network through liven_nn (seeded by ``seed``), its outputs
    then moved by scale_outputs to look like those of that kind of Cool-chic, measured on ``ctx.synthesize``."""
    header = make_coolchic_header(seed_stream.header, img_size, latent_resolution, hyperlatent_resolution,
                                  final_upsampling_type, overrides)
    desc = desc_from_header(header)
    if latents is None:
        latents = tile_latents(seed_stream.desc, seed_stream.latents, desc, seed)
    if nn is None and live is not None:
        nn = liven_nn(seed_stream.desc, seed_stream.nn, desc, seed)
        raw = ctx.synthesize([desc], [nn], [latents], [0])[0][0].cpu().numpy()
        nn = scale_outputs(desc, nn, raw, live)
    elif nn is None:
        nn = adapt_nn(seed_stream.desc, seed_stream.nn, desc)
    nn = np.asarray(nn, dtype=np.int64)
    _, counts = join_nn(desc, split_nn(desc, nn))
    nn_bytes, pad = encode_exp_golomb(nn.tolist(), counts)
    header.set_value("nn_n_bytes", len(nn_bytes))
    header.set_value("nn_n_bit_pad", pad)
    desc = desc_from_header(header)
    lat_dev, payload, _ = ctx.encode_latents(desc, nn, latents=latents)
    header.set_value("n_bytes_latent", len(payload))
    return header.to_bytes() + nn_bytes + payload, header, lat_dev


def make_image_stream(ctx, seed_stream: SeedStream, height: int, width: int, frame_data_type: str = "rgb",
                      bitdepth: int = 8, latent_resolution=(0, 6), hyperlatent_resolution=None, seed: int = 0,
                      final_upsampling_type: Optional[str] = None, overrides: Optional[dict] = None,
                      live: bool = False) -> bytes:
    """A complete single-frame (intra) bitstream.  ``overrides`` sets Cool-chic header fields, e.g.
    ``{"flag_common_randomness": 1}``; ``final_upsampling_type`` matters when latent_resolution[0] > 0.  ``live``:
    every weight of the network live (make_coolchic)."""
    v = VideoHeader()
    v.set_header(1, [0], [])
    f = FrameHeader()
    f._values.update(display_index=0, frame_type="I", frame_data_type=frame_data_type, bitdepth=bitdepth,
                     index_references=[], global_flow=[])
    cc, _, _ = make_coolchic(ctx, seed_stream, (height, width), latent_resolution, hyperlatent_resolution, seed,
                             final_upsampling_type, overrides, live="intra" if live else None)
    return v.to_bytes() + f.to_bytes() + cc


# ---- video (I / P / hierarchical B) -------------------------------------------------------------
def _syn_overrides(width: int, out_ch: int, n_layers: int) -> dict:
    layers = [f"{width}-1-linear-relu", f"{out_ch}-1-linear-none", f"{out_ch}-3-residual-relu",
              f"{out_ch}-3-residual-none"][:n_layers]
    ov = {"n_layer_synthesis": n_layers}
    for i, lay in enumerate(layers):
        ov[f"syn_layer_{i}"] = lay
    return ov


def make_video_stream(ctx, seed_stream: SeedStream, height: int, width: int, n_frames: int,
                      frame_data_type: str = "yuv420", bitdepth: int = 8, warp_filter_size: int = 8,
                      seed: int = 0, live: bool = False) -> bytes:
    """A GOP: I frame, last frame P, hierarchical B in between (codingstructure.py:267-436).
    Architectures follow cfg/dec: intra = hop; residue of P/B = mop widths (ARM 10+2, 16-wide
    synthesis, 4 / 5 output channels); motion = mop (latent_resolution 2-6, ARM 6+2, 16-wide
    synthesis with 2 / 4 outputs, nearest final upsampling).  ``live``: every weight of every network live, with
    residue alpha / beta and flows that vary (make_coolchic)."""
    from .utils.codingstructure import CodingStructure

    p_pos = [n_frames - 1] if n_frames > 1 else []
    cs = CodingStructure(n_frames=n_frames, intra_pos=[0], p_pos=p_pos)
    v = VideoHeader()
    v.set_header(n_frames, [0], p_pos)
    out = v.to_bytes()
    rng = np.random.default_rng(4321 + seed)
    for coding_idx in range(n_frames):
        fr = cs.get_frame_from_coding_order(coding_idx)
        f = FrameHeader()
        n_ref = len(fr.index_references)
        gflow = [int(g) for g in rng.integers(-6, 7, size=2 * n_ref)]
        f._values.update(display_index=fr.display_order, frame_type=fr.frame_type, frame_data_type=frame_data_type,
                         bitdepth=bitdepth, index_references=list(fr.index_references), global_flow=gflow)
        if n_ref:
            f._values["warp_filter_size"] = warp_filter_size
        out += f.to_bytes()
        s = 100 * seed + coding_idx
        if fr.frame_type == "I":
            cc, _, _ = make_coolchic(ctx, seed_stream, (height, width), (0, 6), None, seed=s,
                                     live="intra" if live else None)
            out += cc
        else:
            ov = {"spatial_context_arm": 10, "output_feature_ifce": 2}
            ov.update(_syn_overrides(16, 3 + n_ref, 4))
            cc, _, _ = make_coolchic(ctx, seed_stream, (height, width), (0, 6), None, seed=s, overrides=ov,
                                     live="residue" if live else None)
            out += cc
            ov = {"spatial_context_arm": 6, "output_feature_ifce": 2, "ifce_resolution": [2, 2]}
            ov.update(_syn_overrides(16, 2 * n_ref, 2))
            cc, _, _ = make_coolchic(ctx, seed_stream, (height, width), (2, 6), None, seed=s + 50,
                                     final_upsampling_type="nearest", overrides=ov, live="motion" if live else None)
            out += cc
    return out
