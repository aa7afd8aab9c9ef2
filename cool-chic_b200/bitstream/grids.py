"""Latent-grid analysis of a bitstream: what each latent grid of a ``.cool`` file costs and what it buys.

Per frame and per Cool-chic (the residue, and the motion of P / B frames), one row per latent grid with its model bits
(``ccd_latent_rate``, the numbers of ``video_rate``) and, for a synthesis grid, the quality of the frame re-synthesised
with that grid read as all zeros (**drop**).  For the residue also the progressive view (**coarse**): the frame PSNR
when only the n coarsest synthesis grids are kept, n = 1 .. nl - 1, reported in the row of the finest grid kept.
Hyperlatent grids only feed the entropy model; their rows carry bits and no distortion.  DESIGN §4.7.

The video is decoded once through ``decode_video_bytes``, keeping the latents; every variant is the float tail of
decoding on those latents with some grids masked (``ccd_synthesize_many``).  A P / B variant is reconstructed with the
frame's decoded, unmodified references, so a variant does not drift into later frames.  Per frame, one
``ccd_synthesize_many`` call makes all of its variants and one ``ccd_frame_distortion`` call compares them, and the
decoded frame, with the source: only one frame's variants live on the device at a time.
"""
from dataclasses import dataclass
from typing import Dict, List, Optional, Tuple

import torch

from .. import _native
from .._desc import CcdCoolChicDesc, desc_from_header
from . import decode, quality, rate


@dataclass
class GridRow:
    """One latent grid of a Cool-chic (grid 0 = finest).  PSNRs in dB, planes y / u / v (r / g / b for rgb)."""
    grid: int
    size: Tuple[int, int]
    is_hyper: bool
    bits: float                                       # model bits of the grid's latents
    bpp: float                                        # bits per pixel of the frame
    drop_psnr_db: Optional[float] = None              # the frame with this grid alone read as zeros
    drop_psnr_planes_db: Optional[List[float]] = None
    drop_delta_db: Optional[float] = None             # drop_psnr_db - the decoded frame's PSNR
    coarse_psnr_db: Optional[float] = None            # residue only: the synthesis grids from the coarsest to this one kept


@dataclass
class FrameGrids:
    display_idx: int
    frame_type: str
    img_size: Tuple[int, int]
    bitdepth: int
    psnr_db: float                                    # the decoded frame
    psnr_planes_db: List[float]
    coolchics: Dict[str, List[GridRow]]               # "residue" (+ "motion" for P / B): one row per grid


def synthesis_masks(desc: CcdCoolChicDesc):
    """(synthesis grids finest first, drop masks, coarse masks) of a Cool-chic as ``zero_grids`` bit masks: drop[k]
    zeroes the k-th synthesis grid alone; coarse[n - 1] zeroes all but the n coarsest, n = 1 .. nl - 1.  Hyperlatent
    grids are never masked."""
    syn = [g for g in range(desc.n_grids) if not desc.grid_is_hyper[g]]
    drop = [1 << g for g in syn]
    coarse = [sum(1 << g for g in syn[:len(syn) - n]) for n in range(1, len(syn))]
    return syn, drop, coarse


def _psnr(sse: List[int], n_samples: List[int], bitdepth: int):
    """(frame PSNR, per-plane PSNR) of a frame's per-plane SSE, formed by FrameQuality (training/loss.py:88-118)."""
    q = quality.FrameQuality(display_idx=0, frame_type="", img_size=(0, 0), bitdepth=bitdepth, frame_data_type="",
                             n_bytes=0, sse=sse, n_samples=n_samples, max_abs=[0, 0, 0])
    return q.psnr_db, [q.psnr_y_db, q.psnr_u_db, q.psnr_v_db]


@torch.no_grad()
def video_grid_analysis(bitstream_bytes: bytes, original_path: str, frame_offset: int = 0, max_decoding_order: int = -1,
                        device: int = 0) -> Dict[str, FrameGrids]:
    """Grid analysis of every frame of an image / video bitstream against its source file (.yuv / .png / .ppm):
    ``{str(display_idx): FrameGrids}`` in display order.  The source is checked as by video_quality."""
    frames = quality._frame_layout(memoryview(bytes(bitstream_bytes)), max_decoding_order)
    by_display = quality._read_sources(frames, original_path, frame_offset)
    ctx = _native.get_context(device)
    sources = quality._upload_sources(ctx, by_display)

    cc = {}  # every Cool-chic in decode order: headers, descs, NN integers, latents, frame-tail requests

    def decode_keeping_latents(headers, bytes_nn, bytes_latent, device, finish):
        descs = [desc_from_header(h) for h in headers]
        nn_bytes = [bytes(b) for b in bytes_nn]
        outs, lats = ctx.decode_many(descs, nn_bytes, [bytes(b) for b in bytes_latent], want_latents=True, finish=finish)
        cc.update(headers=list(headers), descs=descs, nns=[_native.decode_nn(d, b) for d, b in zip(descs, nn_bytes)],
                  lats=lats, finish=list(finish))
        return outs

    seen = []  # coding order: (frame header, {name: (decode-order index, decoded output)}, references)

    def reconstruct(frame_header, cc_out, reference_frames, dev):
        first = sum(len(s[1]) for s in seen)
        seen.append((frame_header, {name: (first + k, o) for k, (name, o) in enumerate(cc_out.items())},
                     reference_frames))
        return decode._reconstruct(frame_header, cc_out, reference_frames, dev)

    decoded = decode.decode_video_bytes(bitstream_bytes, max_decoding_order=max_decoding_order, device=device,
                                        output_device="cuda", decode_fn=decode_keeping_latents, reconstruct_fn=reconstruct)
    rates = rate._rates_of_latents(ctx, cc["headers"], cc["descs"], cc["nns"], cc["lats"])

    display_of = {coding_idx: disp for disp, (coding_idx, _, _, _) in by_display.items()}
    out = {}
    for coding_idx in range(len(seen)):
        fh, ccs, refs = seen[coding_idx]
        seen[coding_idx] = (None, {}, None)  # this frame's decoded outputs are not needed past its own variants
        disp = display_of[coding_idx]
        s = by_display[disp][3]
        h, w = s.img_size
        cs = 1 if s.frame_data_type == "yuv420" else 0
        n_samples = [h * w] + [(h >> cs) * (w >> cs)] * 2
        variants = []  # (name, "drop" | "coarse", grid of the row, zero_grids)
        for name, (k, _) in ccs.items():
            syn, drop, coarse = synthesis_masks(cc["descs"][k])
            variants += [(name, "drop", g, m) for g, m in zip(syn, drop)]
            if name == "residue":
                variants += [(name, "coarse", syn[len(syn) - n], m) for n, m in enumerate(coarse, 1)]
        idx = [ccs[name][0] for name, _, _, _ in variants]
        outs = ctx.synthesize([cc["descs"][i] for i in idx], [cc["nns"][i] for i in idx], [cc["lats"][i] for i in idx],
                              [m for _, _, _, m in variants], finish=[cc["finish"][i] for i in idx])
        base = {name: o for name, (_, o) in ccs.items()}
        fds = [decode._reconstruct(fh, {**base, v[0]: o}, refs, device) for v, o in zip(variants, outs)]
        del outs
        dist = ctx.frame_distortion([decoded[str(disp)]] + fds, [sources[disp]] * (1 + len(fds)),
                                    [s.layout] * (1 + len(fds)))
        del fds
        psnr, psnr_planes = _psnr(dist[0]["sse"], n_samples, s.bitdepth)
        got = {v[:3]: _psnr(r["sse"], n_samples, s.bitdepth) for v, r in zip(variants, dist[1:])}
        tables = {}
        for name, (k, _) in ccs.items():
            r = rates[k]
            rows = []
            for g in range(len(r.grid_sizes)):
                row = GridRow(grid=g, size=tuple(r.grid_sizes[g]), is_hyper=r.grid_is_hyper[g], bits=r.grid_bits[g],
                              bpp=r.grid_bpp[g])
                if (name, "drop", g) in got:
                    row.drop_psnr_db, row.drop_psnr_planes_db = got[(name, "drop", g)]
                    row.drop_delta_db = row.drop_psnr_db - psnr
                if (name, "coarse", g) in got:
                    row.coarse_psnr_db = got[(name, "coarse", g)][0]
                rows.append(row)
            tables[name] = rows
        out[str(disp)] = FrameGrids(display_idx=disp, frame_type=fh.get_value("frame_type"), img_size=(h, w),
                                    bitdepth=s.bitdepth, psnr_db=psnr, psnr_planes_db=psnr_planes, coolchics=tables)
    return dict(sorted(out.items(), key=lambda kv: int(kv[0])))
