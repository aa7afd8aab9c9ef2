"""Rate analysis of Cool-chic bitstreams: where the bits of a ``.cool`` file go.

For every latent symbol ``s`` (hyperlatent grids included) the ARM + IFCE are evaluated exactly as decoding does,
on the decoded neighbours, and ``bits = 24 - log2(freq)`` with ``freq = left(s+1) - left(s)`` the integer
frequency of ``s`` in the quantised-Laplace model the range coder used (constriction's leaky cumulative on the
2^24 scale).  This is the information content under the model the coder used, NOT the reference encoder's
training proxy (``detailed_rate_bit`` of component/core/coolchic.py): the two differ by the proxy's relaxation.
Their sum over a Cool-chic is at most the latent payload; the gap is the range coder's seal and word padding.

The per-symbol pass is one libccdec kernel (``ccd_latent_rate``) for every grid of every Cool-chic of a call.
Network bits are the exp-Golomb codeword lengths of the decoded NN integers (neuralnet.py:26-89), computed on
the host; their sum plus ``nn_n_bit_pad`` is exactly ``8 * nn_n_bytes``.
"""
import os
import re
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .. import _native
from .._desc import CcdCoolChicDesc, desc_from_header
from .expgolomb import exp_golomb_bits
from .header import NN_KINDS, NN_MODULES, CoolChicHeader, FrameHeader, VideoHeader

_SCALE_INC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "csrc", "ccd_scale_table.inc")
_scale_table: Optional[np.ndarray] = None


def scale_table() -> np.ndarray:
    """The 2561 normative Laplace scales (float32) the range coder indexes with sc_idx."""
    global _scale_table
    if _scale_table is None:
        words = re.findall(r"0x([0-9a-fA-F]{8})u", open(_SCALE_INC).read())
        _scale_table = np.array([int(w, 16) for w in words], dtype=np.uint32).view(np.float32)
        assert _scale_table.size == 2561
    return _scale_table


def nn_section_counts(d: CcdCoolChicDesc) -> Dict[str, Dict[str, int]]:
    """Number of transmitted integers per module and kind, in bitstream order (neuralnet.py:120-148)."""
    from ..synth import nn_sections

    sec = nn_sections(d)
    return {m: {k: int(sum(int(np.prod(s)) for _, s in sec[f"{m}.{k}"])) for k in NN_KINDS} for m in NN_MODULES}


def nn_bits(d: CcdCoolChicDesc, nn_ints: np.ndarray) -> Dict[str, Dict[str, int]]:
    """Total exp-Golomb codeword length per module and kind (get_network_rate, core/coolchic.py:911-939, counted
    on the transmitted codewords)."""
    counts = nn_section_counts(d)
    out: Dict[str, Dict[str, int]] = {}
    p, j = 0, 0
    for m in NN_MODULES:
        out[m] = {}
        for k in NN_KINDS:
            n = counts[m][k]
            out[m][k] = int(sum(exp_golomb_bits(nn_ints[p:p + n], [int(d.expgol[j])] * n)))
            p += n
            j += 1
    if p != len(nn_ints):
        raise ValueError(f"{len(nn_ints)} NN integers, the architecture transmits {p}")
    return out


@dataclass
class CoolChicRate:
    """Rate of one Cool-chic.  Grid lists are finest first (size_per_latent order); maps are float32 CUDA tensors."""
    img_size: Tuple[int, int]
    grid_sizes: List[Tuple[int, int]]
    grid_is_hyper: List[bool]
    rate_bit: List[torch.Tensor]        # [1, 1, h_i, w_i] bits of each symbol
    mu: List[torch.Tensor]              # [1, 1, h_i, w_i] the mean the coder used, (mu_idx - 16384) / 256
    scale: List[torch.Tensor]           # [1, 1, h_i, w_i] the Laplace scale the coder used
    grid_bits: List[float]              # f64 sum per grid
    spatial_rate_bit: torch.Tensor      # [1, 1, H, W] (training/test.py:217-235, canonical fp32 order)
    nn_bits: Dict[str, Dict[str, int]]  # module -> weight / bias -> codeword bits
    nn_pad_bits: int
    header_bits: int
    nn_payload_bits: int
    latent_payload_bits: int

    @property
    def n_pixels(self) -> int:
        return self.img_size[0] * self.img_size[1]

    @property
    def grid_bpp(self) -> List[float]:
        return [b / self.n_pixels for b in self.grid_bits]

    @property
    def latent_model_bits(self) -> float:
        """Information content of all latents under the coder's model (<= latent_payload_bits)."""
        return float(sum(self.grid_bits))

    @property
    def nn_module_bits(self) -> Dict[str, int]:
        return {m: sum(v.values()) for m, v in self.nn_bits.items()}

    @property
    def total_bits(self) -> int:
        """Header + NN payload + latent payload: 8 x the Cool-chic's bytes."""
        return self.header_bits + self.nn_payload_bits + self.latent_payload_bits


@dataclass
class FrameRate:
    display_idx: int
    coding_idx: int
    frame_type: str
    img_size: Tuple[int, int]
    header_bits: int                                 # the frame header
    n_bytes: int                                     # frame header + its Cool-chics
    coolchics: Dict[str, CoolChicRate] = field(default_factory=dict)  # "residue" (+ "motion" for P / B)

    @property
    def total_bits(self) -> int:
        return self.header_bits + sum(c.total_bits for c in self.coolchics.values())


def _split_coolchic(buf):
    """(header, header_bytes, nn, latent, rest) at the start of ``buf`` (decode.py:134-143)."""
    h = CoolChicHeader()
    rest = h.read_header(buf)
    n_nn, n_lat = h.get_value("nn_n_bytes"), h.get_value("n_bytes_latent")
    if len(rest) < n_nn + n_lat:
        raise ValueError(f"Bitstream truncated: need {n_nn + n_lat} payload bytes, have {len(rest)}.")
    return h, bytes(rest[:n_nn]), bytes(rest[n_nn:n_nn + n_lat]), rest[n_nn + n_lat:]


def _rates(headers: List[CoolChicHeader], nn_bytes: List[bytes], lat_bytes: List[bytes], device: int
           ) -> List[CoolChicRate]:
    """One decode_many for the latents of every Cool-chic, then one ccd_latent_rate call."""
    ctx = _native.get_context(device)
    descs = [desc_from_header(h) for h in headers]
    for h, nb, lb in zip(headers, nn_bytes, lat_bytes):
        if len(nb) < h.get_value("nn_n_bytes") or len(lb) < h.get_value("n_bytes_latent"):
            raise ValueError("Cool-chic payload shorter than its header announces")
    nn_bytes = [bytes(nb[:h.get_value("nn_n_bytes")]) for h, nb in zip(headers, nn_bytes)]
    lat_bytes = [bytes(lb[:h.get_value("n_bytes_latent")]) for h, lb in zip(headers, lat_bytes)]
    _, lats = ctx.decode_many(descs, nn_bytes, lat_bytes, want_latents=True)
    nns = [_native.decode_nn(d, nb) for d, nb in zip(descs, nn_bytes)]
    return _rates_of_latents(ctx, headers, descs, nns, lats)


def _rates_of_latents(ctx, headers: List[CoolChicHeader], descs: List[CcdCoolChicDesc], nns: List[np.ndarray],
                      lats: List[torch.Tensor]) -> List[CoolChicRate]:
    """The rates of Cool-chics whose latents are already decoded: one ccd_latent_rate call."""
    res = ctx.latent_rate(descs, nns, lats, want_mu_sc=True, want_spatial=True)
    table = torch.from_numpy(scale_table()).to(ctx.torch_device)
    out = []
    for h, d, nn, r in zip(headers, descs, nns, res):
        sizes = d.grid_sizes()
        _, offs = _native.latent_layout(d)
        mu_sc = r["mu_sc"]
        mu_idx = (mu_sc & 0xFFFF).to(torch.float32)
        mu_all = (mu_idx - 16384.0) / 256.0
        sc_all = table[(mu_sc >> 16).long()]
        view = lambda t, g: t[offs[g]:offs[g] + sizes[g][0] * sizes[g][1]].view(1, 1, *sizes[g])  # noqa: E731
        out.append(CoolChicRate(
            img_size=(int(d.img_h), int(d.img_w)),
            grid_sizes=sizes,
            grid_is_hyper=[bool(d.grid_is_hyper[g]) for g in range(d.n_grids)],
            rate_bit=[view(r["bits"], g) for g in range(d.n_grids)],
            mu=[view(mu_all, g) for g in range(d.n_grids)],
            scale=[view(sc_all, g) for g in range(d.n_grids)],
            grid_bits=r["grid_bits"],
            spatial_rate_bit=r["spatial"],
            nn_bits=nn_bits(d, nn),
            nn_pad_bits=int(h.get_value("nn_n_bit_pad")),
            header_bits=8 * int(h.get_value("n_bytes_header")),
            nn_payload_bits=8 * int(h.get_value("nn_n_bytes")),
            latent_payload_bits=8 * int(h.get_value("n_bytes_latent")),
        ))
    return out


@torch.no_grad()
def coolchic_rate(header: CoolChicHeader, bytes_nn: bytes, bytes_latent: bytes, device: int = 0) -> CoolChicRate:
    """Rate of one Cool-chic given its parsed header and payloads (the arguments of encode_decode_coolchic)."""
    return _rates([header], [bytes_nn], [bytes_latent], device)[0]


@torch.no_grad()
def video_rate(bitstream_bytes: bytes, max_decoding_order: int = -1, device: int = 0) -> Dict[str, FrameRate]:
    """Rate of every frame of an image / video bitstream: ``{str(display_idx): FrameRate}``.  All Cool-chics
    (residue, and motion for P / B frames) go through one decode and one rate call."""
    buf = memoryview(bytes(bitstream_bytes))
    video_header = VideoHeader()
    buf = video_header.read_header(buf)
    cs = video_header.get_coding_structure()
    if max_decoding_order == -1:
        max_decoding_order = cs.get_max_coding_order()
    frames, flat = [], []
    for coding_idx in range(max_decoding_order + 1):
        n_frame = len(buf)
        fh = FrameHeader()
        buf = fh.read_header(buf)
        names = ["residue"] + (["motion"] if fh.get_value("frame_type") in ["P", "B"] else [])
        ccs = {}
        for name in names:
            h, nb, lb, buf = _split_coolchic(buf)
            ccs[name] = len(flat)
            flat.append((h, nb, lb))
        frames.append((coding_idx, fh, ccs, n_frame - len(buf)))
    rates = _rates([f[0] for f in flat], [f[1] for f in flat], [f[2] for f in flat], device) if flat else []
    out = {}
    for coding_idx, fh, ccs, n_bytes in frames:
        display_idx = cs.get_frame_from_coding_order(coding_idx).display_order
        ccr = {name: rates[i] for name, i in ccs.items()}
        out[str(display_idx)] = FrameRate(
            display_idx=display_idx, coding_idx=coding_idx, frame_type=fh.get_value("frame_type"),
            img_size=ccr["residue"].img_size, header_bits=8 * int(fh.get_value("n_bytes_header")), n_bytes=n_bytes,
            coolchics=ccr)
    return dict(sorted(out.items(), key=lambda kv: int(kv[0])))
