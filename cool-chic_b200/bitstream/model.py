"""Entropy-model analysis of Cool-chic bitstreams: what the ARM's spatial context, the IFCE, the hyperlatents and the
scale calibration are worth, in exact bits under the coder's model (DESIGN §4.10).

Every variant is the coder's model with some ARM inputs read as 0 (the model's own convention for a neighbour outside
the grid and for a grid without IFCE input), evaluated on the decoded latents by ``ccd_latent_rate_edited``:

  decoded      no change (equals ``video_rate``'s bits, bit for bit)
  ctx_k        spatial inputs k .. n_ctx - 1 read as 0 (inputs in neighbour priority order), IFCE kept; k < n_ctx
  no_ifce      every IFCE feature read as 0                                      (flag_ifce)
  no_hyper     every hyperlatent grid read as 0 where it is an IFCE input        (flag_ifce, hyperlatent grids)
  no_context   every ARM input read as 0: one static Laplace for all symbols

The calibration sweep (``ccd_rate_sweep``) re-prices every symbol with the coder's (mu_idx, sc_idx) and sc_idx shifted
by each offset (the scale times exp(offset / 256)), and counts each grid's symbols: the static baseline is the
zeroth-order entropy of those counts, what an ideal static code per grid would spend (its table not counted).
"""
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .._desc import CcdCoolChicDesc
from . import rate

# sc_idx offsets of the calibration sweep: the scale times 0.78 ... 1.28 in steps of exp(1/32)
SIGMA_OFFSETS = tuple(range(-64, 65, 8))


def variant_edits(d: CcdCoolChicDesc) -> Dict[str, Tuple[int, int, int]]:
    """The variants a Cool-chic has, in report order: name -> (zero_ctx, zero_ifce_out, zero_ifce_grids)."""
    all_ctx = (1 << d.n_ctx) - 1
    cf = d.n_ifce_out if d.flag_ifce else 0
    out = {"decoded": (0, 0, 0)}
    for k in range(d.n_ctx):
        out[f"ctx_{k}"] = (all_ctx & ~((1 << k) - 1), 0, 0)
    hyper = sum(1 << g for g in range(d.n_grids) if d.grid_is_hyper[g])
    if d.flag_ifce:
        out["no_ifce"] = (0, (1 << cf) - 1, 0)
        if hyper:
            out["no_hyper"] = (0, 0, hyper)
    out["no_context"] = (all_ctx, (1 << cf) - 1, 0)
    return out


def static_bits(hist: np.ndarray) -> float:
    """Zeroth-order entropy of a symbol histogram, in bits: sum over symbols of -n_s log2(n_s / N)."""
    n = np.asarray(hist, dtype=np.float64)
    n = n[n > 0]
    return float(-(n * np.log2(n / n.sum())).sum()) if n.size else 0.0


@dataclass
class CoolChicModel:
    """Entropy-model analysis of one Cool-chic.  Grid lists are finest first (size_per_latent order)."""
    grid_sizes: List[Tuple[int, int]]
    grid_is_hyper: List[bool]
    n_ctx: int
    variants: Dict[str, List[float]]  # variant -> f64 bits per grid
    nn_bits: Dict[str, int]           # NN module -> codeword bits (weights + biases)
    sigma_offsets: List[int]
    sweep_bits: List[List[float]]     # per grid, the bits at each sigma offset
    hist: np.ndarray                  # int64 [n_grids, 128]: count of symbol s - 64 in bin s

    def total(self, variant: str) -> float:
        return float(sum(self.variants[variant]))

    def delta(self, variant: str) -> List[float]:
        """Bits the variant adds over ``decoded``, per grid."""
        return [v - d for v, d in zip(self.variants[variant], self.variants["decoded"])]

    @property
    def static_bits(self) -> List[float]:
        return [static_bits(h) for h in self.hist]

    @property
    def ctx_curve(self) -> List[float]:
        """Total latent bits with the first k spatial inputs, k = 0 .. n_ctx (k = n_ctx: ``decoded``)."""
        return [self.total(f"ctx_{k}") for k in range(self.n_ctx)] + [self.total("decoded")]

    @property
    def ctx_saved(self) -> List[float]:
        """Bits neighbour k saves, given neighbours 0 .. k - 1."""
        c = self.ctx_curve
        return [c[k] - c[k + 1] for k in range(self.n_ctx)]

    @property
    def arm_net(self) -> float:
        """Bits the whole context (no_context - decoded) saves, minus the ARM's NN bits."""
        return self.total("no_context") - self.total("decoded") - self.nn_bits["arm"]

    @property
    def ifce_net(self) -> Optional[float]:
        """Bits no_ifce adds, minus the IFCE's NN bits (None without IFCE)."""
        if "no_ifce" not in self.variants:
            return None
        return self.total("no_ifce") - self.total("decoded") - self.nn_bits["ifce"]

    @property
    def hyper_net(self) -> Optional[float]:
        """Bits no_hyper adds over the synthesis grids, minus the hyperlatent grids' own bits (None when the variant
        does not exist).  Positive: the hyperlatents pay for themselves."""
        if "no_hyper" not in self.variants:
            return None
        syn = [g for g, h in enumerate(self.grid_is_hyper) if not h]
        hyp = [g for g, h in enumerate(self.grid_is_hyper) if h]
        added = sum(self.delta("no_hyper")[g] for g in syn)
        return added - sum(self.variants["decoded"][g] for g in hyp)

    def _best(self, bits: Sequence[float]) -> Tuple[int, float]:
        # the smallest bits; among equal ones, the smallest shift
        k = min(range(len(bits)), key=lambda j: (bits[j], abs(self.sigma_offsets[j])))
        return self.sigma_offsets[k], float(bits[k])

    @property
    def best_offset(self) -> List[Tuple[int, float]]:
        """Per grid: (the sigma offset with the fewest bits, those bits)."""
        return [self._best(b) for b in self.sweep_bits]

    @property
    def best_offset_all(self) -> Tuple[int, float]:
        """(the one sigma offset for all grids with the fewest total bits, that total)."""
        return self._best([sum(b[k] for b in self.sweep_bits) for k in range(len(self.sigma_offsets))])


@dataclass
class FrameModel:
    display_idx: int
    coding_idx: int
    frame_type: str
    img_size: Tuple[int, int]
    coolchics: Dict[str, CoolChicModel] = field(default_factory=dict)  # "residue" (+ "motion" for P / B)


@torch.no_grad()
def video_model_analysis(bitstream_bytes: bytes, max_decoding_order: int = -1, device: int = 0,
                         sigma_offsets: Sequence[int] = SIGMA_OFFSETS) -> Dict[str, FrameModel]:
    """Entropy-model analysis of every frame of an image / video bitstream: ``{str(display_idx): FrameModel}``.  One
    decode of all Cool-chics, then per frame one rate call with every variant of its Cool-chics (device memory is held
    for one frame's variants at a time) and one sweep call."""
    offsets = [int(o) for o in sigma_offsets]
    cs, frames, flat = rate._split_frames(bitstream_bytes, max_decoding_order)
    if not flat:
        return {}
    ctx, descs, nns, lats = rate._decode_latents([f[0] for f in flat], [f[1] for f in flat], [f[2] for f in flat],
                                                 device)
    out = {}
    for coding_idx, fh, ccs, _ in frames:
        jobs = [(name, i, v, e) for name, i in ccs.items() for v, e in variant_edits(descs[i]).items()]
        res = ctx.latent_rate([descs[i] for _, i, _, _ in jobs], [nns[i] for _, i, _, _ in jobs],
                              [lats[i] for _, i, _, _ in jobs], want_mu_sc=[v == "decoded" for _, _, v, _ in jobs],
                              edits=[e for _, _, _, e in jobs])
        variants = {name: {} for name in ccs}
        mu_sc = {}
        for (name, _, v, _), r in zip(jobs, res):
            variants[name][v] = r["grid_bits"]
            if v == "decoded":
                mu_sc[name] = r["mu_sc"]
        del res
        sweep = ctx.rate_sweep([descs[i] for i in ccs.values()], [lats[i] for i in ccs.values()],
                               [mu_sc[name] for name in ccs], offsets)
        ccm = {}
        for (name, i), sw in zip(ccs.items(), sweep):
            d = descs[i]
            ccm[name] = CoolChicModel(
                grid_sizes=d.grid_sizes(), grid_is_hyper=[bool(d.grid_is_hyper[g]) for g in range(d.n_grids)],
                n_ctx=int(d.n_ctx), variants=variants[name],
                nn_bits={m: sum(v.values()) for m, v in rate.nn_bits(d, nns[i]).items()},
                sigma_offsets=list(offsets), sweep_bits=sw["bits"], hist=sw["hist"])
        display_idx = cs.get_frame_from_coding_order(coding_idx).display_order
        res_d = descs[ccs["residue"]]
        out[str(display_idx)] = FrameModel(display_idx=display_idx, coding_idx=coding_idx,
                                           frame_type=fh.get_value("frame_type"),
                                           img_size=(int(res_d.img_h), int(res_d.img_w)), coolchics=ccm)
    return dict(sorted(out.items(), key=lambda kv: int(kv[0])))
