"""Lossless bitstream optimisation: retune the ARM and IFCE integers of every Cool-chic for the exact coded rate and
rewrite the bitstream.  Every decoded sample is unchanged.

The ARM and the IFCE only shape the entropy model; neither feeds the synthesis.  So a Cool-chic whose ARM / IFCE
integers change, with the same latents range-coded again under the new model, decodes to the same latents and the same
frames.  The cost minimised is what the file pays for the entropy model: the exact latent model bits
(``ccd_latent_rate``: the int64 ARM, the clamped (mu, scale) indices and the range coder's integer frequencies) plus the
exp-Golomb bits of the ARM and IFCE integers.

Per Cool-chic (residue and motion alike), greedy coordinate descent:
  * each round prices every ARM and IFCE integer at +1 and -1, and at twice its last accepted step for an integer that
    improved, in batched ``ccd_rate_candidates`` calls (DESIGN §4.11);
  * the improving candidates (one per integer, the best) are applied together in order of gain, ties to the lower
    integer index; the batch is verified with one exact rate pass and halved until the verified total goes down;
  * a candidate is kept only if |q| <= 65535 and, when the model took the fast entropy kernel, the edited one still does.
Then the exp-Golomb order of each module is chosen again for the final integers (0 .. 12, the header's table), the
upsampling biases -- which the upsampling never reads -- are set to 0, the NN and the latents are encoded again and the
Cool-chic header rewritten.  A Cool-chic whose rewritten bytes are not fewer than the original's keeps its bytes, and
so does one whose NN payload would not fit the header's 14-bit byte count.  Video and frame headers are unchanged.
"""
import time
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Tuple

import numpy as np
import torch

from .. import _native
from .._desc import desc_from_header
from .expgolomb import encode_exp_golomb, exp_golomb_bits
from .header import EXP_GOL_TABLE, NN_KINDS, NN_MODULES, CoolChicHeader, FrameHeader, VideoHeader
from .rate import _split_coolchic, nn_section_counts

Q_MAX = 65535             # largest |q| the reference's quantiser produces (nnquant/quantizemodel.py)
NN_BYTES_MAX = (1 << 14) - 1  # nn_n_bytes is a 14-bit header field


@dataclass
class CoolChicReport:
    name: str                     # "residue" or "motion"
    bytes_before: int             # header + NN + latents
    bytes_after: int
    nn_bytes_before: int
    nn_bytes_after: int
    latent_bytes_before: int
    latent_bytes_after: int
    latent_bits_before: float     # exact latent model bits: the per-grid sums added finest first
    latent_bits_after: float
    arm_bits_saved: float = 0.0   # search gain (latent + NN bits) of the ARM edits
    ifce_bits_saved: float = 0.0  # ... and of the IFCE edits (a verified batch's gain is split by priced gains)
    recount_bits_saved: int = 0   # exp-Golomb orders chosen again
    bias_reset_bits_saved: int = 0  # upsampling biases set to 0
    rounds: int = 0
    candidates: int = 0
    seconds: float = 0.0
    kept_original: bool = False


@dataclass
class FrameReport:
    coding_idx: int
    frame_type: str
    coolchics: List[CoolChicReport] = field(default_factory=list)


@dataclass
class OptimizeReport:
    frames: List[FrameReport]
    bytes_before: int
    bytes_after: int
    seconds: float

    @property
    def coolchics(self) -> List[CoolChicReport]:
        return [c for f in self.frames for c in f.coolchics]


def _sections(d) -> Dict[Tuple[str, str], Tuple[int, int]]:
    """(module, kind) -> [start, end) in the NN integer order."""
    counts = nn_section_counts(d)
    out, p = {}, 0
    for m in NN_MODULES:
        for k in NN_KINDS:
            out[(m, k)] = (p, p + counts[m][k])
            p += counts[m][k]
    return out


def _eg_bits(values, k: int) -> int:
    return int(sum(exp_golomb_bits(values, [k] * len(values))))


def best_expgol_count(values) -> int:
    """The exp-Golomb order in the header's table that codes ``values`` in the fewest bits (the lowest on a tie)."""
    values = [int(v) for v in values]
    return min(EXP_GOL_TABLE, key=lambda k: (_eg_bits(values, k), k))


def _search(ctx, d, nn: np.ndarray, lat: torch.Tensor, sec, max_rounds: int, deadline: Optional[float], rep):
    """Greedy coordinate descent on the ARM and IFCE integers; returns the final integers and their latent bits."""
    eg = [int(d.expgol[j]) for j in range(8)]
    n_arm = sec[("arm", "bias")][1]
    n_model = sec[("ifce", "bias")][1]
    order = np.zeros(n_model, dtype=np.int64)  # exp-Golomb order of each ARM / IFCE integer
    for j, key in enumerate([("arm", "weight"), ("arm", "bias"), ("ifce", "weight"), ("ifce", "bias")]):
        order[sec[key][0]:sec[key][1]] = eg[j]

    def nn_cost(i, v):
        return exp_golomb_bits([int(v)], [int(order[i])])[0]

    def exact(q):  # latent bits (grid sums added finest first) and kernel choice: row 0 is ccd_latent_rate's grid_bits
        bits, fast = ctx.rate_candidates(d, q, lat, [(0, 1)])
        return float(sum(bits[0].tolist())), bool(fast[0])

    cur = nn.copy()
    cur_bits, base_fast = exact(cur)
    rep.latent_bits_before = cur_bits
    step = {}  # integer -> its last accepted delta
    for _ in range(max_rounds):
        if deadline is not None and time.monotonic() > deadline:
            break
        rep.rounds += 1
        cands = []
        for i in range(n_model):
            ds = {1, -1}
            if i in step:
                ds.add(2 * step[i])
            cands += [(i, dl) for dl in sorted(ds) if abs(int(cur[i]) + dl) <= Q_MAX]
        best: Dict[int, Tuple[float, int]] = {}
        for c0 in range(0, len(cands), _native.CCD_CAND_MAX):
            chunk = cands[c0:c0 + _native.CCD_CAND_MAX]
            bits, fast = ctx.rate_candidates(d, cur, lat, chunk)
            tot = bits.sum(axis=1)
            rep.candidates += len(chunk)
            for j, (i, dl) in enumerate(chunk):
                if base_fast and not fast[j + 1]:
                    continue
                gain = (tot[0] - tot[j + 1]) + (nn_cost(i, cur[i]) - nn_cost(i, cur[i] + dl))
                if gain > 0 and (i not in best or gain > best[i][0]):
                    best[i] = (gain, dl)
        ranked = sorted(best.items(), key=lambda kv: (-kv[1][0], kv[0]))
        accepted = False
        while ranked:
            trial = cur.copy()
            for i, (_, dl) in ranked:
                trial[i] += dl
            t_bits, t_fast = exact(trial)
            gain = (cur_bits - t_bits) + sum(nn_cost(i, cur[i]) - nn_cost(i, trial[i]) for i, _ in ranked)
            if gain > 0 and (t_fast or not base_fast):
                priced = sum(g for _, (g, _) in ranked)
                arm = sum(g for i, (g, _) in ranked if i < n_arm)
                rep.arm_bits_saved += gain * arm / priced
                rep.ifce_bits_saved += gain * (priced - arm) / priced
                for i, (_, dl) in ranked:
                    step[i] = dl
                for i in list(step):
                    if i not in best:
                        del step[i]
                cur, cur_bits, accepted = trial, t_bits, True
                break
            ranked = ranked[:len(ranked) // 2]
        if not accepted:
            break
    return cur, cur_bits


@torch.no_grad()
def _optimize_coolchic(ctx, name: str, header: CoolChicHeader, raw: bytes, nn_bytes: bytes, lat_bytes: bytes,
                       lat: torch.Tensor, max_rounds: int, deadline: Optional[float]) -> Tuple[bytes, CoolChicReport]:
    t0 = time.monotonic()
    d = desc_from_header(header)
    nn = _native.decode_nn(d, nn_bytes)
    sec = _sections(d)
    rep = CoolChicReport(name=name, bytes_before=len(raw), bytes_after=len(raw), nn_bytes_before=len(nn_bytes),
                         nn_bytes_after=len(nn_bytes), latent_bytes_before=len(lat_bytes),
                         latent_bytes_after=len(lat_bytes), latent_bits_before=0.0, latent_bits_after=0.0)
    q, q_bits = _search(ctx, d, nn, lat, sec, max_rounds, deadline, rep)
    rep.latent_bits_after = q_bits
    # upsampling biases: transmitted, never read
    a, b = sec[("upsampling", "bias")]
    eg_ups_b = int(d.expgol[NN_MODULES.index("upsampling") * 2 + 1])
    rep.bias_reset_bits_saved = _eg_bits(q[a:b], eg_ups_b) - _eg_bits([0] * (b - a), eg_ups_b)
    q[a:b] = 0
    counts = []
    eg_desc = header.get_value("nn_expgol_cnt")
    new_header = CoolChicHeader()
    new_header.read_header(raw)
    new_eg = new_header.get_value("nn_expgol_cnt")
    for j, (m, k) in enumerate((m, k) for m in NN_MODULES for k in NN_KINDS):
        s, e = sec[(m, k)]
        old_k = int(eg_desc.get_value(m, k))
        new_k = best_expgol_count(q[s:e])
        rep.recount_bits_saved += _eg_bits(q[s:e], old_k) - _eg_bits(q[s:e], new_k)
        new_eg.set_value(new_k, m, k)
        counts += [new_k] * (e - s)
    payload, pad = encode_exp_golomb([int(v) for v in q], counts)
    _, lat_payload, _ = ctx.encode_latents(d, q, lat)
    if len(payload) > NN_BYTES_MAX:
        rep.kept_original, rep.latent_bits_after = True, rep.latent_bits_before
        rep.seconds = time.monotonic() - t0
        return raw, rep
    new_header.set_value("nn_n_bytes", len(payload))
    new_header.set_value("nn_n_bit_pad", pad)
    new_header.set_value("n_bytes_latent", len(lat_payload))
    out = new_header.to_bytes() + payload + lat_payload
    if len(out) < len(raw):
        rep.bytes_after, rep.nn_bytes_after, rep.latent_bytes_after = len(out), len(payload), len(lat_payload)
    else:
        out = raw
        rep.kept_original, rep.latent_bits_after = True, rep.latent_bits_before
    rep.seconds = time.monotonic() - t0
    return out, rep


@torch.no_grad()
def optimize_bitstream(bitstream_bytes: bytes, device: int = 0, max_rounds: int = 8,
                       time_budget_s: Optional[float] = None) -> Tuple[bytes, OptimizeReport]:
    """Losslessly smaller bitstream (image or video, every P / B GOP) and the report of what each Cool-chic saved.
    ``max_rounds``: rounds of the search per Cool-chic; ``time_budget_s``: no new round starts after that many seconds
    (counted over the whole bitstream)."""
    t0 = time.monotonic()
    deadline = None if time_budget_s is None else t0 + float(time_budget_s)
    data = bytes(bitstream_bytes)
    buf = memoryview(data)
    vh = VideoHeader()
    rest = vh.read_header(buf)
    parts = [bytes(buf[:len(buf) - len(rest)])]
    frames, flat = [], []  # flat: (frame, name, header, raw bytes, nn bytes, latent bytes)
    for coding_idx in range(vh.get_coding_structure().get_max_coding_order() + 1):
        fh = FrameHeader()
        after = fh.read_header(rest)
        frames.append((coding_idx, fh, bytes(rest[:len(rest) - len(after)])))
        rest = after
        for name in ["residue"] + (["motion"] if fh.get_value("frame_type") in ("P", "B") else []):
            h, nb, lb, after = _split_coolchic(rest)
            flat.append((coding_idx, name, h, bytes(rest[:len(rest) - len(after)]), nb, lb))
            rest = after
    ctx = _native.get_context(device)
    descs = [desc_from_header(f[2]) for f in flat]
    _, lats = ctx.decode_many(descs, [f[4] for f in flat], [f[5] for f in flat], want_latents=True)
    reports = [FrameReport(coding_idx=c, frame_type=fh.get_value("frame_type")) for c, fh, _ in frames]
    new_cc = []
    for (coding_idx, name, h, raw, nb, lb), lat in zip(flat, lats):
        out, rep = _optimize_coolchic(ctx, name, h, raw, nb, lb, lat, max_rounds, deadline)
        new_cc.append((coding_idx, out))
        reports[coding_idx].coolchics.append(rep)
    for coding_idx, _, fh_bytes in frames:
        parts.append(fh_bytes)
        parts += [out for c, out in new_cc if c == coding_idx]
    parts.append(bytes(rest))
    result = b"".join(parts)
    return result, OptimizeReport(frames=reports, bytes_before=len(data), bytes_after=len(result),
                                  seconds=time.monotonic() - t0)
