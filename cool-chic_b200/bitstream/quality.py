"""Quality analysis of a bitstream against its source: what the bits of a ``.cool`` file buy.

For every decoded frame, the distortion against the source frame it was encoded from (``component/video.py:71``:
display frame ``i`` is source frame ``frame_offset + i``): per-plane sums of squared integer errors, exact, and the
MSE / PSNR of ``training/loss.py:88-118`` (pixel-weighted over the planes, ``dist_to_db`` with its 100 dB clamp,
``metrics/mse.py:18-21``).  For P / B frames also the statistics the reference encoder logs about the prediction
(``training/test.py:169-199``): mean alpha and beta, and the PSNR of the prediction and of the average of the
references, both ``-10 log10(mse + 1e-10)``.

Decoding goes through ``decode_video_bytes``; the prediction statistics are taken from each P / B frame's raw
residue and motion just before that frame is reconstructed (``ccd_inter_stats``), and one ``ccd_frame_distortion``
call then covers every frame.  The source frames are read and uploaded in one pinned host-to-device copy, as the
integers stored in the file.

On request, the motion analysis of every P / B frame (``bitstream/motion.py``, DESIGN §4.9): one
``ccd_inter_analysis`` launch next to ``ccd_inter_stats``, on the same inputs, so there is no second decode.

On request, MS-SSIM (Wang, Simoncelli and Bovik 2003; DESIGN §4.6) from the same integers: one ``ccd_frame_ssim`` call
for every frame whose planes all have both sides of at least 176 samples (five scales of at least 11), formed per plane
on the host from the per-scale means, and per frame the pixel-weighted mean over the planes.  Smaller frames get None.

On request, VIF (Sheikh and Bovik 2006, the multi-scale pixel-domain vifp_mscale; DESIGN §4.12) from the same
integers in 8-bit units: one ``ccd_frame_vif`` call for every frame whose planes all have both sides of at least 41
samples (a valid output at the fourth scale), per plane sum_s num_s / sum_s den_s, and per frame the pixel-weighted
mean over the planes.  Smaller frames, and frames with a flat source plane (no VIF), get None.

On request, PSNR-HVS-M and PSNR-HVS (Ponomarenko et al. 2007; DESIGN §4.13) from the same integers in 8-bit units:
one ``ccd_frame_hvs`` call for every frame whose planes all have both sides of at least 8 samples (one 8 x 8 block),
per plane the masked and unmasked sums of CSF-weighted squared DCT errors over its blocks, and per frame the
coefficient-weighted mean over the planes.  Smaller frames get None.
"""
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from .. import _native
from ..io.io import read_samples
from . import decode
from .header import VideoHeader


def dist_to_db(dist: float, max_db: float = 100) -> float:
    """metrics/mse.py:18-21."""
    min_dist = 10 ** (-max_db / 10)
    return -10 * math.log10(max(dist, min_dist))


def pred_to_db(sse: float, n: int) -> float:
    """training/test.py:188-199: -10 log10(mse + 1e-10), no clamp."""
    return -10 * math.log10(sse / n + 1e-10)


MS_SSIM_WEIGHTS = (0.0448, 0.2856, 0.3001, 0.2363, 0.1333)
MS_SSIM_MIN_SIDE = 176  # 11 samples at the fifth scale


def ms_ssim_from_scales(cs: List[float], ssim: List[float]) -> float:
    """MS-SSIM of one plane from its five per-scale means of cs and of l * cs: prod_{j<4} max(cs_j, 0)^w_j *
    max(ssim_4, 0)^w_4."""
    w = MS_SSIM_WEIGHTS
    v = 1.0
    for j in range(4):
        v *= max(cs[j], 0.0) ** w[j]
    return v * max(ssim[4], 0.0) ** w[4]


VIF_MIN_SIDE = 41  # scales 0..3: 41 -> 17 -> 7 -> 3 samples, and 3 taps at the last


def vif_from_scales(num: List[float], den: List[float]) -> Optional[float]:
    """VIF of one plane from its four per-scale sums: sum num / sum den; None for a flat source plane (sum den = 0)."""
    d = sum(den)
    return None if d == 0 else sum(num) / d


def vif_applies(img_size, frame_data_type: str) -> bool:
    """Whether every plane of an (h, w) frame has both sides >= 41 (4:2:0 chroma: (h / 2, w / 2))."""
    cs = 1 if frame_data_type == "yuv420" else 0
    return min(img_size) >> cs >= VIF_MIN_SIDE


HVS_MIN_SIDE = 8  # one 8 x 8 block


def hvs_from_sums(sums: List[float], n_coeffs: List[int]) -> float:
    """PSNR-HVS(-M) in dB of one or more planes from their sums of weighted squared DCT errors and their coefficient
    counts: dist_to_db(sum S / sum N / 255^2), the rule psnr_db applies to the pixel-weighted MSE."""
    return dist_to_db(sum(sums) / sum(n_coeffs) / 255.0**2)


def hvs_applies(img_size, frame_data_type: str) -> bool:
    """Whether every plane of an (h, w) frame has both sides >= 8 (4:2:0 chroma: (h / 2, w / 2))."""
    cs = 1 if frame_data_type == "yuv420" else 0
    return min(img_size) >> cs >= HVS_MIN_SIDE


def ms_ssim_applies(img_size, frame_data_type: str) -> bool:
    """Whether every plane of an (h, w) frame has both sides >= 176 (4:2:0 chroma: (h / 2, w / 2))."""
    cs = 1 if frame_data_type == "yuv420" else 0
    return min(img_size) >> cs >= MS_SSIM_MIN_SIDE


@dataclass
class FrameQuality:
    """Quality of one decoded frame.  Planes are y / u / v, or r / g / b for rgb frames."""
    display_idx: int
    frame_type: str
    img_size: tuple
    bitdepth: int
    frame_data_type: str
    n_bytes: int                  # frame header + its Cool-chics
    sse: List[int]                # per plane, in integer sample units
    n_samples: List[int]          # per plane
    max_abs: List[int]            # per plane, in integer sample units
    alpha_mean: float = 0.0
    beta_mean: float = 0.0
    pred_psnr_db: float = 0.0
    dummy_pred_psnr_db: float = 0.0
    error_map: Optional[torch.Tensor] = None   # [H, W] fp32(sum_c d_c^2) / fp32(M^2)
    alpha_map: Optional[torch.Tensor] = None   # [H, W] (P / B)
    beta_map: Optional[torch.Tensor] = None    # [H, W] (P / B)
    pred_map: Optional[torch.Tensor] = None    # [3, H, W] (P / B)
    ms_ssim_planes: Optional[List[float]] = None        # per plane; None: not asked for, or a plane below 176
    ssim_maps: Optional[List[torch.Tensor]] = None      # per plane, [h_c - 10, w_c - 10] scale-0 SSIM map
    vif_planes: Optional[List[Optional[float]]] = None  # per plane (None: flat source); None: not asked for, or below 41
    hvs_planes: Optional[List[tuple]] = None            # per plane (S_hvs_m, S_hvs, N_c); None: not asked for, or below 8
    hvs_maps: Optional[List[torch.Tensor]] = None       # per plane, [h_c >> 3, w_c >> 3]: S_hvs_m / 64 / 255^2 per block
    motion: Optional["MotionAnalysis"] = None  # noqa: F821  (bitstream/motion.py; P / B frames with motion=True)
    plane_mse: List[float] = field(init=False)

    def __post_init__(self):
        m2 = float(2**self.bitdepth - 1) ** 2
        self.plane_mse = [s / m2 / n for s, n in zip(self.sse, self.n_samples)]

    @property
    def rate_bpp(self) -> float:
        return 8 * self.n_bytes / (self.img_size[0] * self.img_size[1])

    @property
    def mse(self) -> float:
        return sum(self.sse) / float(2**self.bitdepth - 1) ** 2 / sum(self.n_samples)

    @property
    def psnr_db(self) -> float:
        return dist_to_db(self.mse)

    mse_y = property(lambda self: self.plane_mse[0])
    mse_u = property(lambda self: self.plane_mse[1])
    mse_v = property(lambda self: self.plane_mse[2])
    psnr_y_db = property(lambda self: dist_to_db(self.plane_mse[0]))
    psnr_u_db = property(lambda self: dist_to_db(self.plane_mse[1]))
    psnr_v_db = property(lambda self: dist_to_db(self.plane_mse[2]))

    @property
    def ms_ssim(self) -> Optional[float]:
        """Pixel-weighted mean of the planes' MS-SSIM (the rule of training/loss.py:121-155)."""
        if self.ms_ssim_planes is None:
            return None
        return sum(n * m for n, m in zip(self.n_samples, self.ms_ssim_planes)) / sum(self.n_samples)

    @property
    def ms_ssim_db(self) -> Optional[float]:
        return None if self.ms_ssim_planes is None else dist_to_db(1.0 - self.ms_ssim)

    ms_ssim_y = property(lambda self: None if self.ms_ssim_planes is None else self.ms_ssim_planes[0])
    ms_ssim_u = property(lambda self: None if self.ms_ssim_planes is None else self.ms_ssim_planes[1])
    ms_ssim_v = property(lambda self: None if self.ms_ssim_planes is None else self.ms_ssim_planes[2])

    @property
    def vif(self) -> Optional[float]:
        """Pixel-weighted mean of the planes' VIF (the rule of ms_ssim); None if a plane has none."""
        if self.vif_planes is None or any(v is None for v in self.vif_planes):
            return None
        return sum(n * v for n, v in zip(self.n_samples, self.vif_planes)) / sum(self.n_samples)

    vif_y = property(lambda self: None if self.vif_planes is None else self.vif_planes[0])
    vif_u = property(lambda self: None if self.vif_planes is None else self.vif_planes[1])
    vif_v = property(lambda self: None if self.vif_planes is None else self.vif_planes[2])

    def _hvs_db(self, k: int, planes) -> Optional[float]:
        if self.hvs_planes is None:
            return None
        return hvs_from_sums([self.hvs_planes[c][k] for c in planes], [self.hvs_planes[c][2] for c in planes])

    psnr_hvs_m_db = property(lambda self: self._hvs_db(0, (0, 1, 2)))
    psnr_hvs_db = property(lambda self: self._hvs_db(1, (0, 1, 2)))
    psnr_hvs_m_y_db = property(lambda self: self._hvs_db(0, (0,)))
    psnr_hvs_m_u_db = property(lambda self: self._hvs_db(0, (1,)))
    psnr_hvs_m_v_db = property(lambda self: self._hvs_db(0, (2,)))


def _frame_layout(buf, max_decoding_order: int):
    """Per frame in coding order: (frame header, display index, n_bytes, (h, w)), without decoding anything."""
    video_header = VideoHeader()
    buf = video_header.read_header(buf)
    cs = video_header.get_coding_structure()
    if max_decoding_order == -1:
        max_decoding_order = cs.get_max_coding_order()
    out = []
    for coding_idx in range(max_decoding_order + 1):
        n = len(buf)
        fh, ccs, buf = decode._parse_frame(buf)
        p = ccs["residue"][0].get_coolchic_parameter()
        out.append((fh, cs.get_frame_from_coding_order(coding_idx).display_order, n - len(buf),
                    (int(p.img_size[0]), int(p.img_size[1]))))
    return out


def _read_sources(frames, original_path: str, frame_offset: int):
    """``{display_idx: (coding_idx, frame header, n_bytes, source samples)}`` for the frames of _frame_layout.  A source
    whose format, bitdepth or size differs from the decoded frame, or that has too few frames, raises ValueError."""
    by_display = {}
    for coding_idx, (fh, disp, n_bytes, size) in enumerate(frames):
        fmt, b = fh.get_value("frame_data_type"), fh.get_value("bitdepth")
        try:
            s = read_samples(original_path, frame_offset + disp)
        except ValueError as e:
            raise ValueError(f"source {original_path} has no frame {frame_offset + disp} for decoded frame {disp}: {e}") from None
        if (s.frame_data_type, s.bitdepth, tuple(s.img_size)) != (fmt, b, size):
            raise ValueError(f"source frame {frame_offset + disp} of {original_path} is {s.img_size[1]}x{s.img_size[0]} "
                             f"{s.frame_data_type} {s.bitdepth}-bit, decoded frame {disp} is {size[1]}x{size[0]} {fmt} {b}-bit")
        by_display[disp] = (coding_idx, fh, n_bytes, s)
    return by_display


def _upload_sources(ctx, by_display):
    """Every source frame of _read_sources in one pinned buffer, one host-to-device copy: ``{display_idx: samples}``
    on the device (uint8, or int16 holding the uint16 samples)."""
    offs, total = {}, 0
    for disp, (_, _, _, s) in by_display.items():
        offs[disp] = total
        total += (s.samples.nbytes + 255) // 256 * 256
    host = torch.empty((total,), dtype=torch.uint8, pin_memory=True)
    hv = host.numpy()
    for disp, (_, _, _, s) in by_display.items():
        hv[offs[disp]:offs[disp] + s.samples.nbytes] = s.samples.reshape(-1).view(np.uint8)
    dev_all = host.to(ctx.torch_device, non_blocking=True)
    sources = {}
    for disp, (_, _, _, s) in by_display.items():
        raw = dev_all[offs[disp]:offs[disp] + s.samples.nbytes]
        sources[disp] = raw if s.samples.itemsize == 1 else raw.view(torch.int16)
    return sources


@torch.no_grad()
def video_quality(bitstream_bytes: bytes, original_path: str, frame_offset: int = 0, max_decoding_order: int = -1,
                  device: int = 0, want_maps: bool = False, ms_ssim: bool = False,
                  motion: bool = False, vif: bool = False, psnr_hvs: bool = False) -> Dict[str, FrameQuality]:
    """Quality of every frame of an image / video bitstream against its source file (.yuv / .png / .ppm):
    ``{str(display_idx): FrameQuality}`` in display order.  ``ms_ssim`` adds MS-SSIM for every frame whose planes
    all have both sides >= 176 (``ms_ssim_planes`` stays None for the others), with the SSIM maps if ``want_maps``.
    ``motion`` fills ``FrameQuality.motion`` of every P / B frame (a MotionAnalysis, with the flow maps if
    ``want_maps``); I frames keep None.  ``vif`` adds VIF for every frame whose planes all have both sides >= 41
    (``vif_planes`` stays None for the others).  ``psnr_hvs`` adds PSNR-HVS-M and PSNR-HVS for every frame whose
    planes all have both sides >= 8 (``hvs_planes`` stays None for the others), with the block maps if ``want_maps``.
    A source whose format, bitdepth or size differs from the
    decoded frames, or that has too few frames, raises ValueError before anything runs on the device."""
    frames = _frame_layout(memoryview(bytes(bitstream_bytes)), max_decoding_order)
    by_display = _read_sources(frames, original_path, frame_offset)
    ctx = _native.get_context(device)
    sources = _upload_sources(ctx, by_display)

    display_of = {coding_idx: disp for disp, (coding_idx, _, _, _) in by_display.items()}
    from .motion import motion_analysis

    stats, motions = {}, {}
    calls = [0]

    def reconstruct(frame_header, cc_out, reference_frames, dev):
        disp = display_of[calls[0]]
        calls[0] += 1
        ftype = frame_header.get_value("frame_type")
        if ftype in ("P", "B"):
            refs = [r.to(ctx.torch_device) for r in reference_frames]
            stats[disp] = ctx.inter_stats(
                cc_out["residue"], cc_out["motion"], refs, ftype == "B", frame_header.get_value("frame_data_type"),
                frame_header.get_value("bitdepth"), frame_header.get_value("global_flow"),
                frame_header.get_value("warp_filter_size"), source=sources[disp], layout=by_display[disp][3].layout,
                want_maps=want_maps)
            if motion:
                s = by_display[disp][3]
                r = ctx.inter_analysis(
                    cc_out["residue"], cc_out["motion"], refs, ftype == "B", s.frame_data_type, s.bitdepth,
                    frame_header.get_value("global_flow"), frame_header.get_value("warp_filter_size"),
                    source=sources[disp], layout=s.layout, want_maps=want_maps)
                motions[disp] = motion_analysis(r, ftype, s.bitdepth, s.img_size, s.frame_data_type,
                                                frame_header.get_value("global_flow"))
        return decode._reconstruct(frame_header, cc_out, reference_frames, dev)

    decoded = decode.decode_video_bytes(bitstream_bytes, max_decoding_order=max_decoding_order, device=device,
                                        output_device="cuda", reconstruct_fn=reconstruct)
    order = sorted(by_display)
    dist = ctx.frame_distortion([decoded[str(d)] for d in order], [sources[d] for d in order],
                                [by_display[d][3].layout for d in order], want_maps=want_maps)
    ssim = {}
    if ms_ssim:
        big = [d for d in order if ms_ssim_applies(by_display[d][3].img_size, by_display[d][3].frame_data_type)]
        if big:
            res = ctx.frame_ssim([decoded[str(d)] for d in big], [sources[d] for d in big],
                                 [by_display[d][3].layout for d in big], want_maps=want_maps)
            ssim = dict(zip(big, res))
    vifs = {}
    if vif:
        big = [d for d in order if vif_applies(by_display[d][3].img_size, by_display[d][3].frame_data_type)]
        if big:
            res = ctx.frame_vif([decoded[str(d)] for d in big], [sources[d] for d in big],
                                [by_display[d][3].layout for d in big])
            vifs = dict(zip(big, res))
    hvs = {}
    if psnr_hvs:
        big = [d for d in order if hvs_applies(by_display[d][3].img_size, by_display[d][3].frame_data_type)]
        if big:
            res = ctx.frame_hvs([decoded[str(d)] for d in big], [sources[d] for d in big],
                                [by_display[d][3].layout for d in big], want_maps=want_maps)
            hvs = dict(zip(big, res))
    out = {}
    for d, r in zip(order, dist):
        _, fh, n_bytes, s = by_display[d]
        h, w = s.img_size
        cs = 1 if s.frame_data_type == "yuv420" else 0
        q = FrameQuality(display_idx=d, frame_type=fh.get_value("frame_type"), img_size=(h, w), bitdepth=s.bitdepth,
                         frame_data_type=s.frame_data_type, n_bytes=n_bytes, sse=r["sse"],
                         n_samples=[h * w] + [(h >> cs) * (w >> cs)] * 2, max_abs=r["max_abs"],
                         error_map=r.get("map"))
        if d in stats:
            st = stats[d]
            q.alpha_mean = st["sums"][0] / (h * w)
            q.beta_mean = st["sums"][1] / (h * w)
            q.pred_psnr_db = pred_to_db(st["sums"][2], 3 * h * w)
            q.dummy_pred_psnr_db = pred_to_db(st["sums"][3], 3 * h * w)
            q.alpha_map, q.beta_map, q.pred_map = st.get("alpha"), st.get("beta"), st.get("pred")
        q.motion = motions.get(d)
        if d in ssim:
            q.ms_ssim_planes = [ms_ssim_from_scales(c, s_) for c, s_ in zip(ssim[d]["cs"], ssim[d]["ssim"])]
            q.ssim_maps = ssim[d].get("maps")
        if d in vifs:
            q.vif_planes = [vif_from_scales(n_, d_) for n_, d_ in zip(vifs[d]["num"], vifs[d]["den"])]
        if d in hvs:
            q.hvs_planes = list(zip(hvs[d]["s_hvs_m"], hvs[d]["s_hvs"], hvs[d]["n_coeffs"]))
            q.hvs_maps = hvs[d].get("maps")
        out[str(d)] = q
    return out
