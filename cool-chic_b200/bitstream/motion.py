"""Motion analysis of a P / B frame (DESIGN §4.9): what the motion, each reference and the residue buy.

A variant is the finished frame ``decode_frame`` reconstructs (``bitstream/decode.py:155-206``) with one change to its
decoder inputs; everything else comes from the bitstream.  Its PSNR against the source, whole and per plane, and the
change from the decoded frame's PSNR say what the changed input contributes.  Each override is exact
(``clamp01(±0.5 + 0.5)`` is 0 or 1), so a variant is defined bit for bit by reconstructing the modified inputs.

Per reference, the statistics of its flow over the luma pixels: the mean total displacement (local + global), the
mean and the largest length of the local flow, and how many pixels sample the reference outside its borders (where
the warp reads clamped border samples).

One ``ccd_inter_analysis`` launch per P / B frame computes all of it, from the residue and motion the decoder is about
to use (``video_quality(..., motion=True)``).
"""
from dataclasses import dataclass
from typing import List, Optional

from .quality import dist_to_db

# (name, input change, B only), in the order of ccdec.h's CcdInterAnalysis
VARIANTS = [
    ("decoded", "none", False),
    ("no_local_motion", "every motion channel := 0, global flow kept", False),
    ("no_motion", "every motion channel := 0 and global flow := 0", False),
    ("ref0_only", "residue channel 4 := +0.5 (beta = 1)", True),
    ("ref1_only", "residue channel 4 := -0.5 (beta = 0)", True),
    ("no_residue", "residue channels 0-2 := 0", False),
    ("no_prediction", "residue channel 3 := -0.5 (alpha = 0)", False),
]
VARIANT_NAMES = [v[0] for v in VARIANTS]


def variants_of(frame_type: str) -> List[str]:
    """The variants that apply to a P or B frame."""
    return [name for name, _, b_only in VARIANTS if frame_type == "B" or not b_only]


def _copy(x):
    return x.clone() if hasattr(x, "clone") else x.copy()


def variant_inputs(residue, motion, global_flow, variant: str):
    """(residue, motion, global_flow) of ``variant``: copies of the decoder inputs with the variant's change.  residue
    and motion are numpy arrays or torch tensors whose last three axes are [channel, H, W]; global_flow is the frame
    header's list (x, y per reference)."""
    if variant not in VARIANT_NAMES:
        raise ValueError(f"unknown variant {variant!r}")
    is_b = residue.shape[-3] == 5
    if dict((n, b) for n, _, b in VARIANTS)[variant] and not is_b:
        raise ValueError(f"{variant} applies to B frames only")
    residue, motion, global_flow = _copy(residue), _copy(motion), list(global_flow)
    if variant in ("no_local_motion", "no_motion"):
        motion[..., :, :, :] = 0.0
    if variant == "no_motion":
        global_flow = [0] * len(global_flow)
    if variant == "ref0_only":
        residue[..., 4, :, :] = 0.5
    if variant == "ref1_only":
        residue[..., 4, :, :] = -0.5
    if variant == "no_residue":
        residue[..., 0:3, :, :] = 0.0
    if variant == "no_prediction":
        residue[..., 3, :, :] = -0.5
    return residue, motion, global_flow


@dataclass
class RefMotion:
    """Flow statistics of one reference over the luma pixels (in pixels of the frame)."""
    global_flow: tuple            # (gx, gy)
    mean_flow: tuple              # mean of (fx + gx, fy + gy)
    mean_local: float             # mean of sqrt(fx^2 + fy^2)
    max_local: float              # max of sqrt(fx^2 + fy^2)
    outside: int                  # pixels whose sample position falls outside the reference
    n_pixels: int
    flow_map: Optional[object] = None   # [2, H, W] fp32 fx + gx, fy + gy

    @property
    def outside_fraction(self) -> float:
        return self.outside / self.n_pixels


@dataclass
class MotionAnalysis:
    """Motion analysis of one P / B frame.  ``sse[v]``: per plane, the exact sum of squared integer errors of variant
    v against the source (None where v does not apply); planes are y / u / v, or r / g / b for rgb frames."""
    frame_type: str
    bitdepth: int
    n_samples: List[int]
    sse: dict
    refs: List[RefMotion]

    def _mse(self, s):
        return s / float(2**self.bitdepth - 1) ** 2

    def psnr_db(self, variant: str) -> Optional[float]:
        """Frame PSNR of a variant: the pixel-weighted MSE over the planes (loss.py:88-118), dist_to_db."""
        s = self.sse[variant]
        return None if s is None else dist_to_db(self._mse(sum(s)) / sum(self.n_samples))

    def plane_psnr_db(self, variant: str) -> Optional[List[float]]:
        s = self.sse[variant]
        return None if s is None else [dist_to_db(self._mse(x) / n) for x, n in zip(s, self.n_samples)]

    def delta_db(self, variant: str) -> Optional[float]:
        """The variant's PSNR minus the decoded frame's (negative: the changed input was worth that much)."""
        p = self.psnr_db(variant)
        return None if p is None else p - self.psnr_db("decoded")


def motion_analysis(result: dict, frame_type: str, bitdepth: int, img_size, frame_data_type: str,
                    global_flow) -> MotionAnalysis:
    """MotionAnalysis from what ``Context.inter_analysis`` returns for the frame."""
    h, w = img_size
    cs = 1 if frame_data_type == "yuv420" else 0
    gf = (list(global_flow) + [0, 0, 0, 0])[:4]
    refs = []
    for r, st in enumerate(result["refs"]):
        refs.append(RefMotion(global_flow=(gf[2 * r], gf[2 * r + 1]), mean_flow=(st["sum"][0] / (h * w), st["sum"][1] / (h * w)),
                              mean_local=st["sum"][2] / (h * w), max_local=st["max"], outside=st["outside"],
                              n_pixels=h * w, flow_map=st.get("flow")))
    return MotionAnalysis(frame_type=frame_type, bitdepth=bitdepth, n_samples=[h * w] + [(h >> cs) * (w >> cs)] * 2,
                          sse=dict(zip(VARIANT_NAMES, result["sse"])), refs=refs)
