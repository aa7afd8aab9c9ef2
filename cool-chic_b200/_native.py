"""ctypes binding of ``csrc/libccdec.so`` (C-ABI in ``include/ccdec.h``).

There is no CPU fallback: if the shared library is missing or no CUDA device is present,
loading / context creation raises ``RuntimeError``.  PyTorch tensors are only used as owners
of device memory (``tensor.data_ptr()``) and of the CUDA stream.
"""
import ctypes
import os
import threading
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

from ._desc import CCD_MAX_GRIDS, CcdCoolChicDesc

_HERE = os.path.dirname(os.path.abspath(__file__))
# CCD_LIB lets a developer load the instrumented build (csrc/libccdec_prof.so)
LIB_PATH = os.environ.get("CCD_LIB") or os.path.join(_HERE, "csrc", "libccdec.so")

CCD_OK = 0
ERROR_NAMES = {
    -1: "CCD_ERR_ARG", -2: "CCD_ERR_NN_TRUNCATED", -3: "CCD_ERR_DESYNC", -4: "CCD_ERR_UNSUPPORTED",
    -5: "CCD_ERR_NOMEM", -6: "CCD_ERR_CUDA", -7: "CCD_ERR_NO_DEVICE",
}

EXPORTS = [
    "ccd_version", "ccd_sizeof_desc", "ccd_last_error", "ccd_create", "ccd_destroy", "ccd_nn_count",
    "ccd_latent_count", "ccd_decode_nn", "ccd_decode_many", "ccd_decode_coolchic", "ccd_decode_latents",
    "ccd_encode_latents", "ccd_synthesize_many", "ccd_finish_frame", "ccd_reconstruct_frame", "ccd_pack_frame", "ccd_pack_samples",
    "ccd_latent_rate", "ccd_latent_rate_edited", "ccd_rate_sweep", "ccd_rate_candidates", "ccd_frame_distortion", "ccd_frame_ssim", "ccd_frame_vif", "ccd_frame_hvs", "ccd_inter_stats", "ccd_inter_analysis",
    "ccd_debug_laplace_domain", "ccd_debug_last_status", "ccd_debug_launch_count", "ccd_debug_set_producer_mask", "ccd_last_timing",
    "ccd_debug_entropy_plan", "ccd_debug_cdf_table", "ccd_debug_detmath", "ccd_debug_sinc_coeffs", "ccd_debug_cr_noise",
]


class CcdEntropyState(ctypes.Structure):
    """Where a progressive decode stopped (DESIGN §4.8): ``grids_done`` decode-order grids, ``words_consumed`` payload
    words; the rest is the range decoder's state and the identity of its stream."""
    _fields_ = [
        ("grids_done", ctypes.c_int32),
        ("reserved", ctypes.c_int32),
        ("words_consumed", ctypes.c_int64),
        ("opaque", ctypes.c_uint64 * 6),
    ]


class CcdJob(ctypes.Structure):
    _fields_ = [
        ("desc", ctypes.POINTER(CcdCoolChicDesc)),
        ("nn_bytes", ctypes.c_char_p),
        ("nn_nbytes", ctypes.c_size_t),
        ("latent_bytes", ctypes.c_char_p),
        ("latent_nbytes", ctypes.c_size_t),
        ("d_out", ctypes.c_void_p),
        ("d_latents", ctypes.c_void_p),
        ("status", ctypes.c_int32),
        ("finish_bitdepth", ctypes.c_int32),
        ("finish_type", ctypes.c_int32),
        ("d_out_u", ctypes.c_void_p),
        ("d_out_v", ctypes.c_void_p),
        ("grid_end", ctypes.c_int32),
        ("state", ctypes.POINTER(CcdEntropyState)),
    ]


class CcdSynthJob(ctypes.Structure):
    _fields_ = [
        ("desc", ctypes.POINTER(CcdCoolChicDesc)),
        ("nn_ints", ctypes.c_void_p),
        ("d_latents", ctypes.c_void_p),
        ("zero_grids", ctypes.c_uint32),
        ("d_out", ctypes.c_void_p),
        ("finish_bitdepth", ctypes.c_int32),
        ("finish_type", ctypes.c_int32),
        ("d_out_u", ctypes.c_void_p),
        ("d_out_v", ctypes.c_void_p),
        ("status", ctypes.c_int32),
    ]


class CcdRateJob(ctypes.Structure):
    _fields_ = [
        ("desc", ctypes.POINTER(CcdCoolChicDesc)),
        ("nn_ints", ctypes.c_void_p),
        ("d_latents", ctypes.c_void_p),
        ("d_bits", ctypes.c_void_p),
        ("d_freq", ctypes.c_void_p),
        ("d_mu_sc", ctypes.c_void_p),
        ("d_spatial", ctypes.c_void_p),
        ("grid_bits", ctypes.c_double * CCD_MAX_GRIDS),
        ("bad_index", ctypes.c_int64),
        ("status", ctypes.c_int32),
    ]


class CcdModelEdit(ctypes.Structure):
    """ARM inputs read as 0 (DESIGN §4.10): spatial inputs (bits of ``zero_ctx``), IFCE features (``zero_ifce_out``),
    latent grids wherever they are an IFCE input (``zero_ifce_grids``, bit 0 = the finest grid)."""
    _fields_ = [
        ("zero_ctx", ctypes.c_uint64),
        ("zero_ifce_out", ctypes.c_uint32),
        ("zero_ifce_grids", ctypes.c_uint32),
    ]


SWEEP_MAX_OFFSETS = 32  # CCD_SWEEP_MAX_OFFSETS


class CcdCandidate(ctypes.Structure):
    _fields_ = [("nn_index", ctypes.c_int32), ("delta", ctypes.c_int32)]


CCD_CAND_MAX = 64


class CcdSweepJob(ctypes.Structure):
    _fields_ = [
        ("desc", ctypes.POINTER(CcdCoolChicDesc)),
        ("d_latents", ctypes.c_void_p),
        ("d_mu_sc", ctypes.c_void_p),
        ("n_offsets", ctypes.c_int32),
        ("sc_offset", ctypes.c_int32 * SWEEP_MAX_OFFSETS),
        ("bits", (ctypes.c_double * SWEEP_MAX_OFFSETS) * CCD_MAX_GRIDS),
        ("hist", (ctypes.c_uint64 * 128) * CCD_MAX_GRIDS),
        ("bad_index", ctypes.c_int64),
        ("status", ctypes.c_int32),
    ]


# The frame jobs (CcdDistJob, CcdSsimJob, CcdVifJob, CcdHvsJob): the same inputs, their own results, the same tail
_FRAME_JOB_INPUTS = [
    ("d_planes", ctypes.c_void_p * 3),
    ("d_src", ctypes.c_void_p),
    ("h", ctypes.c_int32),
    ("w", ctypes.c_int32),
    ("chroma_shift", ctypes.c_int32),
    ("bitdepth", ctypes.c_int32),
    ("src_layout", ctypes.c_int32),
]
_FRAME_JOB_TAIL = [("bad_index", ctypes.c_int64), ("status", ctypes.c_int32)]


class CcdDistJob(ctypes.Structure):
    _fields_ = _FRAME_JOB_INPUTS + [("d_map", ctypes.c_void_p), ("sse", ctypes.c_uint64 * 3),
                                    ("max_abs", ctypes.c_uint32 * 3)] + _FRAME_JOB_TAIL


class CcdSsimJob(ctypes.Structure):
    _fields_ = _FRAME_JOB_INPUTS + [("d_map", ctypes.c_void_p * 3), ("cs", (ctypes.c_double * 5) * 3),
                                    ("ssim", (ctypes.c_double * 5) * 3)] + _FRAME_JOB_TAIL


class CcdVifJob(ctypes.Structure):
    _fields_ = _FRAME_JOB_INPUTS + [("num", (ctypes.c_double * 4) * 3), ("den", (ctypes.c_double * 4) * 3)] + _FRAME_JOB_TAIL


class CcdHvsJob(ctypes.Structure):
    _fields_ = _FRAME_JOB_INPUTS + [("d_map", ctypes.c_void_p * 3), ("s_hvs_m", ctypes.c_double * 3),
                                    ("s_hvs", ctypes.c_double * 3)] + _FRAME_JOB_TAIL


def _source_fits(src, h, w, cs, bitdepth):
    """(dtype ok, expected sample count) of source samples for an h x w frame with chroma shift cs: a contiguous CUDA
    tensor, uint8 up to 8 bits and int16 (holding uint16) above, of h w + 2 (h >> cs)(w >> cs) samples"""
    dtype_ok = src.is_cuda and src.is_contiguous() and src.dtype == (torch.uint8 if bitdepth <= 8 else torch.int16)
    return dtype_ok, h * w + 2 * (h >> cs) * (w >> cs)


def _check_symbols(name, t, n, dtype=torch.int8, label="int8"):
    """A ValueError naming t and its type (label) unless t is a contiguous dtype CUDA tensor of n symbols"""
    if not (t.is_cuda and t.dtype == dtype and t.is_contiguous() and t.numel() == n):
        raise ValueError(f"{name} must be a contiguous {label} CUDA tensor of {n} symbols")


class CcdInterFrame(ctypes.Structure):
    _fields_ = [
        ("d_residue", ctypes.c_void_p),
        ("n_res_ch", ctypes.c_int32),
        ("d_motion", ctypes.c_void_p),
        ("n_mot_ch", ctypes.c_int32),
        ("ref0", ctypes.c_void_p * 3),
        ("ref1", ctypes.c_void_p * 3),
        ("frame_data_type", ctypes.c_int32),
        ("bitdepth", ctypes.c_int32),
        ("h", ctypes.c_int32),
        ("w", ctypes.c_int32),
        ("is_b", ctypes.c_int32),
        ("global_flow", ctypes.c_int32 * 4),
        ("warp_filter_size", ctypes.c_int32),
    ]


class CcdInterStats(ctypes.Structure):
    _fields_ = [
        ("d_src", ctypes.c_void_p),
        ("src_layout", ctypes.c_int32),
        ("d_alpha", ctypes.c_void_p),
        ("d_beta", ctypes.c_void_p),
        ("d_pred", ctypes.c_void_p),
        ("sums", ctypes.c_double * 4),
    ]


INTER_VARIANTS = 7  # CCD_INTER_VARIANTS


class CcdInterAnalysis(ctypes.Structure):
    _fields_ = [
        ("d_src", ctypes.c_void_p),
        ("src_layout", ctypes.c_int32),
        ("d_flow", ctypes.c_void_p * 2),
        ("sse", (ctypes.c_uint64 * 3) * INTER_VARIANTS),
        ("flow_sum", (ctypes.c_double * 3) * 2),
        ("flow_max", ctypes.c_double * 2),
        ("outside", ctypes.c_uint64 * 2),
        ("bad_index", ctypes.c_int64),
        ("status", ctypes.c_int32),
    ]


SOURCE_LAYOUTS = {"planar": 0, "hwc": 1}


class CcdError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"{ERROR_NAMES.get(code, code)}: {msg}")
        self.code = code


_lib = None
_lib_lock = threading.Lock()


def load_library():
    """Load libccdec.so (once).  Raises RuntimeError if it has not been built."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(or `make -C cool-chic_b200/csrc`).  There is no CPU fallback."
            )
        L = ctypes.CDLL(LIB_PATH)
        vp, sz, i64, ci = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64, ctypes.c_int
        pd = ctypes.POINTER(CcdCoolChicDesc)
        L.ccd_version.restype = ci
        L.ccd_sizeof_desc.restype = ci
        L.ccd_last_error.restype = ctypes.c_char_p
        L.ccd_last_error.argtypes = [vp]
        L.ccd_create.restype = ci
        L.ccd_create.argtypes = [ci, ctypes.POINTER(vp)]
        L.ccd_destroy.restype = None
        L.ccd_destroy.argtypes = [vp]
        L.ccd_nn_count.restype = i64
        L.ccd_nn_count.argtypes = [pd]
        L.ccd_latent_count.restype = i64
        L.ccd_latent_count.argtypes = [pd, vp]
        L.ccd_decode_nn.restype = i64
        L.ccd_decode_nn.argtypes = [pd, ctypes.c_char_p, sz, vp, sz]
        L.ccd_decode_many.restype = ci
        L.ccd_decode_many.argtypes = [vp, ctypes.POINTER(CcdJob), ci, vp]
        L.ccd_decode_coolchic.restype = ci
        L.ccd_decode_coolchic.argtypes = [vp, pd, ctypes.c_char_p, sz, ctypes.c_char_p, sz, vp, vp, vp]
        L.ccd_decode_latents.restype = ci
        L.ccd_decode_latents.argtypes = [vp, pd, vp, ctypes.c_char_p, sz, vp, vp]
        L.ccd_encode_latents.restype = ci
        L.ccd_encode_latents.argtypes = [vp, pd, vp, ci, ctypes.c_uint64, vp, vp, i64, vp, vp, vp]
        L.ccd_synthesize_many.restype = ci
        L.ccd_synthesize_many.argtypes = [vp, ctypes.POINTER(CcdSynthJob), ci, vp]
        L.ccd_finish_frame.restype = ci
        L.ccd_finish_frame.argtypes = [vp, vp, ci, ci, ci, ci, vp, vp, vp, vp]
        L.ccd_reconstruct_frame.restype = ci
        L.ccd_reconstruct_frame.argtypes = [vp, ctypes.POINTER(CcdInterFrame), vp, vp]
        L.ccd_pack_frame.restype = ci
        L.ccd_pack_frame.argtypes = [vp, vp, ci, ci, ci, ci, ci, ci, vp, vp]
        L.ccd_pack_samples.restype = ci
        L.ccd_pack_samples.argtypes = [vp, vp, ctypes.c_size_t, ci, ci, vp, vp]
        L.ccd_latent_rate.restype = ci
        L.ccd_latent_rate.argtypes = [vp, ctypes.POINTER(CcdRateJob), ci, vp]
        L.ccd_latent_rate_edited.restype = ci
        L.ccd_latent_rate_edited.argtypes = [vp, ctypes.POINTER(CcdRateJob), ctypes.POINTER(CcdModelEdit), ci, vp]
        L.ccd_rate_sweep.restype = ci
        L.ccd_rate_candidates.restype = ci
        L.ccd_rate_candidates.argtypes = [vp, pd, vp, vp, ctypes.POINTER(CcdCandidate), ci, vp, vp, vp]
        L.ccd_rate_sweep.argtypes = [vp, ctypes.POINTER(CcdSweepJob), ci, vp]
        L.ccd_frame_distortion.restype = ci
        L.ccd_frame_distortion.argtypes = [vp, ctypes.POINTER(CcdDistJob), ci, vp]
        L.ccd_frame_ssim.restype = ci
        L.ccd_frame_ssim.argtypes = [vp, ctypes.POINTER(CcdSsimJob), ci, vp]
        L.ccd_frame_vif.restype = ci
        L.ccd_frame_vif.argtypes = [vp, ctypes.POINTER(CcdVifJob), ci, vp]
        L.ccd_frame_hvs.restype = ci
        L.ccd_frame_hvs.argtypes = [vp, ctypes.POINTER(CcdHvsJob), ci, vp]
        L.ccd_inter_stats.restype = ci
        L.ccd_inter_stats.argtypes = [vp, ctypes.POINTER(CcdInterFrame), ctypes.POINTER(CcdInterStats), vp]
        L.ccd_inter_analysis.restype = ci
        L.ccd_inter_analysis.argtypes = [vp, ctypes.POINTER(CcdInterFrame), ctypes.POINTER(CcdInterAnalysis), vp]
        L.ccd_debug_laplace_domain.restype = ci
        L.ccd_debug_laplace_domain.argtypes = [vp, ci, ci, vp, vp]
        L.ccd_debug_cdf_table.restype = ci
        L.ccd_debug_cdf_table.argtypes = [vp, ci, ci, vp]
        L.ccd_debug_detmath.restype = ci
        L.ccd_debug_detmath.argtypes = [vp, ci, vp, vp, ctypes.c_size_t]
        L.ccd_debug_sinc_coeffs.restype = ci
        L.ccd_debug_sinc_coeffs.argtypes = [vp, ci, vp, vp, ctypes.c_size_t]
        L.ccd_debug_cr_noise.restype = ci
        L.ccd_debug_cr_noise.argtypes = [vp, ctypes.c_uint64, ctypes.c_size_t, vp]
        L.ccd_debug_last_status.restype = ci
        L.ccd_debug_last_status.argtypes = [vp, vp]
        L.ccd_debug_launch_count.restype = ctypes.c_uint64
        L.ccd_debug_launch_count.argtypes = []
        L.ccd_debug_set_producer_mask.restype = ci
        L.ccd_debug_set_producer_mask.argtypes = [vp, ctypes.c_uint32]
        L.ccd_last_timing.restype = ci
        L.ccd_last_timing.argtypes = [vp, vp]
        L.ccd_debug_entropy_plan.restype = ci
        L.ccd_debug_entropy_plan.argtypes = [pd, vp, vp]
        if L.ccd_sizeof_desc() != ctypes.sizeof(CcdCoolChicDesc):
            raise RuntimeError("CcdCoolChicDesc layout mismatch between Python and libccdec.so")
        _lib = L
        return _lib


def _check(rc: int, jobs=None) -> None:
    """Raises CcdError for a failing status; given the call's job array (one whose jobs have a bad_index), the error
    carries ``bad_index``, one per job."""
    if rc != CCD_OK:
        msg = load_library().ccd_last_error(None)
        err = CcdError(rc, msg.decode() if msg else "")
        if jobs is not None:
            err.bad_index = [int(j.bad_index) for j in jobs]
        raise err


def decode_nn(desc: CcdCoolChicDesc, nn_bytes: bytes) -> np.ndarray:
    """Host exp-Golomb decode of the NN payload -> int64 array (module/param order)."""
    L = load_library()
    n = L.ccd_nn_count(ctypes.byref(desc))
    if n < 0:
        _check(int(n))
    out = np.zeros(int(n), dtype=np.int64)
    got = L.ccd_decode_nn(ctypes.byref(desc), nn_bytes, len(nn_bytes), out.ctypes.data_as(ctypes.c_void_p), out.size)
    if got < 0:
        _check(int(got))
    return out


def entropy_plan(desc: CcdCoolChicDesc, nn_ints: np.ndarray):
    """Host-side shared-memory plan of the entropy kernel for one Cool-chic: (window-ring slots, row-ring rows,
    bytes).  Raises CcdError (CCD_ERR_UNSUPPORTED) when the stream does not fit, as decoding it would."""
    nn = np.ascontiguousarray(nn_ints, dtype=np.int64)
    out = np.zeros(3, dtype=np.int64)
    _check(load_library().ccd_debug_entropy_plan(ctypes.byref(desc), nn.ctypes.data_as(ctypes.c_void_p),
                                                  out.ctypes.data_as(ctypes.c_void_p)))
    return int(out[0]), int(out[1]), int(out[2])


def latent_layout(desc: CcdCoolChicDesc):
    L = load_library()
    offs = (ctypes.c_int64 * CCD_MAX_GRIDS)()
    n = L.ccd_latent_count(ctypes.byref(desc), offs)
    if n < 0:
        _check(int(n))
    return int(n), [int(offs[i]) for i in range(desc.n_grids)]


class Context:
    """One decoder context per CUDA device (``ccd_create`` / ``ccd_destroy``)."""

    def __init__(self, device: int = 0):
        self._lib = load_library()
        if not torch.cuda.is_available():
            raise RuntimeError("cool-chic_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback.")
        self.device = int(device)
        h = ctypes.c_void_p()
        _check(self._lib.ccd_create(self.device, ctypes.byref(h)))
        self._h = h
        self.torch_device = torch.device("cuda", self.device)

    def close(self) -> None:
        if getattr(self, "_h", None):
            self._lib.ccd_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return ctypes.c_void_p(torch.cuda.current_stream(self.torch_device).cuda_stream)

    # ---- whole Cool-chic(s) -----------------------------------------------------------
    def decode_many(self, descs: Sequence[CcdCoolChicDesc], nn_bytes: Sequence[bytes],
                    latent_bytes: Sequence[bytes], want_latents: bool = False, finish=None):
        """Decode n independent Cool-chics concurrently.  Returns (outputs, latents) where
        outputs[i] is a float32 CUDA tensor [1, C, H, W] (raw synthesis output).
        ``finish[i] = (bitdepth, frame_data_type)`` (or None) asks for decode_frame's frame tail (3-channel
        outputs only): outputs[i] is then the FINISHED frame in FrameData layout ([1, 3, H, W], or the
        y / u / v dictionary for yuv420)."""
        n = len(descs)
        jobs = (CcdJob * n)()
        lats = []
        outs = self._job_outputs(jobs, descs, finish)
        for i in range(n):
            d = descs[i]
            jobs[i].desc = ctypes.pointer(d)
            jobs[i].nn_bytes = nn_bytes[i]
            jobs[i].nn_nbytes = len(nn_bytes[i])
            jobs[i].latent_bytes = latent_bytes[i]
            jobs[i].latent_nbytes = len(latent_bytes[i])
            if want_latents:
                lat = torch.empty((d.n_symbols(),), dtype=torch.int8, device=self.torch_device)
                lats.append(lat)
                jobs[i].d_latents = lat.data_ptr()
            else:
                jobs[i].d_latents = None
        rc = self._lib.ccd_decode_many(self._h, jobs, n, self._stream())
        _check(rc)
        return outs, (lats if want_latents else None)

    def decode_stages(self, descs: Sequence[CcdCoolChicDesc], nn_bytes: Sequence[bytes], latent_bytes: Sequence[bytes],
                      grid_ends: Sequence[int], states=None, latents=None, finish=None):
        """One progressive stage per Cool-chic (``CcdJob.grid_end`` / ``state``, DESIGN §4.8), all in one call: the
        decode-order grids [grids_done, grid_ends[i]) of Cool-chic i (0: to the last), then its preview, every grid not
        decoded yet read as zeros.  ``states[i]``: a CcdEntropyState, read and updated in place, or None (decode from
        the first grid).  ``latents[i]``: an int8 CUDA tensor of n_symbols that keeps the decoded grids from one stage
        to the next (required with a state), or None (library-owned).  Outputs as decode_many's, ``finish`` included."""
        n = len(descs)
        jobs = (CcdJob * n)()
        outs = self._job_outputs(jobs, descs, finish)
        for i in range(n):
            d = descs[i]
            jobs[i].desc = ctypes.pointer(d)
            jobs[i].nn_bytes = nn_bytes[i]
            jobs[i].nn_nbytes = len(nn_bytes[i])
            jobs[i].latent_bytes = latent_bytes[i]
            jobs[i].latent_nbytes = len(latent_bytes[i])
            jobs[i].grid_end = int(grid_ends[i])
            lat = latents[i] if latents is not None else None
            if lat is not None:
                _check_symbols(f"latents[{i}]", lat, d.n_symbols())
                jobs[i].d_latents = lat.data_ptr()
            st = states[i] if states is not None else None
            if st is not None:
                jobs[i].state = ctypes.pointer(st)
        _check(self._lib.ccd_decode_many(self._h, jobs, n, self._stream()))
        return outs

    def _job_outputs(self, jobs, descs, finish):
        """The outputs of a job array whose jobs take CcdJob's output fields (d_out, d_out_u, d_out_v, finish_bitdepth,
        finish_type): per job a raw [1, C, H, W] tensor, or with ``finish[i]`` the finished frame in FrameData layout.
        All outputs are slices of ONE buffer, frame after frame, plane after plane: a batch of finished planar frames is
        then already in output order (pack_frames: one launch, one copy to the host for the whole batch)."""
        n = len(descs)
        fins = [finish[i] if finish is not None else None for i in range(n)]
        sizes = []
        for d, fin in zip(descs, fins):
            if fin is not None and fin[1] == "yuv420":
                sizes.append(d.img_h * d.img_w + 2 * (d.img_h // 2) * (d.img_w // 2))
            else:
                sizes.append(d.n_out_channels * d.img_h * d.img_w)
        slab = torch.empty((sum(sizes),), dtype=torch.float32, device=self.torch_device)
        outs, off = [], 0
        for i, (d, fin) in enumerate(zip(descs, fins)):
            if fin is not None and fin[1] == "yuv420":
                h, w = d.img_h, d.img_w
                ny, nc = h * w, (h // 2) * (w // 2)
                out = {"y": slab[off:off + ny].view(1, 1, h, w),
                       "u": slab[off + ny:off + ny + nc].view(1, 1, h // 2, w // 2),
                       "v": slab[off + ny + nc:off + ny + 2 * nc].view(1, 1, h // 2, w // 2)}
                jobs[i].d_out = out["y"].data_ptr()
                jobs[i].d_out_u = out["u"].data_ptr()
                jobs[i].d_out_v = out["v"].data_ptr()
            else:
                out = slab[off:off + sizes[i]].view(1, d.n_out_channels, d.img_h, d.img_w)
                jobs[i].d_out = out.data_ptr()
            off += sizes[i]
            if fin is not None:
                jobs[i].finish_bitdepth = int(fin[0])
                jobs[i].finish_type = _frame_type_code(fin[1])
            outs.append(out)
        return outs

    def synthesize(self, descs: Sequence[CcdCoolChicDesc], nn_ints: Sequence[np.ndarray],
                   latents: Sequence[torch.Tensor], zero_grids: Sequence[int], finish=None):
        """The float tail of decode_many on given latents (``ccd_synthesize_many``): ``latents[i]`` is an int8 CUDA
        tensor in decode order (what ``decode_many(want_latents=True)`` returns), read only; bit g of ``zero_grids[i]``
        reads grid g (0 = finest, a synthesis grid) as all zeros.  Outputs as decode_many's, ``finish`` included."""
        n = len(descs)
        jobs = (CcdSynthJob * n)()
        outs = self._job_outputs(jobs, descs, finish)
        keep = []
        for i in range(n):
            d = descs[i]
            nn = np.ascontiguousarray(nn_ints[i], dtype=np.int64)
            lat = latents[i]
            _check_symbols(f"latents[{i}]", lat, d.n_symbols())
            keep += [nn, lat]
            jobs[i].desc = ctypes.pointer(d)
            jobs[i].nn_ints = nn.ctypes.data
            jobs[i].d_latents = lat.data_ptr()
            jobs[i].zero_grids = int(zero_grids[i])
        _check(self._lib.ccd_synthesize_many(self._h, jobs, n, self._stream()))
        return outs

    def decode_coolchic(self, desc, nn_bytes: bytes, latent_bytes: bytes, want_latents: bool = False):
        outs, lats = self.decode_many([desc], [nn_bytes], [latent_bytes], want_latents)
        return (outs[0], lats[0]) if want_latents else outs[0]

    # ---- stages -----------------------------------------------------------------------
    def decode_latents(self, desc, nn_ints: np.ndarray, latent_bytes: bytes) -> torch.Tensor:
        nn_ints = np.ascontiguousarray(nn_ints, dtype=np.int64)
        lat = torch.empty((desc.n_symbols(),), dtype=torch.int8, device=self.torch_device)
        _check(self._lib.ccd_decode_latents(self._h, ctypes.byref(desc), nn_ints.ctypes.data_as(ctypes.c_void_p),
                                            latent_bytes, len(latent_bytes), lat.data_ptr(), self._stream()))
        return lat

    def encode_latents(self, desc, nn_ints: np.ndarray, latents: Optional[torch.Tensor] = None,
                       seed: Optional[int] = None):
        """Range-encode ``latents`` (mode 1) or draw them from the ARM with ``seed`` (mode 2).
        Returns (latents int8 CUDA tensor, payload bytes, slow_path_count)."""
        nn_ints = np.ascontiguousarray(nn_ints, dtype=np.int64)
        n = desc.n_symbols()
        if latents is None:
            assert seed is not None
            lat = torch.zeros((n,), dtype=torch.int8, device=self.torch_device)
            mode = 2
        else:
            lat = latents.to(self.torch_device, torch.int8).contiguous().clone()
            mode, seed = 1, 0
        # a symbol costs at most 24 - log2(1 - 2^-8) < 24.0057 bits (freq >= 1 of 2^24, scale truncation at R >= 2^32);
        # 3 words for the initial state, the seal and rounding
        cap = -(-n * 240057 // 320000) + 3
        words = torch.zeros((cap,), dtype=torch.int32, device=self.torch_device)
        n_words = ctypes.c_int64(0)
        slow = ctypes.c_int32(0)
        _check(self._lib.ccd_encode_latents(self._h, ctypes.byref(desc), nn_ints.ctypes.data_as(ctypes.c_void_p),
                                            mode, ctypes.c_uint64(seed), lat.data_ptr(), words.data_ptr(), cap,
                                            ctypes.byref(n_words), ctypes.byref(slow), self._stream()))
        payload = words[: n_words.value].cpu().numpy().astype("<u4").tobytes()
        return lat, payload, int(slow.value)

    def finish_frame(self, raw: torch.Tensor, bitdepth: int, frame_data_type: str):
        """decode_frame tail: round / (420 average) / clamp / round.  raw: [1, 3, H, W] CUDA."""
        assert raw.is_cuda and raw.dtype == torch.float32 and raw.dim() == 4 and raw.size(1) == 3
        raw = raw.contiguous()
        h, w = raw.shape[-2:]
        code = _frame_type_code(frame_data_type)
        out = self._empty_frame(h, w, frame_data_type)
        planes, _ = _planes(out, frame_data_type)
        u, v = (planes[1].data_ptr(), planes[2].data_ptr()) if code == 1 else (None, None)
        _check(self._lib.ccd_finish_frame(self._h, raw.data_ptr(), h, w, bitdepth, 2 if code == 3 else code,
                                          planes[0].data_ptr(), u, v, self._stream()))
        return out

    def _empty_frame(self, h: int, w: int, frame_data_type: str):
        """FrameData.data of an h x w frame on this device: [1, 3, H, W], or the y / u / v dictionary for yuv420."""
        dev = self.torch_device
        if frame_data_type == "yuv420":
            return {"y": torch.empty((1, 1, h, w), dtype=torch.float32, device=dev),
                    "u": torch.empty((1, 1, h // 2, w // 2), dtype=torch.float32, device=dev),
                    "v": torch.empty((1, 1, h // 2, w // 2), dtype=torch.float32, device=dev)}
        return torch.empty((1, 3, h, w), dtype=torch.float32, device=dev)

    @staticmethod
    def _check_inter_shapes(residue, motion, refs, is_b, frame_data_type):
        """The reference fails with a shape error when the Cool-chic outputs or the references do not fit the
        frame (decode.py:159-189); the kernels read raw pointers, so the same conditions are checked here."""
        if residue.dim() != 4 or motion.dim() != 4 or residue.size(0) != 1 or motion.size(0) != 1:
            raise ValueError(f"residue / motion must be [1, C, H, W], found {tuple(residue.shape)} / {tuple(motion.shape)}")
        h, w = residue.shape[-2:]
        if tuple(motion.shape[-2:]) != (h, w):
            raise ValueError(f"motion is {tuple(motion.shape[-2:])}, residue is {(h, w)}")
        n_ref = 2 if is_b else 1
        if residue.size(1) != 3 + n_ref:
            raise ValueError(f"{'B' if is_b else 'P'}-frame residue needs {3 + n_ref} channels, found {residue.size(1)}")
        if motion.size(1) != 2 * n_ref:
            raise ValueError(f"{'B' if is_b else 'P'}-frame motion needs {2 * n_ref} channels, found {motion.size(1)}")
        if len(refs) < n_ref:
            raise ValueError(f"{'B' if is_b else 'P'} frame with {len(refs)} reference frame(s)")
        for r in refs[:n_ref]:
            if r.frame_data_type != frame_data_type:
                raise ValueError(f"reference is {r.frame_data_type}, frame is {frame_data_type}")
            if frame_data_type == "yuv420":
                shapes = [tuple(r.data[k].shape) for k in ("y", "u", "v")]
                if (h | w) & 1 or shapes != [(1, 1, h, w), (1, 1, h // 2, w // 2), (1, 1, h // 2, w // 2)]:
                    raise ValueError(f"yuv420 reference planes {shapes} do not fit a {h}x{w} frame")
            elif tuple(r.data.shape) != (1, 3, h, w):
                raise ValueError(f"reference is {tuple(r.data.shape)}, frame is {(1, 3, h, w)}")
        return h, w

    def _inter_frame(self, residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow, warp_filter_size):
        """(CcdInterFrame, the tensors it points into, h, w) of a P/B frame; bitdepth None: the pre-rounding frame."""
        h, w = self._check_inter_shapes(residue, motion, refs, is_b, frame_data_type)
        residue, motion = residue.contiguous(), motion.contiguous()
        f = CcdInterFrame(d_residue=residue.data_ptr(), n_res_ch=residue.size(1), d_motion=motion.data_ptr(),
                          n_mot_ch=motion.size(1), frame_data_type=_frame_type_code(frame_data_type),
                          bitdepth=int(bitdepth or 0), h=h, w=w, is_b=int(is_b),
                          warp_filter_size=int(warp_filter_size))
        keep = [residue, motion]
        for dst, r in zip((f.ref0, f.ref1), refs[:2 if is_b else 1]):
            ts, _ = _planes(r.data, frame_data_type)
            keep += ts
            dst[:] = [t.data_ptr() for t in ts]
        f.global_flow[:] = (list(global_flow) + [0, 0, 0, 0])[:4]
        return f, keep, h, w

    def reconstruct_frame(self, residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow, warp_filter_size):
        """Whole P/B reconstruction in one kernel (bitstream/decode.py:156-206): prediction from the finished
        reference frames (4:2:0 planes read in place), blending, residue, frame tail.  Returns the finished frame
        in FrameData layout ([1,3,H,W], or the y / u / v dictionary).  ``bitdepth=None`` stops before the frame tail
        (decode.py:156-189): the PRE-ROUNDING frame [1,3,H,W], from 4:4:4 references."""
        if bitdepth is None and frame_data_type == "yuv420":
            raise ValueError("the pre-rounding frame takes 4:4:4 references; yuv420 frames need a bitdepth")
        f, keep, h, w = self._inter_frame(residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow,
                                          warp_filter_size)
        data = self._empty_frame(h, w, frame_data_type)
        outs, _ = _planes(data, frame_data_type)
        _check(self._lib.ccd_reconstruct_frame(self._h, ctypes.byref(f), (ctypes.c_void_p * 3)(*[t.data_ptr() for t in outs]),
                                               self._stream()))
        del keep
        return data

    def inter_predict(self, residue, motion, refs, is_b, frame_data_type, global_flow, warp_filter_size):
        """decode_frame's P/B branch (bitstream/decode.py:156-189) -> PRE-ROUNDING frame [1,3,H,W] from 4:4:4
        references (stage entry point for tests): reconstruct_frame without the frame tail."""
        return self.reconstruct_frame(residue, motion, refs, is_b, frame_data_type, None, global_flow, warp_filter_size)

    def pack_frame(self, data, bitdepth: int, frame_data_type: str, interleaved: bool = False,
                   sample_bytes: Optional[int] = None) -> torch.Tensor:
        """Finished frame (FrameData.data on the device) -> integer samples on the device, uint8 / uint16:
        planar (y, u, v one after the other: the .yuv file order) or pixel-interleaved HWC (PPM / PNG order)."""
        planes, cs = _planes(data, frame_data_type)
        h, w = planes[0].shape[-2:]
        if sample_bytes is None:
            sample_bytes = 1 if bitdepth <= 8 else 2
        n = h * w + 2 * (h >> cs) * (w >> cs)
        out = torch.empty((n,), dtype=torch.uint8 if sample_bytes == 1 else torch.int16, device=self.torch_device)
        pp = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in planes])
        _check(self._lib.ccd_pack_frame(self._h, pp, h, w, cs, int(bitdepth), sample_bytes, int(bool(interleaved)),
                                        out.data_ptr(), self._stream()))
        return out

    def pack_frames(self, frames, bitdepth: int, frame_data_type: str, sample_bytes: Optional[int] = None) -> torch.Tensor:
        """A batch of finished frames (what decode_many returns with ``finish``) -> the planar integer samples of all
        of them, frame after frame, in ONE device tensor.  Frames that are consecutive slices of one buffer (decode_many
        allocates them so) are converted by a single launch; anything else falls back to one pack_frame per frame."""
        if sample_bytes is None:
            sample_bytes = 1 if bitdepth <= 8 else 2
        dt = torch.uint8 if sample_bytes == 1 else torch.int16

        def first_last(fr):
            if frame_data_type == "yuv420":
                return fr["y"], (fr["y"], fr["u"], fr["v"])
            return fr, (fr,)

        total, base, contiguous = 0, None, len(frames) > 0
        for fr in frames:
            head, parts = first_last(fr)
            for t in parts:
                if base is None:
                    base = t.data_ptr()
                contiguous = contiguous and t.is_contiguous() and t.dtype == torch.float32 and t.data_ptr() == base + 4 * total
                total += t.numel()
        if not contiguous:
            return torch.cat([self.pack_frame(fr, bitdepth, frame_data_type, False, sample_bytes) for fr in frames])
        out = torch.empty((total,), dtype=dt, device=self.torch_device)
        _check(self._lib.ccd_pack_samples(self._h, ctypes.c_void_p(base), total, int(bitdepth), sample_bytes, out.data_ptr(),
                                          self._stream()))
        return out

    def latent_rate(self, descs: Sequence[CcdCoolChicDesc], nn_ints: Sequence[np.ndarray],
                    latents: Sequence[torch.Tensor], want_freq: bool = False, want_mu_sc: bool = False,
                    want_spatial: bool = False, edits=None) -> List[dict]:
        """Rate of decoded latents (``ccd_latent_rate``): one kernel launch for all Cool-chics, plus one for the
        spatial maps.  ``latents[i]``: int8 CUDA tensor in decode order (what ``decode_many(want_latents=True)``
        returns).  Per Cool-chic a dict with ``bits`` (float32 CUDA [n_symbols], decode order), ``grid_bits``
        (list of f64, grid 0 = finest), and on request ``freq`` / ``mu_sc`` (int32 CUDA holding the uint32
        values) and ``spatial`` ([1, 1, H, W] float32 CUDA).  ``want_mu_sc`` may also be one flag per Cool-chic.
        ``edits[i]`` (``ccd_latent_rate_edited``, DESIGN §4.10): a (zero_ctx, zero_ifce_out, zero_ifce_grids) triple of
        ARM inputs read as 0 for Cool-chic i; several edits of one Cool-chic are several jobs on the same latents."""
        n = len(descs)
        jobs = (CcdRateJob * n)()
        mu_sc_flags = [bool(want_mu_sc)] * n if isinstance(want_mu_sc, bool) else [bool(f) for f in want_mu_sc]
        keep, res = [], []
        dev = self.torch_device
        for i in range(n):
            d = descs[i]
            nn = np.ascontiguousarray(nn_ints[i], dtype=np.int64)
            lat = latents[i]
            _check_symbols(f"latents[{i}]", lat, d.n_symbols())
            r = {"bits": torch.empty((d.n_symbols(),), dtype=torch.float32, device=dev)}
            if want_freq:
                r["freq"] = torch.empty((d.n_symbols(),), dtype=torch.int32, device=dev)
            if mu_sc_flags[i]:
                r["mu_sc"] = torch.empty((d.n_symbols(),), dtype=torch.int32, device=dev)
            if want_spatial:
                r["spatial"] = torch.empty((1, 1, d.img_h, d.img_w), dtype=torch.float32, device=dev)
            keep += [nn, lat]
            jobs[i].desc = ctypes.pointer(d)
            jobs[i].nn_ints = nn.ctypes.data
            jobs[i].d_latents = lat.data_ptr()
            jobs[i].d_bits = r["bits"].data_ptr()
            jobs[i].d_freq = r["freq"].data_ptr() if want_freq else None
            jobs[i].d_mu_sc = r["mu_sc"].data_ptr() if mu_sc_flags[i] else None
            jobs[i].d_spatial = r["spatial"].data_ptr() if want_spatial else None
            res.append(r)
        if edits is None:
            _check(self._lib.ccd_latent_rate(self._h, jobs, n, self._stream()), jobs)
        else:
            ed = (CcdModelEdit * n)(*[CcdModelEdit(*(int(v) for v in e)) for e in edits])
            _check(self._lib.ccd_latent_rate_edited(self._h, jobs, ed, n, self._stream()), jobs)
        for i in range(n):
            res[i]["grid_bits"] = [float(jobs[i].grid_bits[g]) for g in range(descs[i].n_grids)]
        return res

    def rate_candidates(self, desc: CcdCoolChicDesc, nn_ints: np.ndarray, latents: torch.Tensor,
                        cands: Sequence[Tuple[int, int]]):
        """Exact per-grid latent bits under the model and under one-integer edits of it (``ccd_rate_candidates``,
        DESIGN §4.11), in one launch.  ``cands``: up to CCD_CAND_MAX (nn_index, delta) pairs, nn_index into the
        ``decode_nn`` order (ARM and IFCE integers only).  Returns (bits float64 [1 + k][n_grids], grid 0 = finest,
        row 0 the model itself; fast bool [1 + k]: the model takes the fast entropy kernel)."""
        nn = np.ascontiguousarray(nn_ints, dtype=np.int64)
        _check_symbols("latents", latents, desc.n_symbols())
        k = len(cands)
        arr = (CcdCandidate * max(k, 1))(*[CcdCandidate(int(i), int(dl)) for i, dl in cands])
        bits = np.zeros((k + 1, desc.n_grids), dtype=np.float64)
        fast = np.zeros(k + 1, dtype=np.int32)
        _check(self._lib.ccd_rate_candidates(self._h, ctypes.byref(desc), nn.ctypes.data_as(ctypes.c_void_p),
                                             latents.data_ptr(), arr, k, bits.ctypes.data_as(ctypes.c_void_p),
                                             fast.ctypes.data_as(ctypes.c_void_p), self._stream()))
        return bits, fast.astype(bool)

    def rate_sweep(self, descs: Sequence[CcdCoolChicDesc], latents: Sequence[torch.Tensor],
                   mu_sc: Sequence[torch.Tensor], sc_offsets: Sequence[int]) -> List[dict]:
        """Scale-calibration sweep and symbol histograms of decoded latents (``ccd_rate_sweep``, DESIGN §4.10): one
        launch for all Cool-chics.  ``latents[i]`` as for latent_rate, ``mu_sc[i]`` the (mu_idx, sc_idx) the coder used
        (latent_rate's ``mu_sc``); ``sc_offsets``: 1 to 32 offsets of sc_idx.  Per Cool-chic a dict with ``bits``
        (per grid, finest first, the f64 bits at each offset) and ``hist`` (int64 [n_grids, 128], count of symbol
        s - 64 in bin s)."""
        n = len(descs)
        jobs = (CcdSweepJob * n)()
        offs = [int(o) for o in sc_offsets]
        if not 1 <= len(offs) <= SWEEP_MAX_OFFSETS:
            raise ValueError(f"{len(offs)} scale offsets, the sweep takes 1 to {SWEEP_MAX_OFFSETS}")
        for i in range(n):
            d, lat, ms = descs[i], latents[i], mu_sc[i]
            for name, t, dt in (("latents", lat, torch.int8), ("mu_sc", ms, torch.int32)):
                _check_symbols(f"{name}[{i}]", t, d.n_symbols(), dt, str(dt))
            jobs[i].desc = ctypes.pointer(d)
            jobs[i].d_latents = lat.data_ptr()
            jobs[i].d_mu_sc = ms.data_ptr()
            jobs[i].n_offsets = len(offs)
            jobs[i].sc_offset[:len(offs)] = offs
        _check(self._lib.ccd_rate_sweep(self._h, jobs, n, self._stream()), jobs)
        return [{"bits": [list(jobs[i].bits[g])[:len(offs)] for g in range(descs[i].n_grids)],
                 "hist": np.array([list(jobs[i].hist[g]) for g in range(descs[i].n_grids)], dtype=np.int64)}
                for i in range(n)]

    def _frame_jobs(self, job_type, frames, sources, layouts):
        """The job array of a call that compares finished frames with their source samples (frame_distortion,
        frame_ssim, frame_vif, frame_hvs), the tensors it points into, and each frame's planes."""
        n = len(frames)
        jobs = (job_type * n)()
        keep, planes = [], []
        for i, (fd, src, lay) in enumerate(zip(frames, sources, layouts)):
            ts, cs = _planes(fd.data, fd.frame_data_type)
            h, w = ts[0].shape[-2:]
            dtype_ok, n = _source_fits(src, h, w, cs, fd.bitdepth)
            if not dtype_ok:
                raise ValueError(f"sources[{i}] must be a contiguous {'uint8' if fd.bitdepth <= 8 else 'int16'} CUDA tensor")
            if src.numel() != n:
                raise ValueError(f"sources[{i}] holds {src.numel()} samples, a {h}x{w} {fd.frame_data_type} frame has {n}")
            keep += [ts, src]
            planes.append(ts)
            for c in range(3):
                jobs[i].d_planes[c] = ts[c].data_ptr()
            jobs[i].d_src = src.data_ptr()
            jobs[i].h, jobs[i].w, jobs[i].chroma_shift, jobs[i].bitdepth = h, w, cs, int(fd.bitdepth)
            jobs[i].src_layout = SOURCE_LAYOUTS[lay]
        return jobs, keep, planes

    def _plane_maps(self, jobs, res, planes, shape):
        """Per frame one float32 CUDA map per plane, of shape(h_c, w_c), in res[i]["maps"] and jobs[i].d_map"""
        for job, r, ts in zip(jobs, res, planes):
            r["maps"] = [torch.empty(shape(*t.shape[-2:]), dtype=torch.float32, device=self.torch_device) for t in ts]
            job.d_map[:] = [m.data_ptr() for m in r["maps"]]

    def frame_distortion(self, frames, sources: Sequence[torch.Tensor], layouts: Sequence[str],
                         want_maps: bool = False) -> List[dict]:
        """Distortion of finished frames against their source samples (``ccd_frame_distortion``), one launch for all.
        ``frames[i]``: a FrameData on this device; ``sources[i]``: its source samples on this device as read from the
        file (uint8, or int16 holding the uint16 samples), in layout ``layouts[i]`` ("planar" or "hwc").  Per frame a
        dict with ``sse`` and ``max_abs`` (three ints, one per plane) and on request ``map`` ([H, W] float32 CUDA,
        fp32(sum_c d_c^2) / fp32(M^2)).  An off-grid decoded sample raises CcdError with ``bad_index`` per frame."""
        n = len(frames)
        jobs, keep, planes = self._frame_jobs(CcdDistJob, frames, sources, layouts)
        res = []
        for i in range(n):
            r = {}
            if want_maps:
                r["map"] = torch.empty(tuple(planes[i][0].shape[-2:]), dtype=torch.float32, device=self.torch_device)
                jobs[i].d_map = r["map"].data_ptr()
            res.append(r)
        _check(self._lib.ccd_frame_distortion(self._h, jobs, n, self._stream()), jobs)
        for i in range(n):
            res[i]["sse"] = [int(jobs[i].sse[c]) for c in range(3)]
            res[i]["max_abs"] = [int(jobs[i].max_abs[c]) for c in range(3)]
        return res

    def frame_ssim(self, frames, sources: Sequence[torch.Tensor], layouts: Sequence[str],
                   want_maps: bool = False) -> List[dict]:
        """MS-SSIM statistics of finished frames against their source samples (``ccd_frame_ssim``), five launches for
        all (one per scale).  Arguments as for frame_distortion; every plane needs both sides >= 176.  Per frame a dict
        with ``cs`` and ``ssim``: per plane, the five per-scale means of cs and of l * cs (f64, the same on every run),
        and on request ``maps``: per plane the scale-0 SSIM map ([h_c - 10, w_c - 10] float32 CUDA)."""
        n = len(frames)
        jobs, keep, planes = self._frame_jobs(CcdSsimJob, frames, sources, layouts)
        res = [{} for _ in range(n)]
        if want_maps:
            self._plane_maps(jobs, res, planes, lambda h, w: (max(h - 10, 0), max(w - 10, 0)))
        _check(self._lib.ccd_frame_ssim(self._h, jobs, n, self._stream()), jobs)
        for i in range(n):
            res[i]["cs"] = [list(jobs[i].cs[c]) for c in range(3)]
            res[i]["ssim"] = [list(jobs[i].ssim[c]) for c in range(3)]
        return res

    def frame_vif(self, frames, sources: Sequence[torch.Tensor], layouts: Sequence[str]) -> List[dict]:
        """VIF statistics of finished frames against their source samples (``ccd_frame_vif``), four launches for all
        (one per scale).  Arguments as for frame_distortion; every plane needs both sides >= 41.  Per frame a dict with
        ``num`` and ``den``: per plane, the four per-scale sums of the VIF numerator and denominator terms (f64, the
        same on every run)."""
        n = len(frames)
        jobs, keep, _ = self._frame_jobs(CcdVifJob, frames, sources, layouts)
        _check(self._lib.ccd_frame_vif(self._h, jobs, n, self._stream()), jobs)
        return [{"num": [list(jobs[i].num[c]) for c in range(3)], "den": [list(jobs[i].den[c]) for c in range(3)]}
                for i in range(n)]

    def frame_hvs(self, frames, sources: Sequence[torch.Tensor], layouts: Sequence[str],
                  want_maps: bool = False) -> List[dict]:
        """PSNR-HVS-M sums of finished frames against their source samples (``ccd_frame_hvs``), one launch for all.
        Arguments as for frame_distortion; every plane needs both sides >= 8.  Per frame a dict with ``s_hvs_m`` and
        ``s_hvs`` (per plane, the sums over its 8 x 8 blocks of the masked and unmasked CSF-weighted squared DCT
        errors, f64, the same on every run), ``n_coeffs`` (per plane, 64 per block) and on request ``maps``: per plane
        each block's S_hvs_m / 64 / 255^2 ([h_c >> 3, w_c >> 3] float32 CUDA)."""
        n = len(frames)
        jobs, keep, planes = self._frame_jobs(CcdHvsJob, frames, sources, layouts)
        res = [{"n_coeffs": [64 * (t.shape[-2] >> 3) * (t.shape[-1] >> 3) for t in planes[i]]} for i in range(n)]
        if want_maps:
            self._plane_maps(jobs, res, planes, lambda h, w: (h >> 3, w >> 3))
        _check(self._lib.ccd_frame_hvs(self._h, jobs, n, self._stream()), jobs)
        for i in range(n):
            res[i]["s_hvs_m"] = list(jobs[i].s_hvs_m)
            res[i]["s_hvs"] = list(jobs[i].s_hvs)
        return res

    @staticmethod
    def _check_inter_source(source, h, w, frame_data_type, bitdepth):
        dtype_ok, n = _source_fits(source, h, w, 1 if frame_data_type == "yuv420" else 0, bitdepth)
        if not (dtype_ok and source.numel() == n):
            raise ValueError(f"source must hold the {h}x{w} {frame_data_type} frame's samples, contiguous on the device")

    def inter_stats(self, residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow, warp_filter_size,
                    source: Optional[torch.Tensor] = None, layout: str = "planar", want_maps: bool = False) -> dict:
        """Statistics of a P/B frame's prediction (``ccd_inter_stats``), from the arguments of reconstruct_frame and
        optionally the frame's source samples (as for frame_distortion).  Returns ``sums``: [sum alpha, sum beta,
        sum (pred - orig)^2, sum (dummy - orig)^2] (f64; the last two 0 without a source) and on request the maps
        ``alpha``, ``beta`` ([H, W]) and ``pred`` ([3, H, W]), float32 CUDA."""
        f, keep, h, w = self._inter_frame(residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow,
                                          warp_filter_size)
        if source is not None:
            self._check_inter_source(source, h, w, frame_data_type, bitdepth)
        dev = self.torch_device
        out = {}
        if want_maps:
            out = {"alpha": torch.empty((h, w), dtype=torch.float32, device=dev),
                   "beta": torch.empty((h, w), dtype=torch.float32, device=dev),
                   "pred": torch.empty((3, h, w), dtype=torch.float32, device=dev)}
        st = CcdInterStats(d_src=source.data_ptr() if source is not None else None, src_layout=SOURCE_LAYOUTS[layout])
        if want_maps:
            st.d_alpha, st.d_beta, st.d_pred = (out[k].data_ptr() for k in ("alpha", "beta", "pred"))
        _check(self._lib.ccd_inter_stats(self._h, ctypes.byref(f), ctypes.byref(st), self._stream()))
        del keep
        out["sums"] = [float(s) for s in st.sums]
        return out

    def inter_analysis(self, residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow, warp_filter_size,
                       source: torch.Tensor, layout: str = "planar", want_maps: bool = False) -> dict:
        """Motion analysis of a P/B frame (``ccd_inter_analysis``, DESIGN §4.9), from the arguments of
        reconstruct_frame and the frame's source samples (as for frame_distortion): one launch.  Returns ``sse``, per
        variant (bitstream/motion.py VARIANTS order) the three per-plane sums of squared integer errors (None for the
        beta variants of a P frame), and per reference ``refs``: a dict with ``sum`` (f64 sums of fx + gx, fy + gy and
        |local|), ``max`` (max |local|) and ``outside`` (pixels sampled outside the reference), and on request
        ``flow`` ([2, H, W] float32 CUDA, the total displacement)."""
        f, keep, h, w = self._inter_frame(residue, motion, refs, is_b, frame_data_type, bitdepth, global_flow,
                                          warp_filter_size)
        self._check_inter_source(source, h, w, frame_data_type, bitdepth)
        n_ref = 2 if is_b else 1
        flows = [torch.empty((2, h, w), dtype=torch.float32, device=self.torch_device) for _ in range(n_ref)] if want_maps else []
        an = CcdInterAnalysis(d_src=source.data_ptr(), src_layout=SOURCE_LAYOUTS[layout])
        an.d_flow[:] = [t.data_ptr() for t in flows] + [None] * (2 - len(flows))
        _check(self._lib.ccd_inter_analysis(self._h, ctypes.byref(f), ctypes.byref(an), self._stream()), [an])
        del keep
        sse = [[int(v) for v in an.sse[k]] for k in range(INTER_VARIANTS)]
        if not is_b:
            sse[3] = sse[4] = None
        out = {"sse": sse, "refs": []}
        for r in range(n_ref):
            ref = {"sum": [float(v) for v in an.flow_sum[r]], "max": float(an.flow_max[r]), "outside": int(an.outside[r])}
            if want_maps:
                ref["flow"] = flows[r]
            out["refs"].append(ref)
        return out

    def last_timing(self):
        ms = (ctypes.c_float * 4)()
        _check(self._lib.ccd_last_timing(self._h, ms))
        return {"entropy_ms": ms[0], "synthesis_ms": ms[1], "upload_ms": ms[2], "upload_bytes": int(ms[3])}

    def launch_count(self) -> int:
        return int(self._lib.ccd_debug_launch_count())

    def set_producer_mask(self, mask: int) -> None:
        """Which of warps 0..13 of an entropy CTA produce windows (ccd_debug_set_producer_mask; default 0x3777)."""
        _check(self._lib.ccd_debug_set_producer_mask(self._h, mask))

    def last_status(self):
        st = (ctypes.c_int32 * 16)()
        _check(self._lib.ccd_debug_last_status(self._h, st))
        return list(st)

    def laplace_domain(self, sc_lo: int, sc_hi: int):
        n = (sc_hi - sc_lo) * 32641
        lo = np.zeros(n, dtype=np.uint32)
        hi = np.zeros(n, dtype=np.uint32)
        _check(self._lib.ccd_debug_laplace_domain(self._h, sc_lo, sc_hi, lo.ctypes.data_as(ctypes.c_void_p),
                                                  hi.ctypes.data_as(ctypes.c_void_p)))
        return lo, hi

    def cdf_table(self, sc_lo: int, sc_hi: int) -> np.ndarray:
        """The context's cumulative table for the scales [sc_lo, sc_hi): uint32 [sc_hi - sc_lo, 256, 32]."""
        out = np.zeros((sc_hi - sc_lo, 256, 32), dtype=np.uint32)
        _check(self._lib.ccd_debug_cdf_table(self._h, sc_lo, sc_hi, out.ctypes.data_as(ctypes.c_void_p)))
        return out

    def detmath(self, fn: str, x: np.ndarray) -> np.ndarray:
        """The device's canonical sin / cos / log (ccd_detmath.h) of every element of x: float64 like x."""
        x = np.ascontiguousarray(x, dtype=np.float64)
        y = np.empty_like(x)
        _check(self._lib.ccd_debug_detmath(self._h, {"sin": 0, "cos": 1, "log": 2}[fn],
                                           x.ctypes.data_as(ctypes.c_void_p), y.ctypes.data_as(ctypes.c_void_p), x.size))
        return y

    def sinc_coeffs(self, taps: int, s: np.ndarray) -> np.ndarray:
        """The taps the sinc warp forms at fractional offsets s: float32 [len(s), taps]."""
        s = np.ascontiguousarray(s, dtype=np.float32)
        c = np.empty((s.size, taps), dtype=np.float32)
        _check(self._lib.ccd_debug_sinc_coeffs(self._h, taps, s.ctypes.data_as(ctypes.c_void_p),
                                               c.ctypes.data_as(ctypes.c_void_p), s.size))
        return c

    def cr_noise(self, first: int, n: int) -> np.ndarray:
        """Samples [first, first + n) of the device's common-randomness generator: float32 [n]."""
        out = np.empty(n, dtype=np.float32)
        _check(self._lib.ccd_debug_cr_noise(self._h, first, n, out.ctypes.data_as(ctypes.c_void_p)))
        return out


def _planes(data, frame_data_type: str):
    """(the three contiguous float32 CUDA planes, chroma shift) of FrameData.data: y, u, v for yuv420 (chroma shift
    1), else the channels of the [1, 3, H, W] tensor."""
    if frame_data_type == "yuv420":
        ts, cs = [data[k].contiguous() for k in ("y", "u", "v")], 1
    else:
        t = data.contiguous()
        ts, cs = [t[0, c] for c in range(3)], 0
    assert all(t.is_cuda and t.dtype == torch.float32 for t in ts)
    return ts, cs


def _frame_type_code(frame_data_type: str) -> int:
    """io/types.py:12 order: rgb, yuv420, yuv444, flow.  'flow' frames take the generic (4:4:4) tail like the
    reference's decode.py:191-206 does."""
    try:
        return {"rgb": 0, "yuv420": 1, "yuv444": 2, "flow": 3}[frame_data_type]
    except KeyError:
        raise ValueError(f"unknown frame_data_type {frame_data_type!r}") from None


_contexts = {}
_contexts_lock = threading.Lock()


def get_context(device: int = 0) -> Context:
    with _contexts_lock:
        if device not in _contexts:
            _contexts[device] = Context(device)
        return _contexts[device]
