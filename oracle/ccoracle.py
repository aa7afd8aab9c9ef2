"""ctypes wrapper of the CPU oracle (oracle/_build/libccoracle.so).

TEST INFRASTRUCTURE ONLY -- may be imported by tests/, __graft_entry__.smoke() and the
cpu_baseline / --impl reference legs of bench.py, never by the product package.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "_build", "libccoracle.so")


def build(force: bool = False) -> str:
    src = [os.path.join(_HERE, f) for f in ("ccoracle.c", "ccoracle.h", "detmath.h", "scale_table.inc")]
    stale = (not os.path.exists(_SO)) or any(os.path.getmtime(s) > os.path.getmtime(_SO) for s in src)
    if force or stale:
        subprocess.check_call(["make", "-C", _HERE, "-s"] + (["-B"] if force else []))
    return _SO


_lib = None


def lib():
    global _lib
    if _lib is None:
        build()
        L = ctypes.CDLL(_SO)
        vp, sz, i64 = ctypes.c_void_p, ctypes.c_size_t, ctypes.c_int64
        L.cco_sizeof_desc.restype = ctypes.c_int
        L.cco_set_threads.restype = ctypes.c_int
        L.cco_set_threads.argtypes = [ctypes.c_int]
        L.cco_nn_counts.restype = i64
        L.cco_nn_counts.argtypes = [vp, vp]
        L.cco_decode_nn.restype = i64
        L.cco_decode_nn.argtypes = [vp, vp, sz, vp, sz]
        L.cco_encode_nn.restype = i64
        L.cco_encode_nn.argtypes = [vp, vp, sz, vp, sz, vp]
        L.cco_latent_layout.restype = i64
        L.cco_latent_layout.argtypes = [vp, vp]
        L.cco_decode_latents.restype = ctypes.c_int
        L.cco_decode_latents.argtypes = [vp, vp, vp, sz, vp, vp]
        L.cco_encode_latents.restype = i64
        L.cco_encode_latents.argtypes = [vp, vp, vp, vp, sz]
        L.cco_sample_latents.restype = i64
        L.cco_sample_latents.argtypes = [vp, vp, ctypes.c_uint64, vp, vp, sz]
        L.cco_synthesize.restype = ctypes.c_int
        L.cco_synthesize.argtypes = [vp, vp, vp, vp, vp]
        L.cco_finish_frame.restype = ctypes.c_int
        L.cco_finish_frame.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp, vp]
        L.cco_inter_predict.restype = ctypes.c_int
        L.cco_inter_predict.argtypes = [vp, vp, vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp,
                                        ctypes.c_int, vp]
        L.cco_laplace_domain.restype = None
        L.cco_laplace_domain.argtypes = [ctypes.c_int, ctypes.c_int, vp, vp]
        L.cco_resize.restype = ctypes.c_int
        L.cco_resize.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp] + [ctypes.c_int] * 4
        L.cco_cr_noise.restype = ctypes.c_int
        L.cco_cr_noise.argtypes = [vp, vp]
        L.cco_noise_samples.restype = ctypes.c_int
        L.cco_noise_samples.argtypes = [ctypes.c_uint64, sz, vp]
        L.cco_detmath.restype = ctypes.c_int
        L.cco_detmath.argtypes = [ctypes.c_int, vp, vp, sz]
        L.cco_sinc_coeffs.restype = ctypes.c_int
        L.cco_sinc_coeffs.argtypes = [ctypes.c_int, vp, vp, sz]
        L.cco_laplace_left.restype = ctypes.c_uint32
        L.cco_laplace_left.argtypes = [ctypes.c_int, ctypes.c_float, ctypes.c_float]
        _lib = L
    return _lib


class OracleError(RuntimeError):
    pass


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _chk(rc, what):
    if rc < 0:
        raise OracleError(f"oracle {what} failed with code {rc}")
    return rc


def nn_counts(desc):
    counts = np.zeros(8, dtype=np.int64)
    total = _chk(lib().cco_nn_counts(ctypes.byref(desc), _p(counts)), "nn_counts")
    return int(total), counts


def decode_nn(desc, nn_bytes: bytes) -> np.ndarray:
    total, _ = nn_counts(desc)
    out = np.zeros(total, dtype=np.int64)
    buf = np.frombuffer(nn_bytes, dtype=np.uint8)
    n = _chk(lib().cco_decode_nn(ctypes.byref(desc), _p(buf), buf.size, _p(out), out.size), "decode_nn")
    assert n == total
    return out


def encode_nn(desc, ints: np.ndarray):
    ints = np.ascontiguousarray(ints, dtype=np.int64)
    out = np.zeros(ints.size * 16 + 16, dtype=np.uint8)
    pad = ctypes.c_int32(0)
    n = _chk(lib().cco_encode_nn(ctypes.byref(desc), _p(ints), ints.size, _p(out), out.size,
                                 ctypes.byref(pad)), "encode_nn")
    return out[:n].tobytes(), int(pad.value)


def latent_layout(desc):
    offs = np.zeros(32, dtype=np.int64)
    total = lib().cco_latent_layout(ctypes.byref(desc), _p(offs))
    return int(total), offs[: desc.n_grids].copy()


def decode_latents(desc, nn: np.ndarray, latent_bytes: bytes):
    total, _ = latent_layout(desc)
    out = np.zeros(total, dtype=np.int8)
    stats = np.zeros(8, dtype=np.int64)
    buf = np.frombuffer(latent_bytes, dtype=np.uint8)
    nn = np.ascontiguousarray(nn, dtype=np.int64)
    _chk(lib().cco_decode_latents(ctypes.byref(desc), _p(nn), _p(buf), buf.size, _p(out), _p(stats)),
         "decode_latents")
    return out, stats


def payload_cap_bytes(n_symbols: int) -> int:
    """Largest payload of n symbols: freq >= 1 of 2^24 and the scale truncation (R >= 2^32) cost at most
    24 - log2(1 - 2^-8) < 24.0057 bits per symbol; 3 words for the initial state, the seal and rounding."""
    return 4 * (-(-n_symbols * 240057 // 320000) + 3)


def encode_latents(desc, nn: np.ndarray, latents: np.ndarray) -> bytes:
    latents = np.ascontiguousarray(latents, dtype=np.int8)
    nn = np.ascontiguousarray(nn, dtype=np.int64)
    out = np.zeros(payload_cap_bytes(latents.size), dtype=np.uint8)
    rc = lib().cco_encode_latents(ctypes.byref(desc), _p(nn), _p(latents), _p(out), out.size)
    if rc == -1:
        bad = np.flatnonzero((latents < -64) | (latents > 63))
        if bad.size:
            raise OracleError(f"oracle encode_latents: latent {int(bad[0])} is outside [-64, 63] (code -1)")
    n = _chk(rc, "encode_latents")
    return out[:n].tobytes()


def sample_latents(desc, nn: np.ndarray, seed: int):
    total, _ = latent_layout(desc)
    lat = np.zeros(total, dtype=np.int8)
    nn = np.ascontiguousarray(nn, dtype=np.int64)
    out = np.zeros(payload_cap_bytes(total), dtype=np.uint8)
    n = _chk(lib().cco_sample_latents(ctypes.byref(desc), _p(nn), ctypes.c_uint64(seed), _p(lat), _p(out),
                                      out.size), "sample_latents")
    return lat, out[:n].tobytes()


def synthesize(desc, nn: np.ndarray, latents: np.ndarray, want_dense: bool = False):
    C = desc.n_out_channels
    out = np.zeros((C, desc.img_h, desc.img_w), dtype=np.float32)
    nn = np.ascontiguousarray(nn, dtype=np.int64)
    latents = np.ascontiguousarray(latents, dtype=np.int8)
    dense = None
    if want_dense:
        h0, w0 = [(h, w) for (h, w), hy in zip(desc.grid_sizes(), list(desc.grid_is_hyper)) if not hy][0]
        dense = np.zeros((desc.syn_in, h0, w0), dtype=np.float32)
    _chk(lib().cco_synthesize(ctypes.byref(desc), _p(nn), _p(latents), _p(out),
                              _p(dense) if dense is not None else None), "synthesize")
    return (out, dense) if want_dense else out


def finish_frame(x: np.ndarray, bitdepth: int, data_type: str):
    x = np.ascontiguousarray(x, dtype=np.float32)
    _, h, w = x.shape
    code = {"rgb": 0, "yuv420": 1, "yuv444": 2}[data_type]
    if code == 1:
        a = np.zeros((h, w), np.float32)
        b = np.zeros((h // 2, w // 2), np.float32)
        c = np.zeros((h // 2, w // 2), np.float32)
        _chk(lib().cco_finish_frame(_p(x), h, w, bitdepth, code, _p(a), _p(b), _p(c)), "finish_frame")
        return {"y": a, "u": b, "v": c}
    a = np.zeros((3, h, w), np.float32)
    _chk(lib().cco_finish_frame(_p(x), h, w, bitdepth, code, _p(a), None, None), "finish_frame")
    return a


def laplace_domain(sc_lo: int, sc_hi: int):
    n = (sc_hi - sc_lo) * 32641
    lo = np.zeros(n, dtype=np.uint32)
    hi = np.zeros(n, dtype=np.uint32)
    lib().cco_laplace_domain(sc_lo, sc_hi, _p(lo), _p(hi))
    return lo, hi


def set_threads(n: int = 0) -> int:
    """Threads used by the float tail (0 = leave as is / all cores); returns the count."""
    return int(lib().cco_set_threads(n))


def inter_predict(residue, motion, ref0, ref1, global_flow, warp_filter_size):
    """decode_frame P/B branch before rounding.  residue [4|5,H,W], motion [2|4,H,W], refs [3,H,W]."""
    residue = np.ascontiguousarray(residue, dtype=np.float32)
    motion = np.ascontiguousarray(motion, dtype=np.float32)
    ref0 = np.ascontiguousarray(ref0, dtype=np.float32)
    is_b = ref1 is not None
    if is_b:
        ref1 = np.ascontiguousarray(ref1, dtype=np.float32)
    _, h, w = ref0.shape
    gf = np.zeros(4, dtype=np.int32)
    gf[: len(global_flow)] = global_flow
    out = np.zeros((3, h, w), dtype=np.float32)
    _chk(lib().cco_inter_predict(_p(residue), _p(motion), _p(ref0), _p(ref1) if is_b else None, h, w, int(is_b),
                                 _p(gf), int(warp_filter_size), _p(out)), "inter_predict")
    return out


def resize(x: np.ndarray, size, mode: str, scale_factor_2: bool = False) -> np.ndarray:
    """F.interpolate(x[None], size | scale_factor=2, mode, align_corners=False)[0] for [C,h,w] fp32."""
    x = np.ascontiguousarray(x, dtype=np.float32)
    c, h, w = x.shape
    H, W = size
    out = np.zeros((c, H, W), dtype=np.float32)
    _chk(lib().cco_resize(_p(x), c, h, w, _p(out), H, W, {"bilinear": 1, "bicubic": 2}[mode], int(scale_factor_2)),
         "resize")
    return out


def cr_noise(desc) -> np.ndarray:
    """Common-randomness channels of the synthesis input: [n_latent_resolutions, img_h, img_w]."""
    n = desc.latent_res_hi - desc.latent_res_lo + 1
    out = np.zeros((n, desc.img_h, desc.img_w), dtype=np.float32)
    _chk(lib().cco_cr_noise(ctypes.byref(desc), _p(out)), "cr_noise")
    return out


DETMATH_FN = {"sin": 0, "cos": 1, "log": 2}


def noise_samples(first: int, n: int) -> np.ndarray:
    """Samples [first, first + n) of the common-randomness generator (noise.py:18-34): float32 [n]."""
    out = np.zeros(n, dtype=np.float32)
    _chk(lib().cco_noise_samples(first, n, _p(out)), "noise_samples")
    return out


def detmath(fn: str, x: np.ndarray) -> np.ndarray:
    """The canonical sin / cos / log of detmath.h, element by element: float64 like x."""
    x = np.ascontiguousarray(x, dtype=np.float64)
    y = np.empty_like(x)
    _chk(lib().cco_detmath(DETMATH_FN[fn], _p(x), _p(y), x.size), "detmath")
    return y


def sinc_coeffs(taps: int, s: np.ndarray) -> np.ndarray:
    """Taps of the windowed-sinc warp at fractional offsets s: float32 [len(s), taps]."""
    s = np.ascontiguousarray(s, dtype=np.float32)
    c = np.empty((s.size, taps), dtype=np.float32)
    _chk(lib().cco_sinc_coeffs(taps, _p(s), _p(c), s.size), "sinc_coeffs")
    return c
