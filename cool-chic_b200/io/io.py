"""Frame writers: PNG (8-bit rgb), PPM (rgb), planar YUV (420 / 444, appended per frame); readers of source frames
(``read_samples``, ``load_frame_data_from_file``: io/io.py:19-50, io/format/{yuv,png,ppm}.py of the reference).

Mirror of the reference's ``coolchic/io/io.py:53-105`` (dispatch on the file extension, same
assertions), ``io/format/png.py:44-62``, ``io/format/ppm.py:160-203`` and
``io/format/yuv.py:124-165``.  Samples are ``round(x * (2^b - 1))``; the YUV writer uses
uint16 only when bitdepth == 10 (yuv.py:157, kept as is), PPM stores 2-byte samples MSB first.
"""
import math
import os
from typing import NamedTuple, Tuple

import numpy as np
import torch

from .framedata import FrameData

POSSIBLE_EXT = [".yuv", ".png", ".ppm"]


def _levels(t: torch.Tensor, bitdepth: int) -> np.ndarray:
    return torch.round(t.detach().float().cpu() * (2**bitdepth - 1)).numpy()


def write_png(data: torch.Tensor, file_path: str) -> None:
    from PIL import Image

    arr = data.detach().float().cpu().numpy()
    assert arr.ndim == 4 and arr.shape[0] == 1 and arr.shape[1] == 3, (
        f"Data shape must be [1, 3, H, W], found {arr.shape}"
    )
    arr = np.round(np.clip(arr[0].transpose(1, 2, 0), 0.0, 1.0) * 255).astype(np.uint8)
    Image.fromarray(arr, mode="RGB").save(file_path)


def write_ppm(data: torch.Tensor, bitdepth: int, file_path: str, norm: bool = True) -> None:
    c, h, w = data.size()[-3:]
    t = data.detach().float().cpu().reshape(c, h, w)
    max_val = 2**bitdepth - 1
    vals = torch.round(t * max_val) if norm else t
    hwc = vals.permute(1, 2, 0).contiguous().numpy()
    body = hwc.astype(np.uint8 if max_val <= 255 else ">u2").tobytes()
    with open(file_path, "wb") as f_out:
        f_out.write(f"P6\n{w} {h}\n{max_val}\n".encode("ascii"))
        f_out.write(body)


def write_yuv(data, bitdepth: int, frame_data_type: str, file_path: str, norm: bool = True,
              append: bool = False) -> None:
    assert frame_data_type in ["yuv420", "yuv444"], (
        f"Found incorrect datatype in write_yuv() function: {frame_data_type}. "
        'Data type should be "yuv420" or "yuv444".'
    )
    if frame_data_type == "yuv420":
        raw = torch.cat([data[k].detach().float().cpu().flatten() for k in ("y", "u", "v")])
    else:
        raw = data.detach().float().cpu().flatten()
    if norm:
        raw = raw * (2**bitdepth - 1)
    dtype = np.uint16 if bitdepth == 10 else np.uint8
    out = torch.round(raw).numpy().astype(np.int64).astype(dtype)
    with open(file_path, "ab" if append else "wb") as f_out:
        out.tofile(f_out)


# ---- writers of samples already packed on the device (ccd_pack_frame): no arithmetic left on the host ----------
def write_packed_yuv(planar: np.ndarray, bitdepth: int, frame_data_type: str, file_path: str, append: bool) -> None:
    assert frame_data_type in ["yuv420", "yuv444"], (
        f"Found incorrect datatype in write_yuv() function: {frame_data_type}. "
        'Data type should be "yuv420" or "yuv444".'
    )
    # io/format/yuv.py:157: 2-byte samples only when bitdepth == 10, 1-byte otherwise (kept as is)
    dtype = np.uint16 if bitdepth == 10 else np.uint8
    out = planar if planar.dtype == dtype else planar.astype(np.int64).astype(dtype)
    with open(file_path, "ab" if append else "wb") as f_out:
        out.tofile(f_out)


def write_packed_ppm(hwc: np.ndarray, bitdepth: int, file_path: str) -> None:
    h, w = hwc.shape[:2]
    max_val = 2**bitdepth - 1
    body = hwc.astype(np.uint8 if max_val <= 255 else ">u2").tobytes()
    with open(file_path, "wb") as f_out:
        f_out.write(f"P6\n{w} {h}\n{max_val}\n".encode("ascii"))
        f_out.write(body)


def write_packed_png(hwc_u8: np.ndarray, file_path: str) -> None:
    from PIL import Image

    Image.fromarray(np.ascontiguousarray(hwc_u8), mode="RGB").save(file_path)


# ---- readers: the integer samples of a source frame, as stored in the file ---------------------------------------
class SourceSamples(NamedTuple):
    samples: np.ndarray       # uint8, or native-endian uint16, in file order (flat planar, or [H, W, 3])
    layout: str               # "planar" (YUV) or "hwc" (PNG / PPM)
    img_size: Tuple[int, int]
    bitdepth: int
    frame_data_type: str


def _read_yuv_samples(file_path: str, idx: int) -> SourceSamples:
    """io/format/yuv.py:41-120 and its naming rules (io/io.py:36-40 of the reference)."""
    base = os.path.basename(file_path).split(".")[0]
    try:
        w, h = [int(s) for s in base.split("_")[1].split("x")]
    except (IndexError, ValueError):
        raise ValueError(f"{file_path}: the second '_' field of a .yuv name must be <width>x<height>") from None
    if w < 1 or h < 1:
        raise ValueError(f"{file_path}: bad frame size {w}x{h}")
    bitdepth = 8 if "_8b" in file_path else 10
    fmt = "yuv444" if "444" in file_path else "yuv420"
    h_uv, w_uv = (h // 2, w // 2) if fmt == "yuv420" else (h, w)
    n = h * w + 2 * h_uv * w_uv
    sample_bytes = 1 if bitdepth <= 8 else 2
    size = os.path.getsize(file_path)
    if (idx + 1) * n * sample_bytes > size:
        raise ValueError(f"{file_path}: frame {idx} is past the end of the file ({size // (n * sample_bytes)} frames "
                         f"of {w}x{h} {fmt} {bitdepth}-bit)")
    dt = np.uint8 if sample_bytes == 1 else np.dtype("<u2")
    samples = np.fromfile(file_path, dtype=dt, count=n, offset=idx * n * sample_bytes).astype(
        np.uint8 if sample_bytes == 1 else np.uint16)
    return SourceSamples(samples, "planar", (h, w), bitdepth, fmt)


def _read_png_samples(file_path: str) -> SourceSamples:
    """io/format/png.py:23-41: 8-bit RGB, alpha dropped; other modes are refused."""
    from PIL import Image

    try:
        img = Image.open(file_path)
        img.load()
    except Exception as e:  # noqa: BLE001 -- PIL raises many types for a broken file
        raise ValueError(f"{file_path}: not a readable PNG ({e})") from None
    if img.mode not in ("RGB", "RGBA"):
        raise ValueError(f"{file_path}: PNG mode {img.mode!r}, only 8-bit RGB and RGBA are read")
    hwc = np.ascontiguousarray(np.asarray(img, dtype=np.uint8)[:, :, :3])
    return SourceSamples(hwc, "hwc", hwc.shape[:2], 8, "rgb")


def _read_ppm_samples(file_path: str) -> SourceSamples:
    """io/format/ppm.py:95-157: P6, each header field followed by one whitespace byte, bitdepth = log2(maxval + 1),
    2-byte samples MSB first."""
    with open(file_path, "rb") as f:
        data = f.read()
    blanks = b" \t\n\v\f\r"
    if data[:2] != b"P6":
        raise ValueError(f"{file_path}: a PPM file starts with P6, found {data[:2]!r}")
    pos, fields = 2, []
    for _ in range(3):
        if pos >= len(data) or data[pos] not in blanks:
            raise ValueError(f"{file_path}: malformed PPM header")
        pos += 1
        end = pos
        while end < len(data) and data[end] not in blanks:
            end += 1
        try:
            fields.append(int(data[pos:end].decode("ascii")))
        except ValueError:
            raise ValueError(f"{file_path}: malformed PPM header field {data[pos:end][:16]!r}") from None
        pos = end
    if pos >= len(data):
        raise ValueError(f"{file_path}: PPM header without data")
    pos += 1
    w, h, max_val = fields
    bitdepth = int(math.log2(max_val + 1)) if max_val > 0 else 0
    if w < 1 or h < 1 or not 1 <= bitdepth <= 16 or max_val != 2**bitdepth - 1:
        raise ValueError(f"{file_path}: PPM size {w}x{h} / maxval {max_val} not supported (maxval must be 2^b - 1)")
    dt = np.dtype(np.uint8 if max_val <= 255 else ">u2")
    n = 3 * w * h
    if len(data) - pos < n * dt.itemsize:
        raise ValueError(f"{file_path}: PPM data holds {len(data) - pos} bytes, a {w}x{h} image needs more")
    samples = np.frombuffer(data, dtype=dt, count=n, offset=pos)
    samples = samples.astype(np.uint16) if max_val > 255 else samples.copy()
    return SourceSamples(samples.reshape(h, w, 3), "hwc", (h, w), bitdepth, "rgb")


def read_samples(file_path: str, idx_display_order: int) -> SourceSamples:
    """The integer samples of frame ``idx_display_order`` of a source file (.yuv, .png, .ppm), as stored in the file,
    with their layout, size, bitdepth and frame_data_type.  PNG and PPM files hold one frame.  Raises ValueError for a
    missing file, a frame past the end of the file or a malformed header."""
    ext = os.path.splitext(file_path)[1]
    if ext not in POSSIBLE_EXT:
        raise ValueError(f"read_samples() expects a file ending with {POSSIBLE_EXT}. Found {file_path}")
    if not os.path.isfile(file_path):
        raise ValueError(f"No file found at {file_path}")
    if idx_display_order < 0:
        raise ValueError(f"bad frame index {idx_display_order}")
    if ext == ".yuv":
        return _read_yuv_samples(file_path, idx_display_order)
    if idx_display_order != 0:
        raise ValueError(f"{file_path}: frame {idx_display_order} is past the end of the file (one frame)")
    return _read_png_samples(file_path) if ext == ".png" else _read_ppm_samples(file_path)


def samples_to_frame_data(s: SourceSamples) -> FrameData:
    """Float frame of read_samples' output: fp32(k) / fp32(2^b - 1), the reference readers' values bit for bit."""
    h, w = s.img_size
    t = torch.from_numpy(s.samples.astype(np.float32)) / np.float32(2**s.bitdepth - 1)
    if s.layout == "hwc":
        data = t.permute(2, 0, 1).contiguous().view(1, 3, h, w)
    elif s.frame_data_type == "yuv420":
        n0, n1 = h * w, (h // 2) * (w // 2)
        data = {"y": t[:n0].view(1, 1, h, w), "u": t[n0:n0 + n1].view(1, 1, h // 2, w // 2),
                "v": t[n0 + n1:].view(1, 1, h // 2, w // 2)}
    else:
        data = t.view(1, 3, h, w)
    return FrameData(s.bitdepth, s.frame_data_type, data)


def load_frame_data_from_file(file_path: str, idx_display_order: int) -> FrameData:
    """io/io.py:19-50 of the reference: the frame as a FrameData with values in [0, 1]."""
    return samples_to_frame_data(read_samples(file_path, idx_display_order))


def save_frame_data_to_file(frame_data: FrameData, file_path: str, append: bool = False) -> None:
    ext = os.path.splitext(file_path)[1]
    assert ext in POSSIBLE_EXT, (
        f"The function save_frame_data_to_file() expects a file ending with {POSSIBLE_EXT}. Found {file_path}"
    )
    if ext == ".png":
        assert frame_data.frame_data_type == "rgb", (
            "The function save_frame_data_to_file() can only save a RGB data "
            f"into a PNG file. Found frame_data_type = {frame_data.frame_data_type}."
        )
        assert frame_data.bitdepth == 8, (
            "The function save_frame_data_to_file() can only write 8-bit data "
            f"into a PNG file. Found bitdepth = {frame_data.bitdepth}."
        )
        write_png(frame_data.data, file_path)
    elif ext == ".ppm":
        assert frame_data.frame_data_type == "rgb", (
            "The function save_frame_data_to_file() can only save a RGB data "
            f"into a PPM file. Found frame_data_type = {frame_data.frame_data_type}."
        )
        write_ppm(frame_data.data, frame_data.bitdepth, file_path, norm=True)
    else:
        assert frame_data.frame_data_type in ["yuv420", "yuv444"], (
            "The function save_frame_data_to_file() can only save a YUV data "
            f"into a YUV file. Found frame_data_type = {frame_data.frame_data_type}."
        )
        write_yuv(frame_data.data, frame_data.bitdepth, frame_data.frame_data_type, file_path,
                  norm=True, append=append)
