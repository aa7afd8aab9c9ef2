"""``decode_video`` / ``decode_frame``: the drop-in for the reference's
``coolchic/bitstream/decode.py:26-212`` (same names, arguments, return values, printed
per-frame timing line, exceptions) with every per-pixel operation on the GPU.

Differences that do not change results:
  * all Cool-chics of the video are entropy-decoded CONCURRENTLY up front (they are mutually
    independent, SURVEY 8e: only the final warp+blend of P/B frames needs references), then
    frames are reconstructed in coding order;
  * decoded tensors live on the GPU; ``decode_video`` returns them on ``output_device``
    ("cpu" by default, like the reference).
"""
import time
from typing import Dict, List, Optional, Tuple

import torch

from .. import _native
from ..io.framedata import FrameData
from ..io.io import save_frame_data_to_file
from .coolchic import decode_coolchics, encode_decode_coolchic
from .header import CoolChicHeader, FrameHeader, VideoHeader


def _split_coolchic(bitstream_bytes: bytes) -> Tuple[CoolChicHeader, bytes, bytes, bytes]:
    """decode.py:134-143: header, then nn_n_bytes of NN payload, then n_bytes_latent."""
    cc_header = CoolChicHeader()
    rest = cc_header.read_header(bitstream_bytes)
    n_nn = cc_header.get_value("nn_n_bytes")
    n_lat = cc_header.get_value("n_bytes_latent")
    if len(rest) < n_nn + n_lat:
        raise ValueError(f"Bitstream truncated: need {n_nn + n_lat} payload bytes, have {len(rest)}.")
    return cc_header, rest[:n_nn], rest[n_nn:n_nn + n_lat], rest[n_nn + n_lat:]


def _parse_frame(bitstream_bytes: bytes):
    frame_header = FrameHeader()
    rest = frame_header.read_header(bitstream_bytes)
    names = ["residue"] + (["motion"] if frame_header.get_value("frame_type") in ["P", "B"] else [])
    ccs = {}
    for name in names:
        h, nn, lat, rest = _split_coolchic(rest)
        ccs[name] = (h, nn, lat)
    return frame_header, ccs, rest


def _finish_request(frame_header: FrameHeader, ccs):
    """(bitdepth, frame_data_type) for the Cool-chic of an I frame with 3 output channels: libccdec then returns the
    finished frame (decode.py:191-206 applied) instead of the raw output.  None otherwise."""
    if frame_header.get_value("frame_type") != "I":
        return None
    p = ccs["residue"][0].get_coolchic_parameter()
    if int(p.layers_synthesis[-1].split("-")[0]) != 3:
        return None
    return (frame_header.get_value("bitdepth"), frame_header.get_value("frame_data_type"))


def _reconstruct(frame_header: FrameHeader, cc_out: Dict[str, torch.Tensor], reference_frames: List[FrameData],
                 device: int) -> FrameData:
    """decode.py:155-212."""
    ctx = _native.get_context(device)
    frame_type = frame_header.get_value("frame_type")
    bitdepth = frame_header.get_value("bitdepth")
    frame_data_type = frame_header.get_value("frame_data_type")
    if frame_type == "I":
        # finished by libccdec when it has 3 channels (_finish_request): a tensor or, for yuv420, a dictionary
        data = cc_out["residue"]
        if torch.is_tensor(data) and data.size(1) != 3:
            raise ValueError(f"Frame reconstruction expects 3 channels, found {data.size(1)}")
    else:
        # prediction + blending + residue + frame tail: one kernel, 4:2:0 references read in place
        refs = [r.to(ctx.torch_device) for r in reference_frames]
        data = ctx.reconstruct_frame(
            cc_out["residue"], cc_out["motion"], refs, frame_type == "B", frame_data_type, bitdepth,
            frame_header.get_value("global_flow"), frame_header.get_value("warp_filter_size"),
        )
    return FrameData(bitdepth=bitdepth, frame_data_type=frame_data_type, data=data)


@torch.no_grad()
def decode_frame(bitstream_bytes: bytes, reference_frames: List[FrameData], verbosity: int = 0,
                 device: int = 0) -> Tuple[FrameData, bytes]:
    """Decode the frame at the start of ``bitstream_bytes``; return it and the remaining bytes."""
    frame_header, ccs, rest = _parse_frame(bitstream_bytes)
    if verbosity:
        print(frame_header.pretty_string())
    names = list(ccs)
    fin = _finish_request(frame_header, ccs)
    outs = decode_coolchics([ccs[n][0] for n in names], [ccs[n][1] for n in names], [ccs[n][2] for n in names],
                            device=device, finish=[fin if n == "residue" else None for n in names])
    if verbosity:
        for n in names:
            print(ccs[n][0].pretty_string())
    frame = _reconstruct(frame_header, dict(zip(names, outs)), reference_frames, device)
    return frame, rest


def output_shape(header: CoolChicHeader) -> Tuple[int, int, int, int]:
    """Shape of a Cool-chic's raw output [1, C, H, W] from its header alone (what the ranks that did not
    decode it allocate before the broadcast)."""
    p = header.get_coolchic_parameter()
    c = int(p.layers_synthesis[-1].split("-")[0])
    return (1, c, int(p.img_size[0]), int(p.img_size[1]))


def _decode_all_coolchics(parsed, device: int, decode_fn=None, frames_mine=None) -> List[Dict[str, torch.Tensor]]:
    """Pass 1 of decode_video: the Cool-chics of the frames in ``frames_mine`` (all frames by default), one
    concurrent batch (one persistent CTA per stream).  Under torch.distributed a rank only decodes the Cool-chics
    of the frames it OWNS (see decode_video_bytes)."""
    decode_fn = decode_fn or decode_coolchics
    if frames_mine is None:
        frames_mine = range(len(parsed))
    flat = [(i, name) for i in frames_mine for name in parsed[i][1]]
    cc_out: List[Dict[str, torch.Tensor]] = [dict() for _ in parsed]
    if not flat:
        return cc_out
    fins = [_finish_request(parsed[i][0], parsed[i][1]) if n == "residue" else None for i, n in flat]
    outs = decode_fn([parsed[i][1][n][0] for i, n in flat], [parsed[i][1][n][1] for i, n in flat],
                     [parsed[i][1][n][2] for i, n in flat], device=device, finish=fins)
    for (i, name), o in zip(flat, outs):
        cc_out[i][name] = o
    return cc_out


def _frame_planes(fd: FrameData) -> List[torch.Tensor]:
    return [fd.data[k] for k in ("y", "u", "v")] if fd.frame_data_type == "yuv420" else [fd.data]


def _empty_like_frame(frame_header: FrameHeader, img_size, dev) -> FrameData:
    """Receive buffer for a frame reconstructed by another rank (same layout as the owner's FrameData)."""
    h, w = img_size
    fmt, b = frame_header.get_value("frame_data_type"), frame_header.get_value("bitdepth")
    if fmt == "yuv420":
        data = {"y": torch.empty((1, 1, h, w), dtype=torch.float32, device=dev),
                "u": torch.empty((1, 1, h // 2, w // 2), dtype=torch.float32, device=dev),
                "v": torch.empty((1, 1, h // 2, w // 2), dtype=torch.float32, device=dev)}
    else:
        data = torch.empty((1, 3, h, w), dtype=torch.float32, device=dev)
    return FrameData(bitdepth=b, frame_data_type=fmt, data=data)


@torch.no_grad()
def decode_video_bytes(bitstream_bytes: bytes, decoded_path: Optional[str] = None, max_decoding_order: int = -1,
                       verbosity: int = 0, device: int = 0, output_device: str = "cpu", decode_fn=None,
                       reconstruct_fn=None) -> Dict[str, FrameData]:
    """decode_video on bytes already in memory.  With an initialised torch.distributed process group every
    rank must call it with the same bytes (see dist.broadcast_byte_strings): the frames are dealt to the ranks
    (frame ownership), reconstructed frames are exchanged, every rank returns all frames.  ``decode_fn`` /
    ``reconstruct_fn`` exist for the CPU (gloo) test of the plumbing."""
    reconstruct_fn = reconstruct_fn or _reconstruct
    bitstream_bytes = memoryview(bitstream_bytes)  # every "remaining bytes" below is a view, not a copy
    video_header = VideoHeader()
    bitstream_bytes = video_header.read_header(bitstream_bytes)
    coding_structure = video_header.get_coding_structure()
    if verbosity:
        print(video_header.pretty_string())
        print(coding_structure.pretty_structure_diagram())
    if max_decoding_order == -1:
        max_decoding_order = coding_structure.get_max_coding_order()

    # ---- pass 1: parse every frame, decode the Cool-chics concurrently on the device(s).
    # Multi-GPU (SURVEY 8e, BASELINE configs[4]): FRAME OWNERSHIP -- frame i (coding order) belongs to rank
    # i mod world; a rank entropy-decodes and synthesises only the Cool-chics of its own frames (they need no
    # reference), reconstructs its frames when their references have arrived, and broadcasts each RECONSTRUCTED
    # frame (the only exchange of the path: one NCCL broadcast per plane, 12.4 MB for a 1080p 4:2:0 frame).
    import torch.distributed as dist

    world = dist.get_world_size() if dist.is_available() and dist.is_initialized() else 1
    rank = dist.get_rank() if world > 1 else 0
    t0 = time.time()
    parsed = []
    for coding_idx in range(max_decoding_order + 1):
        frame_header, ccs, bitstream_bytes = _parse_frame(bitstream_bytes)
        parsed.append((frame_header, ccs))
    owner = [i % world for i in range(len(parsed))]
    mine = [i for i in range(len(parsed)) if owner[i] == rank]
    err = None
    try:
        cc_out = _decode_all_coolchics(parsed, device, decode_fn, frames_mine=mine if world > 1 else None)
    except Exception as e:  # noqa: BLE001 -- re-raised on EVERY rank below: nobody is left waiting in a broadcast
        err, cc_out = e, None
    if world > 1:
        dev0 = torch.device("cuda", device) if torch.cuda.is_available() and dist.get_backend() == "nccl" else torch.device("cpu")
        flag = torch.tensor([1 if err is not None else 0], dtype=torch.int32, device=dev0)
        dist.all_reduce(flag, op=dist.ReduceOp.MAX)
        if int(flag.item()) != 0:
            raise err if err is not None else RuntimeError("decode_video: a Cool-chic failed to decode on another rank")
    elif err is not None:
        raise err
    t_cc = (time.time() - t0) / max(1, len(parsed))

    # ---- pass 2: reconstruct in coding order (references looked up by display index)
    for coding_idx, (frame_header, ccs) in enumerate(parsed):
        start_time = time.time()
        frame = coding_structure.get_frame_from_coding_order(coding_idx)
        if verbosity:
            print(frame_header.pretty_string())
            for n in ccs:
                print(ccs[n][0].pretty_string())
        if owner[coding_idx] == rank:
            refs_data = [coding_structure.get_frame_from_display_order(idx_ref).data for idx_ref in frame.index_references]
            fd = reconstruct_fn(frame_header, cc_out[coding_idx], refs_data, device)
            cc_out[coding_idx] = None
        else:
            p = ccs["residue"][0].get_coolchic_parameter()
            any_local = next((f for f in (coding_structure.get_frame_from_coding_order(k) for k in range(coding_idx))
                              if f.data is not None), None)
            dev = _frame_planes(any_local.data)[0].device if any_local is not None else (
                torch.device("cuda", device) if torch.cuda.is_available() else torch.device("cpu"))
            fd = _empty_like_frame(frame_header, (int(p.img_size[0]), int(p.img_size[1])), dev)
        if world > 1:
            if reconstruct_fn is _reconstruct:
                for t in _frame_planes(fd):
                    dist.broadcast(t, src=owner[coding_idx])
            else:  # stand-in reconstruct functions of the CPU test: ship whatever they return
                box = [fd if owner[coding_idx] == rank else None]
                dist.broadcast_object_list(box, src=owner[coding_idx])
                fd = box[0]
        frame.set_frame_data(fd)
        if torch.cuda.is_available():
            torch.cuda.synchronize(device)
        print(f"Decoding frame {frame.display_order:<4} time = {time.time() - start_time + t_cc:6.2f} seconds.")

    all_frames = {}
    for display_idx in range(coding_structure.get_max_display_order() + 1):
        frame = coding_structure.get_frame_from_display_order(display_idx)
        if frame is None or frame.data is None:
            continue
        fd = frame.data
        on_gpu = (fd.data["y"] if fd.frame_data_type == "yuv420" else fd.data).is_cuda
        if on_gpu and output_device != "cuda":
            # device -> host as PACKED integer samples (1 or 2 bytes each instead of 4): the writers take them as they
            # are, the float container of the API is rebuilt on the host (k / (2^b - 1) in fp32: the same values)
            data = _to_host_packed(fd, device, decoded_path, append=display_idx != 0)
        else:
            data = fd if output_device == "cuda" else fd.to(output_device)
            if decoded_path is not None:
                save_frame_data_to_file(data, decoded_path, append=display_idx != 0)
        all_frames[str(display_idx)] = data
    return all_frames


def _to_host_packed(fd: FrameData, device: int, decoded_path: Optional[str], append: bool) -> FrameData:
    import os

    import numpy as np

    from ..io.io import POSSIBLE_EXT, write_packed_ppm, write_packed_png, write_packed_yuv

    ctx = _native.get_context(device)
    b, fmt = fd.bitdepth, fd.frame_data_type
    planar = ctx.pack_frame(fd.data, b, fmt).cpu().numpy()
    planar = planar.view(np.uint8 if b <= 8 else np.uint16)
    M = float(2**b - 1)
    if fmt == "yuv420":
        h, w = fd.data["y"].shape[-2:]
        n0, n1 = h * w, (h // 2) * (w // 2)
        parts = {"y": planar[:n0].reshape(1, 1, h, w), "u": planar[n0:n0 + n1].reshape(1, 1, h // 2, w // 2),
                 "v": planar[n0 + n1:].reshape(1, 1, h // 2, w // 2)}
        data = {k: torch.from_numpy(v.astype(np.float32)) / M for k, v in parts.items()}
    else:
        h, w = fd.data.shape[-2:]
        data = torch.from_numpy(planar.reshape(1, 3, h, w).astype(np.float32)) / M
    host = FrameData(bitdepth=b, frame_data_type=fmt, data=data)
    if decoded_path is not None:
        ext = os.path.splitext(decoded_path)[1]
        assert ext in POSSIBLE_EXT, (
            f"The function save_frame_data_to_file() expects a file ending with {POSSIBLE_EXT}. Found {decoded_path}"
        )
        if ext == ".yuv":
            write_packed_yuv(planar, b, fmt, decoded_path, append)
        else:
            assert fmt == "rgb", (
                "The function save_frame_data_to_file() can only save a RGB data "
                f"into a {ext[1:].upper()} file. Found frame_data_type = {fmt}."
            )
            hwc = ctx.pack_frame(fd.data, b, fmt, interleaved=True).cpu().numpy().view(np.uint8 if b <= 8 else np.uint16)
            if ext == ".png":
                assert b == 8, (
                    "The function save_frame_data_to_file() can only write 8-bit data "
                    f"into a PNG file. Found bitdepth = {b}."
                )
                write_packed_png(hwc.reshape(h, w, 3), decoded_path)
            else:
                write_packed_ppm(hwc.reshape(h, w, 3), b, decoded_path)
    return host


def decode_video(bitstream_path: str, decoded_path: Optional[str] = None, max_decoding_order: int = -1,
                 verbosity: int = 0, device: int = 0, output_device: str = "cpu") -> Dict[str, FrameData]:
    """Decode an image or video bitstream; optionally save the frames (PNG / PPM / YUV by
    extension).  Returns ``{str(display_index): FrameData}``."""
    with open(bitstream_path, "rb") as f_in:
        bitstream_bytes = f_in.read()
    return decode_video_bytes(bitstream_bytes, decoded_path, max_decoding_order, verbosity, device, output_device)
