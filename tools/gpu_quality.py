"""Development tool: time the quality kernels (k_frame_dist, k_frame_ssim, k_inter_stats) with CUDA events, median of
--steps calls.

Workloads:
  * k_frame_dist and k_frame_ssim on the 32 decoded frames of bench.py's gop32_1080p_yuv420 stream (8-bit planar sources);
  * k_frame_dist and k_frame_ssim on 1176 Kodak-size (768x512) rgb frames in one call (8-bit HWC sources);
  * k_inter_stats on one 1080p B frame of that stream, with its source.
Reports, per workload, the whole call (CUDA events around the C-ABI call: staging, kernel, result copy), the kernel
alone (torch.profiler; for MS-SSIM the sum of its five launches), the bytes the kernel must move and that over kernel
time against the H100 SXM's 3.35 TB/s, with the card's name, power limit and max SM clock read in the same run.  For
MS-SSIM also the f64 FLOPs the algorithm needs over kernel time against the card's FP64 rate at its max SM clock
(64 FP64 FMA per SM per cycle on an H100).

    python tools/gpu_quality.py [--steps 20]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import coolchic_b200  # noqa: E402,F401
from coolchic_b200 import _native, synth  # noqa: E402
from coolchic_b200.bitstream import decode  # noqa: E402
from coolchic_b200.io.framedata import FrameData  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                                        "-i", str(torch.cuda.current_device())], text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def ssim_work(shapes):
    """(bytes, f64 FLOPs) the MS-SSIM of planes of the given (h, w) shapes needs.  Bytes: scale 0 reads 4 (fp32
    decoded) + 1 (8-bit source) bytes per sample, every scale below reads 8 bytes per level sample (the two uint32
    sums), and every scale but the last writes the next level.  FLOPs: per scale, 3 products per sample, 5 moments x
    11 taps of FMA (2 FLOPs) per horizontal output (h x (w - 10)) and per vertical output ((h - 10) x (w - 10)), and
    20 for the per-pixel epilogue (a division counted as one)."""
    n_bytes = flops = 0
    for h, w in shapes:
        for j in range(5):
            hj, wj = h >> j, w >> j
            n_bytes += hj * wj * (5 if j == 0 else 8) + (8 * (hj >> 1) * (wj >> 1) if j < 4 else 0)
            flops += 3 * hj * wj + 110 * hj * (wj - 10) + (110 + 20) * (hj - 10) * (wj - 10)
    return n_bytes, flops


def fp64_flops_per_s(card_csv):
    """The card's FP64 FMA rate at its max SM clock (nvidia-smi's clocks.max.sm), 2 FLOPs per FMA."""
    mhz = float(card_csv.split(",")[-1].strip().split()[0])
    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count * 64 * 2 * mhz * 1e6


def measure(fn, kernel, steps, n_bytes, flops=None, fp64=None):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    call = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        call.append(a.elapsed_time(b))
    kern = []
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    for ev in prof.events():
        if kernel in ev.name:
            kern.append(ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3)
    per_call = len(kern) // steps if kern else 1  # MS-SSIM: five launches per call, summed in launch order
    kern = [sum(kern[i:i + per_call]) for i in range(0, len(kern), per_call)]
    k_ms = float(np.median(kern)) if kern else float("nan")
    out = {"call_ms_median": float(np.median(call)), "kernel_ms_median": k_ms, "kernel_bytes": int(n_bytes),
           "kernel_TB_per_s": n_bytes / (k_ms * 1e-3) / 1e12, "share_of_3.35TB_per_s": n_bytes / (k_ms * 1e-3) / HBM_BYTES_PER_S}
    if flops is not None:
        out.update({"kernel_f64_flops": int(flops), "kernel_f64_TFLOP_per_s": flops / (k_ms * 1e-3) / 1e12,
                    "share_of_fp64_rate": flops / (k_ms * 1e-3) / fp64, "fp64_TFLOP_per_s_at_max_clock": fp64 / 1e12})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    ctx = _native.get_context(0)
    out = {"card": card()}
    fp64 = fp64_flops_per_s(out["card"])

    # bench.py's gop32_1080p_yuv420 stream; the first B frame's raw outputs and references are kept for k_inter_stats
    ss = synth.SeedStream(ctx)
    data = synth.make_video_stream(ctx, ss, 1080, 1920, 32, "yuv420", 8, 8, seed=0)
    kept = {}

    def recon(fh, cc_out, refs, dev):
        if fh.get_value("frame_type") == "B" and not kept:
            kept.update(fh=fh, cc=dict(cc_out), refs=[r.to(ctx.torch_device) for r in refs])
        return decode._reconstruct(fh, cc_out, refs, dev)

    frames = decode.decode_video_bytes(data, output_device="cuda", reconstruct_fn=recon)
    frames = [frames[str(i)] for i in range(len(frames))]
    srcs = [ctx.pack_frame(f.data, 8, "yuv420") for f in frames]  # the decoded frames as 8-bit planar sources
    n_samples = sum(s.numel() for s in srcs)
    out["gop32_1080p_yuv420"] = measure(lambda: ctx.frame_distortion(frames, srcs, ["planar"] * len(frames)),
                                        "k_frame_dist", args.steps, 5 * n_samples)
    shapes = [(1080, 1920), (540, 960), (540, 960)] * len(frames)
    out["ssim_gop32_1080p_yuv420"] = measure(lambda: ctx.frame_ssim(frames, srcs, ["planar"] * len(frames)),
                                             "k_frame_ssim", args.steps, *ssim_work(shapes), fp64)

    fh, cc, refs = kept["fh"], kept["cc"], kept["refs"]
    src = srcs[0]  # any 1080p 4:2:0 source: the timing does not depend on the values
    h, w = 1080, 1920
    # residue 5 + motion 4 planes (fp32), two 4:2:0 references (fp32, each sample read at least once), the source
    inter_bytes = 4 * 9 * h * w + 2 * 4 * (3 * h * w // 2) + 3 * h * w // 2
    out["inter_stats_1080p_B"] = measure(
        lambda: ctx.inter_stats(cc["residue"], cc["motion"], refs, True, "yuv420", 8, fh.get_value("global_flow"),
                                fh.get_value("warp_filter_size"), source=src, layout="planar"),
        "k_inter_stats", args.steps, inter_bytes)
    del frames, srcs, cc, refs, kept
    torch.cuda.empty_cache()

    n, h, w = 1176, 512, 768
    g = torch.Generator(device=ctx.torch_device).manual_seed(0)
    kframes, ksrcs = [], []
    for _ in range(n):
        k = torch.randint(0, 256, (3, h, w), generator=g, device=ctx.torch_device, dtype=torch.int32)
        kframes.append(FrameData(8, "rgb", (k.float() / 255).view(1, 3, h, w)))
        ksrcs.append(k.permute(1, 2, 0).reshape(-1).to(torch.uint8))
    out["kodak_x1176_rgb"] = measure(lambda: ctx.frame_distortion(kframes, ksrcs, ["hwc"] * n), "k_frame_dist",
                                     args.steps, 5 * 3 * h * w * n)
    out["ssim_kodak_x1176_rgb"] = measure(lambda: ctx.frame_ssim(kframes, ksrcs, ["hwc"] * n), "k_frame_ssim",
                                          args.steps, *ssim_work([(h, w)] * 3 * n), fp64)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
