"""Development tool: time the quality kernels (k_frame_dist, k_inter_stats) with CUDA events, median of --steps calls.

Workloads:
  * k_frame_dist on the 32 decoded frames of bench.py's gop32_1080p_yuv420 stream (8-bit planar sources);
  * k_frame_dist on 1176 Kodak-size (768x512) rgb frames in one call (8-bit HWC sources);
  * k_inter_stats on one 1080p B frame of that stream, with its source.
Reports, per workload, the whole call (CUDA events around the C-ABI call: staging, kernel, result copy), the kernel
alone (torch.profiler), the bytes the kernel must move and that over kernel time against the H100 SXM's 3.35 TB/s,
with the card's name and power limit read in the same run.

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


def measure(fn, kernel, steps, n_bytes):
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
    k_ms = float(np.median(kern)) if kern else float("nan")
    return {"call_ms_median": float(np.median(call)), "kernel_ms_median": k_ms, "kernel_bytes": int(n_bytes),
            "kernel_TB_per_s": n_bytes / (k_ms * 1e-3) / 1e12, "share_of_3.35TB_per_s": n_bytes / (k_ms * 1e-3) / HBM_BYTES_PER_S}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    ctx = _native.get_context(0)
    out = {"card": card()}

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
    print(json.dumps(out))


if __name__ == "__main__":
    main()
