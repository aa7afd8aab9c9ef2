"""Development tool: time the motion analysis (k_inter_analysis) next to the reconstruction (k_inter_predict) on one
synthetic 1080p 4:2:0 B frame, at warp filter sizes 4, 8 and 14.

The frame is the first B frame of a 3-frame stream of synth.make_video_stream (the generator of bench.py's video
workloads), decoded once; its raw residue and motion, references and global flow are kept and reused at every filter
size (the filter size is an argument of both calls).  The source is the decoded frame as 8-bit planar samples: the
timing does not depend on the values.  Per filter size: the whole ccd_inter_analysis call (CUDA events around the
C-ABI call: staging, kernel, result copy) and each kernel alone (torch.profiler), median of --steps calls, with the
card's name, power limit and max SM clock read in the same run.

    python tools/gpu_motion.py [--steps 20]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import coolchic_b200  # noqa: E402,F401
from coolchic_b200 import _native, synth  # noqa: E402
from coolchic_b200.bitstream import decode  # noqa: E402
from gpu_quality import card  # noqa: E402


def median_ms(fn, kernel, steps):
    """(whole call, kernel) medians in ms: CUDA events around fn, then torch.profiler in a run of its own."""
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
    return float(np.median(call)), (float(np.median(kern)) if kern else float("nan"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    ctx = _native.get_context(0)
    out = {"card": card()}

    ss = synth.SeedStream(ctx)
    data = synth.make_video_stream(ctx, ss, 1080, 1920, 3, "yuv420", 8, 8, seed=0)
    kept = {}

    def recon(fh, cc_out, refs, dev):
        if fh.get_value("frame_type") == "B":
            kept.update(fh=fh, cc=dict(cc_out), refs=[r.to(ctx.torch_device) for r in refs])
        return decode._reconstruct(fh, cc_out, refs, dev)

    frames = decode.decode_video_bytes(data, output_device="cuda", reconstruct_fn=recon)
    fh, cc, refs = kept["fh"], kept["cc"], kept["refs"]
    src = ctx.pack_frame(frames[str(fh.get_value("display_index"))].data, 8, "yuv420")
    gf = fh.get_value("global_flow")
    for fs in (4, 8, 14):
        args_ = (cc["residue"], cc["motion"], refs, True, "yuv420", 8, gf, fs)
        a_call, a_kern = median_ms(lambda: ctx.inter_analysis(*args_, source=src), "k_inter_analysis", args.steps)
        r_call, r_kern = median_ms(lambda: ctx.reconstruct_frame(*args_), "k_inter_predict", args.steps)
        out[f"1080p_B_fs{fs}"] = {"inter_analysis_call_ms": a_call, "k_inter_analysis_ms": a_kern,
                                  "reconstruct_call_ms": r_call, "k_inter_predict_ms": r_kern,
                                  "analysis_over_predict": a_kern / r_kern}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
