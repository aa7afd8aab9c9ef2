"""Development tool: time the latent-grid analysis (DESIGN §4.7) with CUDA events, median of --steps calls.

Workloads:
  * ccd_synthesize_many for every variant of bench.py's 1080p_rgb_7grids frame in one call (7 drop + 6 coarse masks,
    with the I-frame tail), against the float tail of decoding that frame (ccd_last_timing's synthesis time);
  * video_grid_analysis of bench.py's gop32_1080p_yuv420 stream against its decoded frames written as an 8-bit .yuv
    source (host clock around the whole call, which ends in a device synchronise).
Reports the whole synthesize call (CUDA events), its kernels (torch.profiler, the sum of the call's launches) and its
launch count, with the card's name, power limit and max SM clock read in the same run.

    python tools/gpu_grids.py [--steps 10]
"""
import argparse
import json
import os
import re
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import coolchic_b200  # noqa: E402,F401
from coolchic_b200 import _native, synth  # noqa: E402
from coolchic_b200._desc import desc_from_header  # noqa: E402
from coolchic_b200.bitstream import decode  # noqa: E402
from coolchic_b200.bitstream.grids import synthesis_masks, video_grid_analysis  # noqa: E402
from gpu_quality import card  # noqa: E402


def events_ms(fn, steps):
    out = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        out.append(a.elapsed_time(b))
    return float(np.median(out))


def kernel_ms(fn, steps):
    """Median over calls of the summed device time of the call's kernels (torch.profiler, a run of its own)."""
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    ks = [ev for ev in prof.events() if re.search(r"\bk_\w+", ev.name) and not ev.name.startswith(("Memcpy", "Memset"))]
    t = [ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3 for ev in ks]
    per = len(t) // steps
    return float(np.median([sum(t[i:i + per]) for i in range(0, per * steps, per)])), per


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    ctx = _native.get_context(0)
    out = {"card": card()}
    ss = synth.SeedStream(ctx)

    # bench.py's 1080p_rgb_7grids frame
    data = synth.make_image_stream(ctx, ss, 1080, 1920, "rgb", 8, (0, 6), None, seed=0)
    fh, ccs, _ = decode._parse_frame(_after_video_header(data))
    h, nb, lb = ccs["residue"]
    d = desc_from_header(h)
    nb, lb = bytes(nb), bytes(lb)
    fin = decode._finish_request(fh, ccs)
    _, lats = ctx.decode_many([d], [nb], [lb], want_latents=True, finish=[fin])
    tails = []
    for _ in range(args.steps):
        ctx.decode_many([d], [nb], [lb], finish=[fin])
        tails.append(ctx.last_timing()["synthesis_ms"])
    nn = _native.decode_nn(d, nb)
    _, drop, coarse = synthesis_masks(d)
    masks = drop + coarse
    n = len(masks)
    call = lambda: ctx.synthesize([d] * n, [nn] * n, [lats[0]] * n, masks, finish=[fin] * n)  # noqa: E731
    for _ in range(3):
        call()
    torch.cuda.synchronize()
    k_ms, launches = kernel_ms(call, args.steps)
    out["synthesize_1080p_rgb_7grids"] = {
        "variants": n, "call_ms_median": events_ms(call, args.steps), "kernel_ms_median": k_ms, "launches": launches,
        "decode_float_tail_ms_median": float(np.median(tails))}
    out["synthesize_1080p_rgb_7grids"]["kernel_ms_per_variant"] = k_ms / n
    del lats
    torch.cuda.empty_cache()

    # bench.py's gop32_1080p_yuv420 stream against its decoded frames as the source
    data = synth.make_video_stream(ctx, ss, 1080, 1920, 32, "yuv420", 8, 8, seed=0)
    frames = decode.decode_video_bytes(data, output_device="cuda")
    samples = ctx.pack_frames([frames[str(i)].data for i in range(len(frames))], 8, "yuv420").cpu().numpy()
    del frames
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "src_1920x1080_30p_yuv420_8b.yuv")
        samples.tofile(path)
        video_grid_analysis(data, path)  # warm
        t = []
        for _ in range(max(1, args.steps // 5)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            video_grid_analysis(data, path)
            torch.cuda.synchronize()
            t.append(time.perf_counter() - t0)
        peak = torch.cuda.max_memory_allocated(ctx.device)
    out["analysis_gop32_1080p_yuv420"] = {"frames": 32, "call_s_median": float(np.median(t)),
                                          "torch_peak_allocated_GB": peak / 1e9}
    print(json.dumps(out))


def _after_video_header(data):
    from coolchic_b200.bitstream.header import VideoHeader

    return VideoHeader().read_header(memoryview(data))


if __name__ == "__main__":
    main()
