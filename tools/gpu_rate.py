"""Development tool: time the rate pass (ccd_latent_rate) with CUDA events.

Workloads: the synthetic 1080p 7-grid frame of bench.py, and 132 copies of kodim14 (768x512) in one call.
Reports, per workload, the median of the whole call (host preparation, upload, kernels, sums) and of the kernels
alone (k_latent_rate, k_rate_spatial; from torch.profiler), with the card and its power limit.

    python tools/gpu_rate.py [--steps 20]
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
from coolchic_b200._desc import desc_from_header  # noqa: E402


def card():
    try:
        q = subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader",
                                     "-i", str(torch.cuda.current_device())], text=True).strip()
        return q
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def measure(ctx, descs, nns, lats, steps, spatial):
    for _ in range(3):
        ctx.latent_rate(descs, nns, lats, want_spatial=spatial)
    torch.cuda.synchronize()
    call = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        ctx.latent_rate(descs, nns, lats, want_spatial=spatial)
        b.record()
        torch.cuda.synchronize()
        call.append(a.elapsed_time(b))
    kern = {}
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            ctx.latent_rate(descs, nns, lats, want_spatial=spatial)
        torch.cuda.synchronize()
    for ev in prof.events():
        if "k_latent_rate" in ev.name or "k_rate_spatial" in ev.name:
            k = "k_latent_rate" if "k_latent_rate" in ev.name else "k_rate_spatial"
            kern.setdefault(k, []).append(ev.device_time_total / 1e3 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1e3)
    n_sym = sum(d.n_symbols() for d in descs)
    return {"symbols": n_sym, "call_ms_median": float(np.median(call)),
            "kernel_ms_median": {k: float(np.median(v)) for k, v in kern.items()},
            "ns_per_symbol": float(np.median(kern.get("k_latent_rate", [np.nan]))) * 1e6 / n_sym}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    ctx = _native.get_context(0)
    out = {"card": card()}

    ss = synth.SeedStream(ctx)
    data = synth.make_image_stream(ctx, ss, 1080, 1920)
    _, _, h, nb, lb = synth.parse_single_image(data)
    d = desc_from_header(h)
    _, lats = ctx.decode_many([d], [nb], [lb], want_latents=True)
    nn = _native.decode_nn(d, nb)
    out["1080p_rgb_7grids"] = measure(ctx, [d], [nn], lats, args.steps, spatial=True)

    with open(os.path.join(ROOT, "tests", "golden", "kodim14.cool"), "rb") as f:
        _, _, h, nb, lb = synth.parse_single_image(f.read())
    d = desc_from_header(h)
    n = 132
    _, lats = ctx.decode_many([d] * n, [nb] * n, [lb] * n, want_latents=True)
    nn = _native.decode_nn(d, nb)
    out["kodim14_x132"] = measure(ctx, [d] * n, [nn] * n, lats, args.steps, spatial=True)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
