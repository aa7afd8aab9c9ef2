"""Development tool: time the entropy-model analysis (DESIGN §4.10).

- bench.py's 1080p RGB 7-grid frame (n_ctx 14, no hyperlatents): the whole per-frame rate call with every variant
  (CUDA events around the call), k_latent_rate over all variants and for one variant (torch.profiler), and the
  calibration sweep's call and k_rate_sweep (17 offsets);
- kodim14 (hyperlatents and IFCE): the same per-frame calls;
- the whole video_model_analysis of bench.py's gop32_1080p_yuv420 stream (decode included, host clock around a
  synchronised call).

Medians of --steps runs, with the card's name, power limit and max SM clock read in the same run.

    python tools/gpu_model.py [--steps 10]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import coolchic_b200  # noqa: E402,F401
from coolchic_b200 import synth  # noqa: E402
from coolchic_b200.bitstream import model, rate  # noqa: E402
from gpu_motion import median_ms  # noqa: E402
from gpu_quality import card  # noqa: E402


def frame_calls(ctx, data, steps):
    """Timings of the per-frame calls of video_model_analysis on the first Cool-chic of an image stream."""
    _, _, flat = rate._split_frames(data)
    _, descs, nns, lats = rate._decode_latents([flat[0][0]], [flat[0][1]], [flat[0][2]], ctx.device)
    d, nn, lat = descs[0], nns[0], lats[0]
    edits = list(model.variant_edits(d).values())
    n = len(edits)
    run_all = lambda: ctx.latent_rate([d] * n, [nn] * n, [lat] * n, edits=edits)  # noqa: E731
    run_one = lambda: ctx.latent_rate([d], [nn], [lat], edits=edits[:1])  # noqa: E731
    mu_sc = ctx.latent_rate([d], [nn], [lat], want_mu_sc=True)[0]["mu_sc"]
    run_sweep = lambda: ctx.rate_sweep([d], [lat], [mu_sc], model.SIGMA_OFFSETS)  # noqa: E731
    all_call, all_kern = median_ms(run_all, "k_latent_rate", steps)
    one_call, one_kern = median_ms(run_one, "k_latent_rate", steps)
    sw_call, sw_kern = median_ms(run_sweep, "k_rate_sweep", steps)
    return {"n_ctx": int(d.n_ctx), "n_grids": int(d.n_grids), "n_symbols": int(d.n_symbols()), "variants": n,
            "rate_call_all_variants_ms": all_call, "k_latent_rate_all_variants_ms": all_kern,
            "rate_call_one_variant_ms": one_call, "k_latent_rate_one_variant_ms": one_kern,
            "sweep_call_ms": sw_call, "k_rate_sweep_ms": sw_kern, "sweep_offsets": len(model.SIGMA_OFFSETS),
            "sweep_over_one_rate_pass": sw_kern / one_kern}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    from coolchic_b200 import _native

    ctx = _native.get_context(0)
    out = {"card": card()}
    ss = synth.SeedStream(ctx)
    out["1080p_rgb_7grids"] = frame_calls(ctx, synth.make_image_stream(ctx, ss, 1080, 1920, "rgb", 8, (0, 6), None, seed=0),
                                          args.steps)
    out["kodim14"] = frame_calls(ctx, open(os.path.join(ROOT, "tests", "golden", "kodim14.cool"), "rb").read(), args.steps)
    video = synth.make_video_stream(ctx, ss, 1080, 1920, 32, "yuv420", 8, 8, seed=0)
    out["gop32_1080p_yuv420"] = {"video_model_analysis_ms": wall_ms(lambda: model.video_model_analysis(video)),
                                 "video_rate_ms": wall_ms(lambda: rate.video_rate(video))}
    print(json.dumps(out))


def wall_ms(fn, runs=3):
    """Median host time of fn in ms, each run between two device synchronisations, after one warm-up run."""
    fn()
    times = []
    for _ in range(runs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        times.append(1e3 * (time.perf_counter() - t0))
    return float(np.median(times))


if __name__ == "__main__":
    main()
