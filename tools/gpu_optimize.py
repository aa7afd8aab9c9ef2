"""Lossless optimiser on the GPU (DESIGN §4.11): bytes saved and wall time on kodim14, the seed 1080p frame and one GOP,
and the time of one ccd_rate_candidates call (K candidates) against one ccd_latent_rate pass.

    python tools/gpu_optimize.py [--rounds N] [--out results.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import coolchic_b200  # noqa: E402,F401
from coolchic_b200 import _native, synth  # noqa: E402
from coolchic_b200._desc import desc_from_header  # noqa: E402
from coolchic_b200.bitstream.optimize import optimize_bitstream  # noqa: E402


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unknown ({e})"


def timed(fn, n):
    fn()
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / n


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--rounds", type=int, default=8)
    p.add_argument("--out", default=None, help="also write the results to this JSON file")
    a = p.parse_args()
    ctx = _native.get_context(0)
    golden = os.path.join(ROOT, "tests", "golden")
    streams = {
        "kodim14": open(os.path.join(golden, "kodim14.cool"), "rb").read(),
        "seed_1080p": synth.make_image_stream(ctx, synth.SeedStream(ctx), 1080, 1920),
        "gop5_64x96_yuv420": open(os.path.join(golden, "gop5_64x96_yuv420.cool"), "rb").read(),
    }
    res = {"gpu": gpu_info(), "streams": {}}
    for name, data in streams.items():
        t = time.perf_counter()
        out, rep = optimize_bitstream(data, max_rounds=a.rounds)
        wall = time.perf_counter() - t
        ccs = [dict(name=c.name, bytes=(c.bytes_before, c.bytes_after), nn=(c.nn_bytes_before, c.nn_bytes_after),
                    latent=(c.latent_bytes_before, c.latent_bytes_after),
                    latent_bits=(c.latent_bits_before, c.latent_bits_after), arm=c.arm_bits_saved,
                    ifce=c.ifce_bits_saved, recount=c.recount_bits_saved, bias=c.bias_reset_bits_saved,
                    rounds=c.rounds, candidates=c.candidates, seconds=c.seconds, kept=c.kept_original)
               for c in rep.coolchics]
        res["streams"][name] = dict(bytes_before=len(data), bytes_after=len(out), wall_s=wall, coolchics=ccs)
        print(name, len(data), "->", len(out), f"bytes, {wall:.2f} s", flush=True)
        for c in ccs:
            print("   ", c, flush=True)
    # one candidate call against one rate pass, on the first Cool-chic of each image stream
    for name in ("kodim14", "seed_1080p"):
        data = streams[name]
        v, f, h, nb, lb = synth.parse_single_image(data)
        d = desc_from_header(h)
        nn = _native.decode_nn(d, nb)
        _, (lat,) = ctx.decode_many([d], [nb], [lb], want_latents=True)
        t_rate = timed(lambda: ctx.latent_rate([d], [nn], [lat]), 20)
        row = {"latent_rate_ms": 1e3 * t_rate}
        for k in (1, 16, 64):
            cands = [(i % 900, 1 if i % 2 else -1) for i in range(k)]
            row[f"candidates_{k}_ms"] = 1e3 * timed(lambda: ctx.rate_candidates(d, nn, lat, cands), 10)
        row["per_candidate_ms_at_64"] = (row["candidates_64_ms"] - row["candidates_1_ms"]) / 63
        res[f"timing_{name}"] = row
        print(name, row, flush=True)
    print("gpu:", res["gpu"])
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
