"""Development tool: decode synthetic hop streams of 4K and wider frames and time them.

Streams: 3840x2160 (the entropy kernel's natural plan: a 1024-slot window ring), 5120x2880 and 7680x4320 (1024-row
row ring, 512-slot window ring) and 16383x1040 (2048-row row ring, 512-slot window ring), 8-bit RGB.  Per stream,
the median over the steps of: the whole decode call with its frame tail (CUDA events), the entropy stage and the
float tail (the library's own CUDA events, ccd_last_timing), ns per latent symbol of the entropy stage, and the
shared-memory plan (ring, rows, bytes).  The card and its power limit are read in the same run.  With the
instrumented library (CCD_LIB=.../libccdec_prof.so) the entropy kernel's cycle counters are printed too.

    python tools/gpu_wide.py [--steps 5] [--streams 4k,8k] [--out wide.json]
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

STREAMS = [("4k", (2160, 3840), (0, 7)), ("5k", (2880, 5120), (0, 7)), ("8k", (4320, 7680), (0, 8)),
           ("16383x1040", (1040, 16383), (0, 6))]


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm",
                                        "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                                       text=True).strip()
    except (OSError, subprocess.CalledProcessError):
        return torch.cuda.get_device_name()


def measure(ctx, ss, hw, lr, steps):
    cc, h, _ = synth.make_coolchic(ctx, ss, hw, lr, None, seed=1)
    h2 = type(h)()
    rest = h2.read_header(cc)
    n_nn, n_lat = h2.get_value("nn_n_bytes"), h2.get_value("n_bytes_latent")
    d = desc_from_header(h2)
    nb, lb = rest[:n_nn], rest[n_nn:n_nn + n_lat]
    ring, rows, smem = _native.entropy_plan(d, _native.decode_nn(d, nb))
    ctx.decode_many([d], [nb], [lb], finish=[(8, "rgb")])  # warm-up
    torch.cuda.synchronize()
    call, ent, tail, prof = [], [], [], []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        out, _ = ctx.decode_many([d], [nb], [lb], finish=[(8, "rgb")])
        b.record()
        torch.cuda.synchronize()
        del out
        call.append(a.elapsed_time(b))
        t = ctx.last_timing()
        ent.append(t["entropy_ms"])
        tail.append(t["synthesis_ms"])
        st = ctx.last_status()
        assert st[0] == 0, st
        prof.append(st[4:16])
    n_sym = d.n_symbols()
    r = {"size": f"{hw[1]}x{hw[0]}", "grids": d.n_grids, "symbols": n_sym, "payload_bytes": len(lb),
         "ring": ring, "rows": rows, "smem": smem,
         "device_ms": float(np.median(call)), "entropy_ms": float(np.median(ent)),
         "ns_per_symbol": float(np.median(ent)) * 1e6 / n_sym, "float_tail_ms": float(np.median(tail))}
    if any(any(p) for p in prof):
        r["prof_status_4_15"] = [int(x) for x in prof[-1]]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--streams", default=",".join(s[0] for s in STREAMS))
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    ctx = _native.get_context(0)
    ss = synth.SeedStream(ctx)
    res = {"card": card(), "lib": os.path.basename(_native.LIB_PATH), "streams": {}}
    for name, hw, lr in STREAMS:
        if name not in args.streams.split(","):
            continue
        res["streams"][name] = measure(ctx, ss, hw, lr, args.steps)
        print(name, json.dumps(res["streams"][name]), flush=True)
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
