"""Development tool: the device's canonical log / cos and common-randomness noise against the oracle's, over every
argument the noise can reach.

- log(u) and cos(fl(2 pi_ref) u) for u = s / m, every s in [1, m - 1] (m = 2^31 - 1): ccd_debug_detmath against
  the oracle's detmath.h, bit for bit;
- the noise over the generator's whole period, samples [0, (m - 1) / 2): ccd_debug_cr_noise against
  cco_noise_samples, bit for bit.

Both run in chunks of 2^24, with the oracle spread over the host's cores, so the host holds a few hundred MB at
a time.  Prints one JSON line per comparison, then the whole result.

    python tools/gpu_detmath.py [--chunk-log2 24]
"""
import argparse
import json
import os
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import ccoracle  # noqa: E402  (the checker)
import coolchic_b200  # noqa: E402,F401
from coolchic_b200 import _native  # noqa: E402

M = 2**31 - 1
PI_REF = 3.14159265359
PERIOD = (M - 1) // 2  # noise samples per period of the LCG (two draws each)


def split(n, parts):
    edges = np.linspace(0, n, parts + 1).astype(np.int64)
    return list(zip(edges[:-1].tolist(), edges[1:].tolist()))


def oracle_detmath(pool, threads, fn, x):
    y = np.empty_like(x)

    def run(lo_hi):
        lo, hi = lo_hi
        y[lo:hi] = ccoracle.detmath(fn, x[lo:hi])

    list(pool.map(run, split(x.size, threads)))
    return y


def oracle_noise(pool, threads, first, n):
    y = np.empty(n, dtype=np.float32)

    def run(lo_hi):
        lo, hi = lo_hi
        y[lo:hi] = ccoracle.noise_samples(first + lo, hi - lo)

    list(pool.map(run, split(n, threads)))
    return y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--chunk-log2", type=int, default=24)
    args = ap.parse_args()
    chunk = 1 << args.chunk_log2
    threads = max(1, len(os.sched_getaffinity(0)))
    ctx = _native.get_context(0)
    ccoracle.lib()
    res = {"gpu": torch.cuda.get_device_name(), "host_threads": threads}
    with ThreadPoolExecutor(threads) as pool:
        t0 = time.time()
        bad = {"log": [], "cos": []}
        n_bad = {"log": 0, "cos": 0}
        for lo in range(1, M, chunk):
            s = np.arange(lo, min(lo + chunk, M), dtype=np.int64)
            u = s.astype(np.float64) / float(M)
            for fn, x in (("log", u), ("cos", (2 * PI_REF) * u)):
                d = ctx.detmath(fn, x).view(np.uint64)
                o = oracle_detmath(pool, threads, fn, x).view(np.uint64)
                diff = np.flatnonzero(d != o)
                n_bad[fn] += int(diff.size)
                bad[fn] += s[diff[:4]].tolist()
        res["box_muller_arguments"] = {"s": [1, M - 1], "count": M - 1, "log_differ": n_bad["log"],
                                       "cos_differ": n_bad["cos"], "first_differing_s": bad,
                                       "seconds": round(time.time() - t0, 1)}
        print(json.dumps(res["box_muller_arguments"]), flush=True)

        t0 = time.time()
        n_diff, first_diff = 0, []
        for first in range(0, PERIOD, chunk):
            n = min(chunk, PERIOD - first)
            d = ctx.cr_noise(first, n).view(np.uint32)
            o = oracle_noise(pool, threads, first, n).view(np.uint32)
            diff = np.flatnonzero(d != o)
            n_diff += int(diff.size)
            first_diff += (first + diff[:4]).tolist()
        res["noise_period"] = {"samples": [0, PERIOD], "count": PERIOD, "differ": n_diff, "first_differing": first_diff,
                               "seconds": round(time.time() - t0, 1)}
    res["ok"] = n_bad["log"] == n_bad["cos"] == n_diff == 0
    print(json.dumps(res))
    return 0 if res["ok"] else 1


if __name__ == "__main__":
    sys.exit(main())
