"""Development tool: 1080p synthetic stream: timings + entropy-kernel status / profile counters.

With the instrumented library (CCD_LIB=cool-chic_b200/csrc/libccdec_prof.so, `make prof`) it also tabulates the coder
warp's per-grid breakdown, which the kernel prints once per grid (CCDPROF lines): cycles and counts of matched steady
rounds, failed rounds, window moves, reads of `ready`, exits for want of ready symbols, waits, one-round and
single-symbol steps."""
import os, re, sys, tempfile, time
import numpy as np, torch
ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
import coolchic_b200
from coolchic_b200 import _native, synth
from coolchic_b200._desc import desc_from_header
ctx = _native.get_context(0)
ss = synth.SeedStream(ctx)
hyp = (4, 6) if "hyper" in sys.argv else None
for a_ in sys.argv[1:]:
    if a_.startswith("mask="): ctx._lib.ccd_debug_set_producer_mask(ctx._h, int(a_[5:], 0))
zeros = "zeros" in sys.argv
lat_in = None
if zeros:  # all-zero latents: (almost) every symbol is the mode -> time per symbol = the coder's hot path
    tmp_h = synth.make_coolchic_header(ss.header, (1080, 1920), (0, 6), hyp)
    lat_in = torch.zeros(desc_from_header(tmp_h).n_symbols(), dtype=torch.int8, device="cuda")
cc, h, lat = synth.make_coolchic(ctx, ss, (1080, 1920), (0, 6), hyp, seed=0, latents=lat_in)
h2 = type(h)(); rest = h2.read_header(cc); d = desc_from_header(h2)
nnb = rest[:h2.get_value("nn_n_bytes")]; lb = rest[h2.get_value("nn_n_bytes"):][:h2.get_value("n_bytes_latent")]
nn = _native.decode_nn(d, nnb)
print("symbols", d.n_symbols(), "payload", len(lb), "bpp %.3f" % (len(lb) * 8 / (1080 * 1920)))


def decode_capturing():
    """one decode with the process's C-level stdout (where device printf lands) captured; returns (latents, text)"""
    sys.stdout.flush()
    saved = os.dup(1)
    with tempfile.TemporaryFile(mode="w+b") as f:
        os.dup2(f.fileno(), 1)
        try:
            o = ctx.decode_latents(d, nn, lb); torch.cuda.synchronize()
        finally:
            sys.stdout.flush()
            os.dup2(saved, 1)
            os.close(saved)
        f.seek(0)
        return o, f.read().decode(errors="replace")


def prof_table(text):
    rows = []
    for line in text.splitlines():
        if line.startswith("CCDPROF"):
            v = [int(x) for x in re.findall(r"-?\d+", line)]
            rows.append(dict(zip(("ord", "n", "st_c", "st_n", "fa_c", "fa_n", "pre", "mv_n", "rf_n", "sv_n", "wt_c", "wt_n",
                                  "one_c", "one_n", "one_ok", "sg_c", "sg_n", "rare_c", "cta", "a0", "a1", "a2", "b0",
                                  "b1", "b2", "o0", "o1", "o2", "fmove", "fexact", "tier", "sexact"), v)))
    if not rows:
        return
    print("coder warp per grid (decode order; kcyc = kilo-cycles; cyc/x = cycles per round / case):")
    print("%6s %9s | %9s %8s %6s | %8s %6s %6s | %5s | %7s %5s | %7s %6s | %7s %6s %7s | %7s %6s | %8s"
          % ("grid", "symbols", "matched", "rounds", "cyc/r", "fail", "n", "cyc/f", "move", "ready", "starve", "wait",
             "n", "1-round", "n", "matched", "single", "n", "rare"))
    tot = dict.fromkeys(rows[0], 0)
    for i, r in enumerate(rows):
        for k_ in r:
            tot[k_] += r[k_]
    for name, r in [(str(i), r) for i, r in enumerate(rows)] + [("all", tot)]:
        print("%6s %9d | %9.1f %8d %6.1f | %8.1f %6d %6.0f | %5d | %7d %5d | %7.1f %6d | %7.1f %6d %7d | %7.1f %6d | %8.1f"
              % (name, r["n"], r["st_c"] / 1e3, r["st_n"], r["st_c"] / max(1, r["st_n"]), r["fa_c"] / 1e3, r["fa_n"],
                 r["fa_c"] / max(1, r["fa_n"]), r["mv_n"], r["rf_n"], r["sv_n"], r["wt_c"] / 1e3, r["wt_n"],
                 r["one_c"] / 1e3, r["one_n"], r["one_ok"], r["sg_c"] / 1e3, r["sg_n"], r["rare_c"] / 1e3))
    print("  matched: the steady loop less its rare path; fail: failed rounds of the steady loop, from the loop's exit "
          "to the next round; move: window moves; ready: reads of `ready` in the steady loop; starve: exits for want "
          "of ready symbols; rare: the steady loop's rare path in all")
    print("failed rounds by path and decided prefix 0/1/2 (A, B: the steady loop's two rounds; one: the one-round path):")
    print("%6s | %14s %14s %14s | %9s %10s | %7s %6s" % ("grid", "A", "B", "one", "fail+move", "fail exact", "tier 2",
                                                       "exact"))
    for name, r in [(str(i), r) for i, r in enumerate(rows)] + [("all", tot)]:
        print("%6s | %4d %4d %4d %4d %4d %4d %4d %4d %4d | %9d %10d | %7d %6d"
              % (name, r["a0"], r["a1"], r["a2"], r["b0"], r["b1"], r["b2"], r["o0"], r["o1"], r["o2"], r["fmove"],
                 r["fexact"], r["tier"], r["sexact"]))
    print("  tier 2 / exact: single-symbol steps through tier 2 / with the exact model")


for it in range(3):
    if it == 2:
        out, text = decode_capturing()
    else:
        out = ctx.decode_latents(d, nn, lb); torch.cuda.synchronize()
    st = ctx.last_status()
    print(ctx.last_timing(), st[:4])
    if any(st[4:]):
        print("  prof kcyc: coder wait %d total %d | producers wait %d arm %d win %d total %d | far %d redo-groups %d singles %d fast %d chunks %d | helper total %d" % tuple(st[4:16]))
prof_table(text)
print("round trip ok:", torch.equal(out, lat))
l = lat.cpu().numpy().astype(int); off = 0
for g in range(d.n_grids - 1, -1, -1):
    n = d.grid_h[g] * d.grid_w[g]; a = l[off:off + n]; off += n
    print("grid", g, (d.grid_h[g], d.grid_w[g]), "zeros %.2f mean|x| %.2f max %d" % ((a == 0).mean(), np.abs(a).mean(), np.abs(a).max()))
