"""Which paths of the range coder a stream reaches, counted on the device, and every symbol accounted for.

The bit-exact tests of test_coder_loop and test_entropy_edges only prove the paths a decode actually runs.  Here the
instrumented library (`make prof`, -DCCD_PROFILE: libccdec_prof.so) decodes crafted streams in one subprocess (the
library is loaded once per process) and prints one CCDPROF line per grid.  Per grid it counts matched rounds of the
steady loop and of the one-round path, every failed round by where it ran (steady round A, steady round B, one-round
path) and by its decided prefix (0, 1 or 2 symbols), failed rounds followed by a window move, failed rounds whose far
symbol took the exact f64 model, exits of the steady loop for want of ready symbols, and single-symbol steps (through
tier 2, and with the exact model).  What is checked, for every stream and every producer mask:
  1. the instrumented decode is bit-exact too: latents and status [1] (words consumed), [2] (exact-model symbols) are
     the oracle's and [0] is 0;
  2. one line per grid, in decode order, with the grid's offset and size;
  3. every symbol accounted for: n = 3 (matched rounds) + decided prefixes + failed rounds + single steps, and on the
     grid's own latents: failed rounds <= #symbols outside {M-1, M, M+1} <= failed rounds + tier-2 single steps,
     exact-model decisions == #symbols outside the 32-entry window;
  4. each stream reaches the paths its name says (counts > 0), and a deep generic ARM under a one-warp producer mask
     starves the steady loop hundreds of times;
  5. the five fast kernel instances and the generic one, 8-warp CTAs (more streams than SMs in one call) and the
     512-slot window ring of a frame wider than 5 070 pixels each show failed rounds of the steady loop, window moves
     and failed rounds of the one-round path;
  6. an all-mode stream has no failed round, prefix or exact decision, and still satisfies 3.
Counts that depend on timing (starvation, waits, single steps, how matched rounds split between the steady loop and the
one-round path) are only checked as lower bounds or through 3."""
import json
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
from conftest import ROOT
from test_coder_loop import HW, LR, SMAX, STREAMS, loop_stream
from test_entropy_edges import DEFAULT_MASK, EXTRA_MODELS, MODELS, _oracle_backend, build_stream, classes, mode_of
from test_rate import _latent_offsets, model_indices

PROF_LIB = os.path.join(ROOT, "cool-chic_b200", "csrc", "libccdec_prof.so")
# the numbers of a CCDPROF line, in order (tools/gpu_1080.py reads the same line)
FIELDS = ("ord", "n", "st_c", "st_n", "fa_c", "fa_n", "pre", "mv_n", "rf_n", "sv_n", "wt_c", "wt_n", "one_c", "one_n",
          "one_ok", "sg_c", "sg_n", "rare_c", "cta", "a0", "a1", "a2", "b0", "b1", "b2", "o0", "o1", "o2", "fmove",
          "fexact", "tier", "sexact")
CELLS = ("a0", "a1", "a2", "b0", "b1", "b2", "o0", "o1", "o2")
MASKS = (DEFAULT_MASK, 0x0001, 0x3FFF)
INSTANCE_HW, INSTANCE_LR = (64, 640), (0, 3)  # 64-symbol diagonals on the finest grid: the steady loop runs
INSTANCES = [((6, 2), False), ((10, 2), False), ((10, 4), False), ((14, 6), False), ((20, 6), False), ((8, 6), False),
             ((14, 6), True)]
WIDE_HW, WIDE_LR = (128, 5120), (0, 2)  # 128-symbol diagonals of 5 120-pixel rows: a 512-slot ring
DEEP_HW, DEEP_LR = (64, 640), (0, 3)


# ---- the counter table ----------------------------------------------------------------------------------------------
def parse_prof(text):
    """The CCDPROF lines of a decode's output, as dicts of FIELDS (in the order printed)."""
    import re

    rows = []
    for line in text.splitlines():
        if line.startswith("CCDPROF"):
            v = [int(x) for x in re.findall(r"-?\d+", line)]
            assert len(v) == len(FIELDS), line
            rows.append(dict(zip(FIELDS, v)))
    return rows


def n_failed(r):
    return sum(r[c] for c in CELLS)


def accounted(r):
    """Identity 3: the symbols the counters decide, each counted once."""
    return 3 * (r["st_n"] + r["one_ok"]) + r["pre"] + n_failed(r) + r["sg_n"]


def check_row(r, cls):
    """Every symbol of one grid accounted for; `cls` the classes (test_entropy_edges.classes) of its symbols."""
    far, exact = int((cls >= 2).sum()), int((cls == 3).sum())
    assert accounted(r) == r["n"] == len(cls), r
    assert r["pre"] == sum(k * r[c] for c in CELLS for k in (int(c[1]),) if k), r
    assert r["fa_n"] == sum(r[c] for c in CELLS[:6]), r  # n_fail: every steady failed round, starving ones included
    assert n_failed(r) <= far <= n_failed(r) + r["tier"], (r, far)
    assert r["fexact"] + r["sexact"] == exact, (r, exact)
    assert r["fmove"] <= min(r["mv_n"], r["fa_n"]) and r["fexact"] <= n_failed(r), r
    assert r["sexact"] <= r["tier"] <= r["sg_n"] and r["one_ok"] <= r["one_n"], r


def test_identity_on_hand_made_tables():
    """Identity 3 on a hand-made grid of 40 symbols: 4 matched steady rounds, 2 matched one-round rounds, failed
    rounds with prefixes 2 (round A), 0 (round B, the loop then starves) and 1 (one-round path), 16 single steps.  The
    counter as it was before the fix left the starving failed round out of n_fail and of the table: then the identity
    and the n_fail check fail."""
    r = dict.fromkeys(FIELDS, 0)
    r.update(n=40, st_n=4, one_ok=2, one_n=3, a2=1, b0=1, o1=1, pre=3, fa_n=2, mv_n=1, fmove=1, sg_n=16, tier=3,
             sexact=1, fexact=1, sv_n=1)
    # the far symbols of the three failed rounds (one exact), two far single steps (one exact), a near one through tier 2
    cls = np.array([0] * 34 + [1, 2, 2, 2, 3, 3])
    assert accounted(r) == 40
    check_row(r, cls)
    old = dict(r, b0=0, fa_n=1)
    assert accounted(old) == 39
    with pytest.raises(AssertionError):
        check_row(old, cls)
    with pytest.raises(AssertionError):
        check_row(dict(old, fa_n=2), cls)


# ---- the streams --------------------------------------------------------------------------------------------------
def _deep_arch():
    from test_arm_space import Arch

    return Arch(40, 7, 0, DEEP_HW, DEEP_LR, seed=3)  # the deepest and widest generic ARM without IFCE


def _streams():
    """name -> (desc, nn, nn bytes, latent bytes, latents, mu_idx), all written by the oracle on the CPU."""
    backend = _oracle_backend()
    out = {}
    for kind in STREAMS:
        s, _ = loop_stream(backend, kind, seed=1)
        out[kind] = (s.desc, s.nn, s.nb, s.lb, s.lat, s.mu)
    s = build_stream(backend, None, SMAX, "P0", hw=HW, lr=LR)
    out["all_mode"] = (s.desc, s.nn, s.nb, s.lb, s.lat, s.mu)
    for shape, big in INSTANCES:
        for pattern in ("P2", "P5"):
            if pattern == "P5" and shape != (14, 6):
                continue
            s = build_stream(backend, None, EXTRA_MODELS["G"] if big else MODELS["D"], pattern, seed=21, shape=shape,
                             hw=INSTANCE_HW, lr=INSTANCE_LR)
            out[f"inst_{shape[0]}_{shape[1]}{'_G' if big else ''}_{pattern}"] = (s.desc, s.nn, s.nb, s.lb, s.lat, s.mu)
    s = build_stream(backend, None, MODELS["D"], "P2", seed=22, hw=WIDE_HW, lr=WIDE_LR)
    out["wide"] = (s.desc, s.nn, s.nb, s.lb, s.lat, s.mu)
    from test_arm_space import build

    a = build(_deep_arch())
    out["deep"] = (a.desc, a.nn, a.nb, a.lb, a.lat, model_indices(a.desc, a.nn, a.lat)[0])
    return out


def _calls(names, n_sm):
    """(stream names, producer mask) of each decode call."""
    calls = [([k], m) for k in list(STREAMS) + ["all_mode"] for m in MASKS]
    calls += [([k], DEFAULT_MASK) for k in names if k.startswith("inst_") or k == "wide"]
    calls += [(["deep"], DEFAULT_MASK), (["deep"], 0x0001)]
    calls.append(([("inst_14_6_P2", "inst_14_6_P5")[i % 2] for i in range(n_sm + 4)], DEFAULT_MASK))  # 8-warp CTAs
    return calls


def test_stream_designs():
    """Host only: the streams are what their names say, and each has the class counts the checks below rely on."""
    from test_arm_space import refused, rule_fast

    st = _streams()
    for name, (d, nn, nb, lb, lat, mu) in st.items():
        cls = classes(lat, mode_of(mu))
        if name == "all_mode":
            assert (cls == 0).all()
        elif name == "deep":
            assert d.n_ctx == 40 and d.arm_hidden == 7 and not rule_fast(d, nn) and not refused(d, nn)
            assert (cls >= 2).sum() > 0
        else:
            assert (cls >= 2).sum() > 0.01 * lat.size, name
        if name == "exact":
            assert ((cls == 2).sum(), (cls == 3).sum() > 0) == (0, True)
    from test_arm_f64 import FAST_SHAPES

    for shape, big in INSTANCES:
        d, nn = st[f"inst_{shape[0]}_{shape[1]}{'_G' if big else ''}_P2"][:2]
        assert rule_fast(d, nn) == (shape in FAST_SHAPES and not big)
    assert {s for s, big in INSTANCES if not big} >= set(FAST_SHAPES)
    from coolchic_b200 import _native

    assert st["wide"][0].img_w > 5070 and _native.entropy_plan(*st["wide"][:2])[0] == 512
    # 8-warp CTAs, two per SM, for more streams of one kernel key than SMs: two CTAs' shared memory fit an SM
    assert max(2 * (_native.entropy_plan(*st[k][:2])[2] + 1024) for k in ("inst_14_6_P2", "inst_14_6_P5")) <= 227 * 1024


# ---- the device ---------------------------------------------------------------------------------------------------
def _decode_all(path_in, path_out):
    """Run in a fresh process with CCD_LIB = the instrumented library: every call of the input, its latents, status
    words and CCDPROF lines (the process's fd 1, where device printf lands, captured around each call)."""
    import ctypes

    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native
    from coolchic_b200._desc import CcdCoolChicDesc

    assert os.path.samefile(_native.LIB_PATH, PROF_LIB)
    libc = ctypes.CDLL(None)
    ctx = _native.get_context(0)
    z = np.load(path_in)
    calls = json.loads(str(z["calls"]))
    out = {}
    for ci, (names, mask) in enumerate(calls):
        descs = [CcdCoolChicDesc.from_buffer_copy(z[f"{k}/desc"].tobytes()) for k in names]
        nbs = [z[f"{k}/nb"].tobytes() for k in names]
        lbs = [z[f"{k}/lb"].tobytes() for k in names]
        ctx.set_producer_mask(mask)
        sys.stdout.flush()
        saved = os.dup(1)
        with tempfile.TemporaryFile(mode="w+b") as f:
            os.dup2(f.fileno(), 1)
            try:
                _, lats = ctx.decode_many(descs, nbs, lbs, want_latents=True)
                torch.cuda.synchronize()
            finally:
                libc.fflush(None)
                sys.stdout.flush()
                os.dup2(saved, 1)
                os.close(saved)
            f.seek(0)
            rows = parse_prof(f.read().decode(errors="replace"))
        out[f"{ci}/status"] = np.array(ctx.last_status())
        out[f"{ci}/prof"] = np.array([[r[k] for k in FIELDS] for r in rows], np.int64).reshape(-1, len(FIELDS))
        for i, lat in enumerate(lats):
            out[f"{ci}/lat{i}"] = lat.cpu().numpy()
    ctx.set_producer_mask(DEFAULT_MASK)
    out["n_sm"] = np.array(torch.cuda.get_device_properties(0).multi_processor_count)
    np.savez(path_out, **out)


def _grid_spans(d):
    """(offset, size, grid index) of each grid in decode order."""
    offs = _latent_offsets(d)
    return [(offs[g], d.grid_h[g] * d.grid_w[g], g) for g in range(d.n_grids - 1, -1, -1)]


def _fmt(r):
    return (f"n {r['n']:7d} | steady {r['st_n']:6d} one {r['one_ok']:5d}/{r['one_n']:<5d} | fails A {r['a0']}/{r['a1']}/"
            f"{r['a2']} B {r['b0']}/{r['b1']}/{r['b2']} one {r['o0']}/{r['o1']}/{r['o2']} | move {r['mv_n']} "
            f"fail+move {r['fmove']} | exact {r['fexact']}+{r['sexact']} | starve {r['sv_n']} | single {r['sg_n']} "
            f"tier2 {r['tier']}")


@pytest.mark.gpu
def test_coder_paths_on_device(oracle, tmp_path):
    import torch

    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    assert os.path.exists(PROF_LIB), "libccdec_prof.so is missing: build() makes it (make -C cool-chic_b200/csrc prof)"
    n_sm = torch.cuda.get_device_properties(0).multi_processor_count
    st = _streams()
    calls = _calls(list(st), n_sm)
    arrays = {"calls": np.array(json.dumps(calls))}
    for k, (d, nn, nb, lb, lat, mu) in st.items():
        arrays.update({f"{k}/desc": np.frombuffer(bytes(d), np.uint8), f"{k}/nn": nn,
                       f"{k}/nb": np.frombuffer(nb, np.uint8), f"{k}/lb": np.frombuffer(lb, np.uint8)})
    np.savez(tmp_path / "in.npz", **arrays)
    here = os.path.dirname(os.path.abspath(__file__))
    code = (f"import sys; sys.path[:0] = [{here!r}, {os.path.join(ROOT, 'oracle')!r}, {ROOT!r}]; import test_coder_paths; "
            f"test_coder_paths._decode_all({str(tmp_path / 'in.npz')!r}, {str(tmp_path / 'out.npz')!r})")
    subprocess.run([sys.executable, "-c", code], check=True, cwd=here, env=dict(os.environ, CCD_LIB=PROF_LIB))
    z = np.load(tmp_path / "out.npz")
    assert int(z["n_sm"]) == n_sm

    # per stream: words consumed (oracle), classes of every symbol in decode order
    ref = {}
    for k, (d, nn, nb, lb, lat, mu) in st.items():
        lat_o, stats = oracle.decode_latents(d, nn, lb)
        assert np.array_equal(lat_o, lat), k
        ref[k] = (int(stats[0]), classes(lat, mode_of(mu)))

    seen = {}  # (name, mask) -> per-grid rows of the stream's decode
    print()
    for ci, (names, mask) in enumerate(calls):
        rows = [dict(zip(FIELDS, (int(x) for x in v))) for v in z[f"{ci}/prof"]]
        if len(names) == 1:
            print(f"{names[0]} mask {mask:#06x}")
            for r, (_, _, g) in zip(rows, _grid_spans(st[names[0]][0])):
                print(f"  grid {g}: {_fmt(r)}")
        else:
            tot = {f: sum(r[f] for r in rows) for f in FIELDS}
            print(f"{len(names)} streams in one call, mask {mask:#06x}: {len(rows)} lines, "
                  f"{len({r['cta'] for r in rows})} CTAs: {_fmt(tot)}")
    for ci, (names, mask) in enumerate(calls):
        rows = [dict(zip(FIELDS, (int(x) for x in v))) for v in z[f"{ci}/prof"]]
        n_lines = sum(st[k][0].n_grids for k in names)
        assert len(rows) == n_lines, f"call {ci} ({names[0]}, {hex(mask)}): {len(rows)} CCDPROF lines, want {n_lines}"
        status = [int(x) for x in z[f"{ci}/status"][:4]]
        for i, k in enumerate(names):
            d, nn, nb, lb, lat, mu = st[k]
            assert np.array_equal(z[f"{ci}/lat{i}"], lat), (k, hex(mask))
            mine = [r for r in rows if r["cta"] == i]  # one stream per CTA, the call's order (one kernel key)
            spans = _grid_spans(d)
            assert [(r["ord"], r["n"]) for r in mine] == [(o, n) for o, n, _ in spans], (k, hex(mask))
            words, cls = ref[k]
            for r, (o, n, _) in zip(mine, spans):
                check_row(r, cls[o:o + n])
            if i == len(names) - 1:
                want = [0, words, int((cls == 3).sum()), 0]
                assert status == want and sum(r["fexact"] + r["sexact"] for r in mine) == status[2], (k, status, want)
            if len(names) == 1:
                seen[(k, mask)] = mine
        if len(names) > 1:
            seen[("narrow", mask)] = rows

    def total(rows, f):
        return sum(r[f] for r in rows)

    # 4. each stream reaches what its name says (default mask), and the coarse grids take the one-round path
    finest = seen[("positions", DEFAULT_MASK)][-1]
    assert all(finest[c] > 0 for c in CELLS[:6]), _fmt(finest)
    assert sum(total(seen[("back2back", DEFAULT_MASK)], c) for c in ("a0", "b0", "o0")) > 0
    assert total(seen[("move", DEFAULT_MASK)], "fmove") > 0
    assert total(seen[("exact", DEFAULT_MASK)], "fexact") > 0
    for k in STREAMS:
        coarse = seen[(k, DEFAULT_MASK)][:-1]
        assert sum(n_failed(r) - sum(r[c] for c in CELLS[:6]) for r in coarse) > 0 and total(coarse, "sg_n") > 0, k
    starve = total(seen[("deep", 0x0001)], "sv_n")
    print(f"starvation: deep ARM (40 contexts, 7 hidden layers, {DEEP_HW[0]}x{DEEP_HW[1]}) one-warp mask: {starve}; "
          f"loop streams one-warp mask: {[total(seen[(k, 0x0001)], 'sv_n') for k in STREAMS]}")
    assert starve >= 200
    # 5. every kernel instance, the 8-warp shape and the 512-slot ring: steady failed rounds, moves, one-round fails
    shapes = [(k, DEFAULT_MASK) for k in st if k.startswith("inst_") and k.endswith("_P2")]
    shapes += [("wide", DEFAULT_MASK), ("narrow", DEFAULT_MASK)]
    for key in shapes:
        rows = seen[key]
        assert total(rows, "fa_n") > 0 and total(rows, "mv_n") > 0, key
        assert sum(n_failed(r) - r["fa_n"] for r in rows) > 0, key
    narrow = seen[("narrow", DEFAULT_MASK)]
    assert len({r["cta"] for r in narrow}) == n_sm + 4 > n_sm
    # 6. the all-mode stream: nothing fails, nothing is decided by the exact model
    for mask in MASKS:
        for r in seen[("all_mode", mask)]:
            assert n_failed(r) == r["pre"] == r["fexact"] == r["sexact"] == r["fmove"] == 0, _fmt(r)
