"""The speculative coder's steady loop around its matched path: failed rounds, window moves and the reads of `ready`.

A round decides three symbols when all are in {M-1, M, M+1}.  A failed round takes the decided prefix (0, 1 or 2
symbols) and decides the next symbol, which is outside those three, from its 32-entry window, or with the exact f64
model outside the window; the loop then starts again at the new position.  The loop runs two rounds per iteration, so
a far symbol at a gap g after the previous one falls at position (g - 1) mod 6 of the iteration that follows it.

The streams are built on the crafted constant ARMs of test_entropy_edges (every symbol has the same mode), with a
background of the B(3, 3) de Bruijn sequence over {M-1, M, M+1} so that matched rounds come from every lane, and far
symbols placed in coding order:
  positions   gaps 7 ... 18: a failed round at each of the six positions of an iteration, twice over;
  back2back   runs of 2 ... 5 adjacent far symbols: failed rounds back to back, with an empty decided prefix;
  move        sigma min and gaps 1 ... 4: every far symbol costs about a word, so the word window moves every few
              rounds, and the move coincides with a failed round;
  exact       far symbols outside the window: the exact model decides the first undecided symbol of a failed round.
Each stream is decoded under the default, a one-warp and an all-warp producer mask, and must equal the oracle bit for
bit, status words included: [1] words consumed and [2] the symbols decided by the exact model.  Under the one-warp
mask the producers fall so far behind that on `positions` and `move` the coder never enters the steady loop (one-round
and single-symbol steps only); on `back2back` and `exact` the loop runs and leaves for want of ready symbols (about
1 400 and 2 800 times on an H100).  tests/test_coder_paths.py counts these paths on the device."""
import numpy as np
import pytest
from test_entropy_edges import (DB28, WIN_HALF, Model, _check_stream, _oracle_backend, build_stream, classes,  # noqa: F401
                                masks, mode_of)
from test_rate import _coding_order, model_indices

HW, LR = (256, 640), (0, 6)  # finest-grid diagonals of 64 symbols: the steady loop
SMAX, SMIN = Model(16384, 2560), Model(16384, 0)
WINDOW = [-WIN_HALF, -9, -5, -2, 2, 5, 9, WIN_HALF + 2]  # inside the window, outside {M-1, M, M+1}
EXACT = [-WIN_HALF - 1, -40, WIN_HALF + 3, 50]           # outside the window


def far_positions(kind, n, rng):
    """Coding-order positions of the far symbols."""
    pos, p, k = [], 0, 0
    while True:
        if kind in ("positions", "exact"):
            p += 7 + k % 12
            run = 1
        elif kind == "back2back":
            p += 6 + int(rng.integers(0, 15))
            run = 2 + k % 4
        else:  # move
            p += 1 + k % 4
            run = 1
        if p + run > n:
            return np.array(pos, np.int64)
        pos.extend(range(p, p + run))
        p += run - 1
        k += 1


STREAMS = {
    "positions": (SMAX, WINDOW),
    "back2back": (SMAX, WINDOW + EXACT),
    "move": (SMIN, WINDOW),
    "exact": (SMAX, EXACT),
}


def loop_stream(backend, kind, seed=0):
    model, offsets = STREAMS[kind]
    s0 = build_stream(backend, None, model, "P0", hw=HW, lr=LR)
    n = s0.desc.n_symbols()
    rng = np.random.default_rng(seed)
    M = int(mode_of(model.mu))
    off = DB28[np.arange(n) % 28].copy()  # coding order
    far = far_positions(kind, n, rng)
    off[far] = rng.choice(offsets, size=len(far))
    lat = np.empty(n, np.int64)
    lat[_coding_order(s0.desc)] = np.clip(M + off, -64, 63)
    s = build_stream(backend, None, model, None, latents=(lat, s0.mu, s0.sc), hw=HW, lr=LR)
    mi, si = model_indices(s.desc, s.nn, s.lat)
    assert np.array_equal(mi, s.mu) and np.array_equal(si, s.sc)
    return s, far


@pytest.mark.parametrize("kind", list(STREAMS))
def test_streams_have_their_design(kind):
    """Host only: the far symbols sit where the stream's name says, and the classes count as intended."""
    s, far = loop_stream(_oracle_backend(), kind)
    cls = classes(s.lat, mode_of(s.mu))[_coding_order(s.desc)]
    assert set(np.flatnonzero(cls >= 2).tolist()) == set(far.tolist())
    gaps = np.diff(far)
    if kind == "positions":
        assert set(((gaps - 1) % 6).tolist()) == set(range(6))
    if kind == "back2back":
        assert (gaps == 1).sum() > len(far) // 2
    if kind == "move":
        assert gaps.max() <= 4 and len(s.lb) > 2 * len(far)  # more than two bytes a far symbol
    n_exact = int((cls == 3).sum())
    assert (n_exact == len(far)) if kind == "exact" else ((n_exact > 0) == (kind == "back2back"))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", list(STREAMS))
def test_coder_loop_streams(ctx, oracle, masks, kind):
    """Device encode == oracle encode; the decode gives the latents with status [0, oracle words consumed, #far, 0]
    under the default, a one-warp and an all-warp producer mask."""
    s, _ = loop_stream(ctx, kind, seed=1)
    _check_stream(ctx, oracle, masks, s)
