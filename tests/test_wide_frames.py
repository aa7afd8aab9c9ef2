"""Shared-memory plan of the entropy kernel for every frame width the header allows (1 .. 16383), on the host.

The row ring's size follows from the width alone; the window ring keeps its natural size (2 slots per symbol of the
longest diagonal + 64, 64 .. 1024) whenever that fits in the 227 KB a CTA may use, and is halved until it fits
otherwise.  A stream that fits with its natural ring gets exactly that plan."""
import math

import numpy as np
import pytest

SMEM_MAX = 227 * 1024
SLOT_BYTES = 16 + 32 * 4 + 16 + 4   # meta, window, hot entry, result word
ROW_BYTES = 64
MASK_STRIDE = 10
HEIGHTS = (1, 224, 225, 1024, 1025, 16383)
# (spatial_context_arm, n_hidden_layers_arm, output_feature_ifce) of the reference's decoder presets
# (cfg/dec/{intra,residue,motion}/*.cfg), all with the linear stabiliser
PRESET_ARMS = [(6, 1, 0), (6, 1, 2), (6, 2, 0), (6, 2, 2), (10, 2, 2), (10, 2, 4), (14, 2, 6), (20, 2, 6)]
N_GRIDS = 7


@pytest.fixture(scope="module")
def seed():
    import coolchic_b200  # noqa: F401
    from coolchic_b200 import _native, synth
    from coolchic_b200._desc import desc_from_header

    data = open(synth.SEED_STREAM, "rb").read()
    _, _, c, nn_bytes, _ = synth.parse_single_image(data)
    d = desc_from_header(c)
    return c, d, _native.decode_nn(d, nn_bytes)


def _arm_desc(seed, arm, h, w):
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    c, d0, nn0 = seed
    n_ctx, hidden, cf = arm
    ov = {"spatial_context_arm": n_ctx, "n_hidden_layers_arm": hidden, "linear_stabiliser_arm": 1,
          "output_feature_ifce": cf}
    if cf == 0:
        ov["ifce_resolution"] = None
    else:
        ov["ifce_resolution"] = [0, 2]
    hd = synth.make_coolchic_header(c, (h, w), (0, N_GRIDS - 1), None, overrides=ov)
    d = desc_from_header(hd)
    return d, synth.adapt_nn(d0, nn0, d)


def _set_width(d, w):
    """The same Cool-chic at another width: only the grid widths depend on it (core/coolchic.py:149-190)."""
    d.img_w = w
    for g in range(d.n_grids):
        d.grid_w[g] = -(-w // 2**g)


def _natural(d):
    n_max, rows_need = 1, 8
    for g in range(d.n_grids):
        h, w = d.grid_h[g], d.grid_w[g]
        raster = w <= 9
        n_max = max(n_max, 1 if raster else min(h, -(-w // MASK_STRIDE)))
        rows_need = max(rows_need, 8 if raster else (w - 1) // MASK_STRIDE + 6)
    ring = min(1024, max(64, 1 << math.ceil(math.log2(2 * n_max + 64))))
    return ring, 1 << math.ceil(math.log2(rows_need))


def test_width_only_changes_grid_widths(seed):
    from coolchic_b200 import _native

    for arm in (PRESET_ARMS[0], PRESET_ARMS[-1]):
        for h in (1, 225, 1025):
            d, nn = _arm_desc(seed, arm, h, 64)
            for w in (1, 9, 10, 5071, 10237, 16383):
                want, nn_w = _arm_desc(seed, arm, h, w)
                _set_width(d, w)
                assert bytes(d) == bytes(want) and np.array_equal(nn, nn_w)
                assert _native.entropy_plan(d, nn) == _native.entropy_plan(want, nn_w)


@pytest.mark.parametrize("arm", PRESET_ARMS, ids=[f"arm{a}-{b}-ifce{c}" for a, b, c in PRESET_ARMS])
def test_plan_for_every_width(seed, arm):
    from coolchic_b200 import _native

    widths = range(1, 16384)
    for h in HEIGHTS:
        d, nn = _arm_desc(seed, arm, h, 64)
        base = None
        for w in widths:
            _set_width(d, w)
            ring, rows, smem = _native.entropy_plan(d, nn)
            # the parts of the plan that do not depend on the ring sizes: control words, grid, ARM / IFCE blobs
            b = smem - ring * SLOT_BYTES - rows * ROW_BYTES
            assert base is None or b == base, (h, w)
            base = b
            assert smem <= SMEM_MAX, (h, w)
            assert rows >= (w - 1) // MASK_STRIDE + 6 and rows & (rows - 1) == 0, (h, w)
            assert rows * ROW_BYTES < 2**24, (h, w)       # the meta word's row index
            assert ring >= 64 and ring & (ring - 1) == 0, (h, w)
            nat_ring, nat_rows = _natural(d)
            assert ring >= min(nat_ring, 512), (h, w)     # preset ARMs keep at least 512 slots at every width
            assert rows == nat_rows, (h, w)
            if b + nat_ring * SLOT_BYTES + nat_rows * ROW_BYTES <= SMEM_MAX:
                assert ring == nat_ring, (h, w)           # fits as it is: exactly the natural plan
            else:
                assert ring < nat_ring and b + 2 * ring * SLOT_BYTES + rows * ROW_BYTES > SMEM_MAX, (h, w)


def test_wide_plans_at_the_sizes_the_issue_names(seed):
    """Frames the entropy kernel used to refuse: the natural 1024-slot ring no longer fits beside the row ring."""
    from coolchic_b200 import _native

    d, nn = _arm_desc(seed, (14, 2, 6), 2160, 3840)
    assert _native.entropy_plan(d, nn)[:2] == (1024, 512)        # 4K: unchanged
    for (h, w), rows in (((2880, 5120), 1024), ((4320, 7680), 1024), ((1040, 16383), 2048)):
        d, nn = _arm_desc(seed, (14, 2, 6), h, w)
        ring, r, smem = _native.entropy_plan(d, nn)
        assert (ring, r) == (512, rows) and smem <= SMEM_MAX


def test_refused_only_when_a_64_slot_ring_does_not_fit(seed):
    """The largest ARM a descriptor may describe (40 contexts, 7 hidden layers, int64 parameters: ~93 KB) still plans
    at 4K, but beside the 2048-row ring of a 16383-wide grid not even 64 slots fit: refused, with the bytes it
    needs and the bytes available."""
    from coolchic_b200 import _native

    big = {"spatial_context_arm": 40, "n_hidden_layers_arm": 7, "linear_stabiliser_arm": 1,
           "output_feature_ifce": 0, "ifce_resolution": None}
    from coolchic_b200 import synth
    from coolchic_b200._desc import desc_from_header

    c, d0, nn0 = seed
    plans = []
    for w in (3840, 16383):
        d = desc_from_header(synth.make_coolchic_header(c, (1040, w), (0, N_GRIDS - 1), None, overrides=big))
        nn = synth.adapt_nn(d0, nn0, d)
        if w == 3840:
            plans.append(_native.entropy_plan(d, nn))
        else:
            with pytest.raises(_native.CcdError) as e:
                _native.entropy_plan(d, nn)
    ring, rows, smem = plans[0]
    assert rows == 512 and 64 <= ring < 1024 and smem <= SMEM_MAX
    assert e.value.code == -4 and f"{SMEM_MAX} are available" in str(e.value)
