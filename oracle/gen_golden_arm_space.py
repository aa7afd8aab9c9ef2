"""Generate the reference fixtures of the entropy model's extreme architectures (tests/test_arm_space.py):

  * tests/golden/arch_space_<name>.cool: one 8-bit rgb I frame per architecture of GOLDEN_ARCHS, built exactly as the
    test builds its streams (synth.liven_nn weights scaled by test_arm_space.calibrate, latents tiled from the sample
    stream with noise, the oracle as range encoder);
  * arch_space_<name>.npz: the UNMODIFIED REFERENCE's decode (through oracle/refshim): its latents in decode order
    (key "latents", coarsest grid first, as entropy_coding_latent_arm returned them) and the integer samples ("rgb");
  * arch_space_<name>_raw.npz: the reference's raw fp32 output (key c0).

Needs a reference checkout (COOLCHIC_REFERENCE=<path>).  Output is byte for byte reproducible.  TEST INFRASTRUCTURE
ONLY.

    python oracle/gen_golden_arm_space.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "..", "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from gen_golden_archs import GOLD, levels, ref_decode, report, save_npz  # noqa: E402  (sets the import paths)
import test_arm_space as space  # noqa: E402


def ref_decode_with_latents(path):
    """ref_decode, with the latent grids the reference's entropy decoder returned, in decode order."""
    import coolchic.bitstream.component.coolchic as cc

    grids = []
    orig = cc.entropy_coding_latent_arm

    def recording(*a, **k):
        out = orig(*a, **k)
        grids.append(out.detach().to(torch.int64).flatten().numpy().copy())
        return out

    cc.entropy_coding_latent_arm = recording
    try:
        frames, raws = ref_decode(path)
    finally:
        cc.entropy_coding_latent_arm = orig
    return frames, raws, np.concatenate(grids).astype(np.int8)


def main():
    for name, arch in space.GOLDEN_ARCHS.items():
        s = space.build(arch)
        path = os.path.join(GOLD, f"arch_space_{name}.cool")
        with open(path, "wb") as f:
            f.write(s.data)
        frames, raws, lat = ref_decode_with_latents(path)
        assert np.array_equal(lat, s.lat), name  # the reference decodes what the oracle encoded
        ints = levels(frames)
        save_npz(os.path.join(GOLD, f"arch_space_{name}.npz"), {"rgb": ints["0"], "latents": lat})
        save_npz(os.path.join(GOLD, f"arch_space_{name}_raw.npz"), {"c0": raws[0]})
        report(name, s.data, ints, raws)
        print(f"arch_space_{name}: {arch.label}, {len(s.data)} bytes")


if __name__ == "__main__":
    main()
