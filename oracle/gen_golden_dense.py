"""Generate the reference fixtures with every network weight live (tests/test_live_networks.py):

  * tests/golden/<name>.cool: small synthetic streams written by coolchic_b200.synth with ``live=True`` and the oracle
    as range encoder.  synth.adapt_nn pads every network the sample stream does not cover with zeros (residue channels
    3 and 4, the second flow of a B frame, synthesis units past 48, latent grids past the seventh, ARM units past
    14 + 6); synth.liven_nn fills them, and synth.scale_outputs gives every output channel the range of a real one
    (alpha and beta below 0, inside (0, 1) and above 1; flows of a few pixels);
  * <name>.npz (I frames; planes "rgb") or <name>_frames.npz (GOPs; "<display>" or "<display>_<plane>"): the integer
    samples of the UNMODIFIED REFERENCE's decode (through oracle/refshim);
  * <name>_raw.npz: the reference's raw fp32 output of every Cool-chic, in coding order (key c<i>).

Needs a reference checkout (COOLCHIC_REFERENCE=<path>).  Output is byte for byte reproducible.  TEST INFRASTRUCTURE
ONLY.

    python oracle/gen_golden_dense.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import pipeline  # noqa: E402
from gen_golden_archs import GOLD, levels, ref_decode, report, save_npz  # noqa: E402  (sets the import paths)
from coolchic_b200 import synth  # noqa: E402

VHOP = {"spatial_context_arm": 20, "output_feature_ifce": 6, "n_layer_synthesis": 4,
        "syn_layer_0": "64-1-linear-relu", "syn_layer_1": "3-1-linear-none", "syn_layer_2": "3-3-residual-relu",
        "syn_layer_3": "3-3-residual-none"}
# name -> (h, w, latent_resolution, header overrides): 8-bit RGB intra
IMAGES = {
    "img_64x96_rgb_vhop_dense": (64, 96, (0, 6), VHOP),  # cfg/dec/intra/vhop: ARM 20 + 6, 64-wide synthesis
    "img_96x128_rgb_12grids_dense": (96, 128, (0, 11), None),  # grids 7 ... 11 (1 x 1 from grid 7 on)
}
# name -> (h, w, format, warp filter size): I, B, P
GOPS = {
    "gop3_40x56_rgb_sinc8_dense": (40, 56, "rgb", 8),
    "gop3_48x72_yuv420_bicubic_dense": (48, 72, "yuv420", 4),
}
SEED = 11


def streams(backend, ss):
    """{name: bytes} of every fixture (the tests rebuild none of them: they read the committed files)."""
    out = {}
    for name, (h, w, lat, ov) in IMAGES.items():
        out[name] = synth.make_image_stream(backend, ss, h, w, "rgb", 8, lat, None, seed=SEED, overrides=ov, live=True)
    for name, (h, w, fmt, fs) in GOPS.items():
        out[name] = synth.make_video_stream(backend, ss, h, w, 3, fmt, 8, fs, seed=SEED, live=True)
    return out


def main():
    be = pipeline.OracleBackend()
    ss = synth.SeedStream(be)
    for name, data in streams(be, ss).items():
        path = os.path.join(GOLD, name + ".cool")
        with open(path, "wb") as f:
            f.write(data)
        frames, raws = ref_decode(path)
        ints = levels(frames)
        if name.startswith("img"):  # gen_golden_modes.py's keys: the planes only
            save_npz(os.path.join(GOLD, name + ".npz"), {k.split("_")[-1] if "_" in k else "rgb": v
                                                         for k, v in ints.items()})
        else:
            save_npz(os.path.join(GOLD, name + "_frames.npz"), ints)
        save_npz(os.path.join(GOLD, name + "_raw.npz"), {f"c{i}": r for i, r in enumerate(raws)})
        report(name, data, ints, raws)
        print(f"{name}: {len(data)} bytes, {len(raws)} Cool-chics")


if __name__ == "__main__":
    main()
