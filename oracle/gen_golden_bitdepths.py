"""Generate the reference fixtures above 10 bits (tests/test_bitdepths.py, tests/test_reference64.py):

  * tests/golden/<name>.cool: small synthetic streams at 9, 12, 13 and 16 bits, written by coolchic_b200.synth with
    the oracle as range encoder.  The output transform of every intra and residue Cool-chic is stretched so that
    its 5th / 95th percentiles land just outside [0, 1] (or around 0, for a residue): each frame then has samples
    at 0, at M = 2^b - 1 and, at 16 bits, well above 32768;
  * <name>.npz (I frames; planes "rgb" or "y" / "u" / "v") or <name>_frames.npz (GOPs; "<display>" or
    "<display>_<plane>"): the integer samples of the UNMODIFIED REFERENCE's decode (through oracle/refshim);
  * <name>_raw.npz: the reference's raw fp32 output of every Cool-chic, in coding order (key c<i>);
  * <name>.yuv / <name>.ppm: the bytes the reference's own decode_video writes for the stream (yuv: every frame
    appended, 2-byte samples only at 10 bits; ppm: the last frame in display order, 2-byte samples MSB first).

Needs a reference checkout (COOLCHIC_REFERENCE=<path>).  Output is byte for byte reproducible.  TEST INFRASTRUCTURE
ONLY.

    python oracle/gen_golden_bitdepths.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import torch  # noqa: E402

import ccoracle  # noqa: E402
import pipeline  # noqa: E402
from gen_golden_archs import GOLD, levels, ref_decode, report, save_npz  # noqa: E402  (sets the import paths)
from coolchic_b200 import synth  # noqa: E402
from coolchic_b200._desc import desc_from_header  # noqa: E402
from coolchic_b200.bitstream.header import NN_KINDS, NN_MODULES  # noqa: E402

# name -> (h, w, frames, format, bitdepth, warp filter size); the writer's extension follows the format
STREAMS = {
    "img_40x56_rgb_9bit": (40, 56, 1, "rgb", 9, None),
    "img_44x60_yuv420_12bit": (44, 60, 1, "yuv420", 12, None),
    "img_40x56_yuv444_16bit": (40, 56, 1, "yuv444", 16, None),
    "img_37x53_rgb_16bit": (37, 53, 1, "rgb", 16, None),
    "gop3_40x56_yuv420_16bit": (40, 56, 3, "yuv420", 16, 8),
    "gop3_39x57_rgb_13bit": (39, 57, 3, "rgb", 13, 4),
}
SYN_BIAS = NN_MODULES.index("synthesis") * len(NN_KINDS) + NN_KINDS.index("bias")
# where the 5th and 95th percentiles of the output transform's first three channels are moved to
TARGET_INTRA = (-0.06, 1.06)
TARGET_RESIDUE = (-0.45, 0.45)


def stretch(desc, ints, raw, lo, hi):
    """The network integers with output channels 0..2 mapped affinely so that their 5th / 95th percentiles (on
    ``raw``, the unmodified output) go to about lo / hi: the rows of the output transform scaled, its biases shifted."""
    t = synth.split_nn(desc, ints)
    w, b = t["synthesis.weight"]["out"], t["synthesis.bias"]["out"]
    qb = 2.0 ** desc.qshift[SYN_BIAS]
    for c in range(3):
        p5, p95 = np.percentile(raw[c].astype(np.float64), [5, 95])
        a = (hi - lo) / max(p95 - p5, 1e-3)
        w[c] = np.round(a * w[c])
        b[c] = int(round(a * b[c] + (lo - a * p5) / qb))
    out, _ = synth.join_nn(desc, t)
    return out


def stretching_make_coolchic(orig):
    """synth.make_coolchic with the output transform of full-resolution Cool-chics (intra and residue; motion
    Cool-chics start at grid 2) stretched by ``stretch``."""

    def make(ctx, ss, img_size, latent_resolution=(0, 6), hyperlatent_resolution=None, seed=0,
             final_upsampling_type=None, overrides=None, latents=None, nn=None):
        if latent_resolution[0] != 0:
            return orig(ctx, ss, img_size, latent_resolution, hyperlatent_resolution, seed, final_upsampling_type,
                        overrides)
        header = synth.make_coolchic_header(ss.header, img_size, latent_resolution, hyperlatent_resolution,
                                            final_upsampling_type, overrides)
        desc = desc_from_header(header)
        ints = synth.adapt_nn(ss.desc, ss.nn, desc)
        lat = synth.tile_latents(ss.desc, ss.latents, desc, seed)
        raw = ccoracle.synthesize(desc, ints, lat.numpy())
        lo, hi = TARGET_INTRA if desc.syn_out[desc.n_syn_layers - 1] == 3 else TARGET_RESIDUE
        return orig(ctx, ss, img_size, latent_resolution, hyperlatent_resolution, seed, final_upsampling_type,
                    overrides, latents=lat, nn=stretch(desc, ints, raw, lo, hi))

    return make


def coverage(name, ints, bd):
    """Per frame: the counts of samples at 0, at M and >= 32768; every frame must have all three (the last at 16 bits,
    1 % of its samples at least)."""
    M = 2**bd - 1
    frames = {}
    for k, v in ints.items():
        frames.setdefault(k.split("_")[0], []).append(v.astype(np.int64))
    for k, planes in sorted(frames.items()):
        n0 = sum(int((p == 0).sum()) for p in planes)
        nm = sum(int((p == M).sum()) for p in planes)
        nhi = sum(int((p >= 32768).sum()) for p in planes)
        n = sum(p.size for p in planes)
        print(f"{name} frame {k}: {n0} samples at 0, {nm} at M = {M}, {nhi} >= 32768, of {n}")
        assert n0 > 0 and nm > 0 and (bd < 16 or nhi >= n // 100), (name, k)


def main():
    be = pipeline.OracleBackend()
    ss = synth.SeedStream(be)
    synth.make_coolchic = stretching_make_coolchic(synth.make_coolchic)
    for name, (h, w, n, fmt, bd, fs) in STREAMS.items():
        if n == 1:
            data = synth.make_image_stream(be, ss, h, w, fmt, bd, (0, 4), None, seed=7)
        else:
            data = synth.make_video_stream(be, ss, h, w, n, fmt, bd, fs, seed=7)
        path = os.path.join(GOLD, name + ".cool")
        with open(path, "wb") as f:
            f.write(data)
        frames, raws = ref_decode(path)
        ints = levels(frames)
        coverage(name, ints, bd)
        if n == 1:  # gen_golden_modes.py's keys: the planes only
            save_npz(os.path.join(GOLD, name + ".npz"), {k.split("_")[-1] if "_" in k else "rgb": v
                                                         for k, v in ints.items()})
        else:
            save_npz(os.path.join(GOLD, name + "_frames.npz"), ints)
        save_npz(os.path.join(GOLD, name + "_raw.npz"), {f"c{i}": r for i, r in enumerate(raws)})
        # the reference's own writers, through its decode_video
        from coolchic.bitstream.decode import decode_video as ref_decode_video

        out = os.path.join(GOLD, name + (".ppm" if fmt == "rgb" else ".yuv"))
        if os.path.exists(out):
            os.remove(out)  # the yuv writer appends from the second frame on
        ref_decode_video(path, out, verbosity=0)
        report(name, data, ints, raws)
        print(f"{name}: {len(data)} bytes, writer output {os.path.getsize(out)} bytes")


if __name__ == "__main__":
    main()
