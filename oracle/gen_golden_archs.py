"""Generate the reference answers the float64 restatement (tests/test_reference64.py) is pinned to:

  * tests/golden/arch_*.cool + .npz: small synthetic streams for the architectures and sizes no other fixture covers
    (other upsampling kernel sizes, five synthesis layers, a 3x3 first layer, one latent grid, odd and tiny sizes,
    nearest x4 at an odd size, P and B frames with sinc-10 / sinc-14 below the filter length), written by
    coolchic_b200.synth with the oracle as range encoder and DECODED BY THE UNMODIFIED REFERENCE (through
    oracle/refshim): the reference's integer samples;
  * tests/golden/<name>_raw.npz for those streams and for the older img_* / gop* fixtures: the reference's raw fp32
    output of every Cool-chic, in coding order (key c<i>), as encode_decode_coolchic returned it.

Needs a reference checkout (COOLCHIC_REFERENCE=<path>).  Output is byte for byte reproducible.  TEST INFRASTRUCTURE
ONLY.

    python oracle/gen_golden_archs.py
"""
import io
import os
import sys
import zipfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, ".."))
sys.path.insert(0, os.path.join(HERE, "refshim"))
sys.path.insert(0, os.environ["COOLCHIC_REFERENCE"])

import torch  # noqa: E402

torch.set_num_threads(1)
import coolchic_b200  # noqa: E402,F401
import pipeline  # noqa: E402
from coolchic_b200 import synth  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")


def _syn(*layers, **fields):
    ov = {"n_layer_synthesis": len(layers), **{f"syn_layer_{i}": lay for i, lay in enumerate(layers)}}
    ov.update(fields)
    return ov


# name -> (h, w, latent_resolution, final_upsampling_type, header overrides); 8-bit RGB intra
IMAGES = {
    "arch_37x61_ups_6_5": (37, 61, (0, 3), None, {"ups_k_size": 6, "ups_preconcat_k_size": 5}),
    "arch_40x56_five_layers": (40, 56, (0, 3), None, _syn("48-1-linear-relu", "3-1-linear-none", "3-3-residual-relu",
                                                          "3-3-residual-relu", "3-3-residual-none")),
    "arch_40x56_3x3_first_layer": (40, 56, (0, 3), None, _syn("8-3-linear-relu", "3-1-linear-none",
                                                              linear_stabiliser_synth=0)),
    "arch_40x56_single_grid": (40, 56, (0, 0), None, None),
    "arch_17x33": (17, 33, (0, 4), None, None),
    "arch_129x7": (129, 7, (0, 3), None, None),
    "arch_1x1": (1, 1, (0, 1), None, None),
    "arch_45x70_nearest_2_5": (45, 70, (2, 5), "nearest", None),
}
# name -> (h, w, warp filter size): I, B, P in 8-bit RGB, smaller than the filter in both directions
GOPS = {"arch_gop3_7x9_sinc10": (7, 9, 10), "arch_gop3_7x9_sinc14": (7, 9, 14)}
OLDER = ["img_48x72_rgb_common_randomness", "img_50x70_rgb_final_bicubic", "img_44x60_yuv420_final_bilinear",
         "img_48x64_rgb_arm8_1hidden", "img_40x56_yuv444_10bit_arm24", "gop5_64x96_yuv420", "gop3_40x56_rgb",
         "gop3_48x72_yuv420_bilinear", "gop3_40x56_rgb_bicubic", "gop3_48x72_yuv420_sinc6", "gop4_40x56_rgb_sinc12"]


def save_npz(path, arrays):
    """np.savez_compressed with fixed member timestamps, so that a rerun writes the same bytes."""
    buf = io.BytesIO()
    with zipfile.ZipFile(buf, "w", zipfile.ZIP_DEFLATED) as z:
        for k in sorted(arrays):
            a = io.BytesIO()
            np.lib.format.write_array(a, np.asarray(arrays[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            z.writestr(info, a.getvalue())
    with open(path, "wb") as f:
        f.write(buf.getvalue())


def ref_decode(path):
    """-> (frames, raw outputs of every Cool-chic in coding order) from the unmodified reference."""
    import coolchic.bitstream.decode as ref

    raws = []
    orig = ref.encode_decode_coolchic

    def recording(*a, **k):
        out, b = orig(*a, **k)
        raws.append(out[0].detach().to(torch.float32).numpy().copy())
        return out, b

    ref.encode_decode_coolchic = recording
    try:
        frames = ref.decode_video(path, None, verbosity=0)
    finally:
        ref.encode_decode_coolchic = orig
    return frames, raws


def levels(frames):
    out = {}
    for k, fd in frames.items():
        M = 2**fd.bitdepth - 1
        if fd.frame_data_type == "yuv420":
            for c in "yuv":
                out[f"{k}_{c}"] = torch.round(fd.data[c][0, 0] * M).to(torch.int32).numpy().astype(np.uint16)
        else:
            out[k] = torch.round(fd.data[0] * M).to(torch.int32).numpy().astype(np.uint16)
    return out


def report(name, data, ints, raws):
    """The oracle's deviation from the reference: integer samples and raw outputs."""
    worst = nbad = 0
    for k, (fmt, bd, d) in pipeline.decode_video(data).items():
        M = 2**bd - 1
        for c in ("yuv" if fmt == "yuv420" else [None]):
            a = np.round((d[c] if c else d) * M).astype(np.int32)
            b = ints[f"{k}_{c}" if c else str(k)].astype(np.int32)
            worst = max(worst, int(np.abs(a - b).max()))
            nbad += int((a != b).sum())
    rest, i, raw_dev = data, 0, 0.0
    from coolchic_b200.bitstream.header import FrameHeader, VideoHeader

    rest = VideoHeader().read_header(rest)
    while rest and i < len(raws):
        f = FrameHeader()
        rest = f.read_header(rest)
        for _ in range(1 if f.get_value("frame_type") == "I" else 2):
            c = synth.CoolChicHeader()
            rest = c.read_header(rest)
            n_nn, n_lat = c.get_value("nn_n_bytes"), c.get_value("n_bytes_latent")
            o = pipeline.decode_coolchic(c, rest[:n_nn], rest[n_nn:n_nn + n_lat])
            raw_dev = max(raw_dev, float(np.abs(o - raws[i]).max()))
            rest = rest[n_nn + n_lat:]
            i += 1
    print(f"{name}: oracle vs reference: max level diff {worst}, differing samples {nbad}, "
          f"max raw |diff| {raw_dev:.3g}")


def main():
    be = pipeline.OracleBackend()
    ss = synth.SeedStream(be)
    streams = []
    for name, (h, w, lat, fin, ov) in IMAGES.items():
        streams.append((name, synth.make_image_stream(be, ss, h, w, "rgb", 8, lat, None, seed=6,
                                                      final_upsampling_type=fin, overrides=ov), ".npz"))
    for name, (h, w, fs) in GOPS.items():
        streams.append((name, synth.make_video_stream(be, ss, h, w, 3, "rgb", 8, fs, seed=6), "_frames.npz"))
    for name, data, suffix in streams:
        path = os.path.join(GOLD, name + ".cool")
        with open(path, "wb") as f:
            f.write(data)
        frames, raws = ref_decode(path)  # the reference decodes every one of them, 1x1 included
        ints = levels(frames)
        save_npz(os.path.join(GOLD, name + suffix), ints)
        save_npz(os.path.join(GOLD, name + "_raw.npz"), {f"c{i}": r for i, r in enumerate(raws)})
        report(name, data, ints, raws)
    for name in OLDER:
        path = os.path.join(GOLD, name + ".cool")
        frames, raws = ref_decode(path)
        gold = np.load(os.path.join(GOLD, name + (".npz" if name.startswith("img") else "_frames.npz")))
        ints = levels(frames)
        for k in gold.files:  # the committed integer samples are what the reference still decodes
            assert np.array_equal(gold[k], ints[k if k in ints else "0" if k == "rgb" else f"0_{k}"]), (name, k)
        save_npz(os.path.join(GOLD, name + "_raw.npz"), {f"c{i}": r for i, r in enumerate(raws)})
        report(name, open(path, "rb").read(), ints, raws)


if __name__ == "__main__":
    main()
