"""Generate the source-reader fixtures: copies a few source files of the reference checkout's test/data/ into
tests/golden/ and stores, for every frame of each, what the UNMODIFIED reference's load_frame_data_from_file returns,
as integer samples (tests/golden/originals_frames.npz, key "<file>/<frame>/<plane>").  It checks on the way that the
reference's float values are fp32(k) / fp32(2^b - 1) of those integers, so the integers pin the floats bit for bit.
Needs a reference checkout (COOLCHIC_REFERENCE=<path>).  TEST INFRASTRUCTURE ONLY.

    python oracle/gen_golden_originals.py
"""
import os
import shutil
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ["COOLCHIC_REFERENCE"]
sys.path.insert(0, os.path.join(HERE, "refshim"))
sys.path.insert(0, REF)

import torch  # noqa: E402

GOLD = os.path.join(HERE, "..", "tests", "golden")
FILES = {  # file name -> number of frames
    "kodim15_192x128_01p_yuv420_10b.yuv": 1,
    "kodim15_192x128_01p_yuv444_8b.yuv": 1,
    "192x128_kodim15.png": 1,
    "D-BQSquare-3frames_224x128_60p_yuv420_8b.yuv": 3,
}


def main():
    from coolchic.io.io import load_frame_data_from_file

    out = {}
    for name, n_frames in FILES.items():
        src = os.path.join(REF, "test", "data", name)
        dst = os.path.join(GOLD, name)
        shutil.copyfile(src, dst)
        for i in range(n_frames):
            fd = load_frame_data_from_file(dst, i)
            M = 2**fd.bitdepth - 1
            planes = [(c, fd.data[c][0, 0]) for c in "yuv"] if fd.frame_data_type == "yuv420" else \
                [(str(c), fd.data[0, c]) for c in range(3)]
            for c, t in planes:
                k = torch.round(t * M).to(torch.int32)
                assert torch.equal(k.to(torch.float32) / np.float32(M), t), (name, i, c)
                out[f"{name}/{i}/{c}"] = k.numpy().astype(np.uint16)
            out[f"{name}/{i}/meta"] = np.array([fd.bitdepth, *fd.img_size], dtype=np.int32)
            out[f"{name}/{i}/type"] = np.array(fd.frame_data_type)
    np.savez_compressed(os.path.join(GOLD, "originals_frames.npz"), **out)


if __name__ == "__main__":
    main()
