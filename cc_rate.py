"""Rate analysis of a Cool-chic bitstream: where the bits go, per frame, per latent grid and per network module.

    python cc_rate.py -i <bitstream.cool> [--maps out.npz] [--device N]

Latent bits are the information content of every decoded symbol under the model the range coder used
(``coolchic_b200.bitstream.rate``); they are not the encoder's training rate proxy.  ``--maps`` writes, per
Cool-chic, the per-grid bit maps, the mu / scale maps the coder used and the per-pixel spatial rate map.
"""
import argparse

import numpy as np

import coolchic_b200  # noqa: F401  (import alias of the cool-chic_b200/ package)
from coolchic_b200.bitstream.header import NN_MODULES
from coolchic_b200.bitstream.rate import video_rate


def print_frame(key, f):
    h, w = f.img_size
    print(f"frame {key:<4} {f.frame_type}  {w}x{h}  {f.n_bytes} bytes = {8 * f.n_bytes} bits "
          f"({8 * f.n_bytes / (h * w):.4f} bpp); frame header {f.header_bits} bits")
    for name, c in f.coolchics.items():
        print(f"  {name}: header {c.header_bits}  NN payload {c.nn_payload_bits}  latent payload {c.latent_payload_bits}"
              f"  total {c.total_bits} bits")
        print(f"    {'grid':>4} {'size':>11} {'hyper':>5} {'bits':>14} {'bpp':>9}")
        for g, ((gh, gw), hyp, b, bpp) in enumerate(zip(c.grid_sizes, c.grid_is_hyper, c.grid_bits, c.grid_bpp)):
            print(f"    {g:>4} {f'{gw}x{gh}':>11} {'yes' if hyp else '':>5} {b:>14.2f} {bpp:>9.5f}")
        gap = c.latent_payload_bits - c.latent_model_bits
        print(f"    model bits {c.latent_model_bits:.2f} vs payload bits {c.latent_payload_bits}: "
              f"{gap:.2f} bits of range-coder seal and scale truncation")
        nn = "  ".join(f"{m} {c.nn_bits[m]['weight']}+{c.nn_bits[m]['bias']}" for m in NN_MODULES)
        print(f"    NN bits (weight+bias): {nn}  pad {c.nn_pad_bits}")


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--input", "-i", type=str, required=True, help="Bitstream path.")
    parser.add_argument("--maps", type=str, default=None, help="Write the rate / mu / scale maps to this .npz file.")
    parser.add_argument("--device", type=int, help="CUDA device ordinal.", default=0)
    args = parser.parse_args()

    with open(args.input, "rb") as f_in:
        frames = video_rate(f_in.read(), device=args.device)
    maps = {}
    for key, fr in frames.items():
        print_frame(key, fr)
        for name, c in fr.coolchics.items():
            p = f"frame{key}_{name}"
            maps[f"{p}_spatial_rate_bit"] = c.spatial_rate_bit[0, 0].cpu().numpy()
            for g in range(len(c.grid_sizes)):
                maps[f"{p}_grid{g}_rate_bit"] = c.rate_bit[g][0, 0].cpu().numpy()
                maps[f"{p}_grid{g}_mu"] = c.mu[g][0, 0].cpu().numpy()
                maps[f"{p}_grid{g}_scale"] = c.scale[g][0, 0].cpu().numpy()
    if args.maps:
        np.savez_compressed(args.maps, **maps)
