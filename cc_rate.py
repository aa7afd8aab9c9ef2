"""Rate analysis of a Cool-chic bitstream: where the bits go, per frame, per latent grid and per network module.

    python cc_rate.py -i <bitstream.cool> [--maps out.npz] [--model] [--device N]

Latent bits are the information content of every decoded symbol under the model the range coder used
(``coolchic_b200.bitstream.rate``); they are not the encoder's training rate proxy.  ``--maps`` writes, per
Cool-chic, the per-grid bit maps, the mu / scale maps the coder used and the per-pixel spatial rate map.  ``--model``
appends what the ARM's context, the IFCE, the hyperlatents and the scale calibration are worth
(``coolchic_b200.bitstream.model``).
"""
import argparse

import numpy as np

import coolchic_b200  # noqa: F401  (import alias of the cool-chic_b200/ package)
from coolchic_b200.bitstream.header import NN_MODULES
from coolchic_b200.bitstream.model import video_model_analysis
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


def print_model(f):
    """The entropy-model analysis of one frame (DESIGN §4.10); n/a where a variant does not exist."""
    def col(c, name, g):
        return f"{c.variants[name][g]:>12.1f}" if name in c.variants else f"{'n/a':>12}"

    def net(v):
        return f"{v:+.1f} bits" if v is not None else "n/a"

    for name, c in f.coolchics.items():
        print(f"  {name} entropy model:")
        print(f"    {'grid':>4} {'size':>11} {'hyper':>5} {'decoded':>12} {'static':>12} {'no_ifce':>12} {'no_hyper':>12}"
              f" {'no_context':>12} {'best d':>6} {'sigma x':>7} {'calibrated':>12}")
        for g, ((gh, gw), hyp) in enumerate(zip(c.grid_sizes, c.grid_is_hyper)):
            off, bits = c.best_offset[g]
            print(f"    {g:>4} {f'{gw}x{gh}':>11} {'yes' if hyp else '':>5} {col(c, 'decoded', g)} {c.static_bits[g]:>12.1f}"
                  f" {col(c, 'no_ifce', g)} {col(c, 'no_hyper', g)} {col(c, 'no_context', g)} {off:>6}"
                  f" {np.exp(off / 256):>7.3f} {bits:>12.1f}")
        off, bits = c.best_offset_all
        print(f"    one offset for all grids: {off} (sigma x {np.exp(off / 256):.3f}) saves "
              f"{c.total('decoded') - bits:.1f} bits")
        print("    ctx_k bits, k = 0 .. n_ctx: " + " ".join(f"{b:.1f}" for b in c.ctx_curve))
        print(f"    ARM net (no_context - decoded - ARM NN bits): {net(c.arm_net)}")
        print(f"    IFCE net (no_ifce - decoded - IFCE NN bits): {net(c.ifce_net)}")
        print(f"    hyperlatent net (no_hyper over synthesis grids - hyperlatent bits): {net(c.hyper_net)}")


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--input", "-i", type=str, required=True, help="Bitstream path.")
    parser.add_argument("--maps", type=str, default=None, help="Write the rate / mu / scale maps to this .npz file.")
    parser.add_argument("--model", action="store_true",
                        help="Also report what the ARM's context, the IFCE, the hyperlatents and the scale calibration "
                             "are worth, per frame and Cool-chic.")
    parser.add_argument("--device", type=int, help="CUDA device ordinal.", default=0)
    args = parser.parse_args()

    with open(args.input, "rb") as f_in:
        data = f_in.read()
    frames = video_rate(data, device=args.device)
    models = video_model_analysis(data, device=args.device) if args.model else {}
    maps = {}
    for key, fr in frames.items():
        print_frame(key, fr)
        if args.model:
            print_model(models[key])
        for name, c in fr.coolchics.items():
            p = f"frame{key}_{name}"
            maps[f"{p}_spatial_rate_bit"] = c.spatial_rate_bit[0, 0].cpu().numpy()
            for g in range(len(c.grid_sizes)):
                maps[f"{p}_grid{g}_rate_bit"] = c.rate_bit[g][0, 0].cpu().numpy()
                maps[f"{p}_grid{g}_mu"] = c.mu[g][0, 0].cpu().numpy()
                maps[f"{p}_grid{g}_scale"] = c.scale[g][0, 0].cpu().numpy()
    if args.maps:
        np.savez_compressed(args.maps, **maps)
