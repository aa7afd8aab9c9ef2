"""Lossless bitstream optimisation: retune the ARM and IFCE integers of every Cool-chic for the exact coded rate and
rewrite the bitstream; every decoded sample is unchanged (``coolchic_b200.bitstream.optimize``).

    python cc_optimize.py -i in.cool -o out.cool [--max_rounds N] [--time_budget S] [--device D]
"""
import argparse

import coolchic_b200  # noqa: F401  (import alias of the cool-chic_b200/ package)
from coolchic_b200.bitstream.optimize import optimize_bitstream


def main():
    p = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    p.add_argument("-i", "--input", required=True)
    p.add_argument("-o", "--output", required=True)
    p.add_argument("--max_rounds", type=int, default=8)
    p.add_argument("--time_budget", type=float, default=None, help="seconds; no new search round starts after it")
    p.add_argument("--device", type=int, default=0)
    a = p.parse_args()
    data = open(a.input, "rb").read()
    out, rep = optimize_bitstream(data, device=a.device, max_rounds=a.max_rounds, time_budget_s=a.time_budget)
    with open(a.output, "wb") as f:
        f.write(out)
    for fr in rep.frames:
        for c in fr.coolchics:
            print(f"frame {fr.coding_idx} {fr.frame_type} {c.name}: {c.bytes_before} -> {c.bytes_after} bytes "
                  f"(NN {c.nn_bytes_before} -> {c.nn_bytes_after}, latents {c.latent_bytes_before} -> "
                  f"{c.latent_bytes_after}){' kept' if c.kept_original else ''}")
            print(f"    latent model bits {c.latent_bits_before:.1f} -> {c.latent_bits_after:.1f}; saved: ARM "
                  f"{c.arm_bits_saved:.1f}, IFCE {c.ifce_bits_saved:.1f}, exp-Golomb recount {c.recount_bits_saved}, "
                  f"bias reset {c.bias_reset_bits_saved} bits; {c.rounds} rounds, {c.candidates} candidates, "
                  f"{c.seconds:.2f} s")
    print(f"total {rep.bytes_before} -> {rep.bytes_after} bytes ({rep.bytes_before - rep.bytes_after} saved) "
          f"in {rep.seconds:.2f} s")


if __name__ == "__main__":
    main()
