"""Quality analysis of a Cool-chic bitstream against its source: PSNR per plane and per frame, rate, and the
prediction statistics of P / B frames, with the reference encoder's column names.

    python cc_eval.py -i <bitstream.cool> --original <src.yuv|png|ppm> [--frame_offset N] [--ms_ssim] [--maps out.npz]
                      [--grids] [--device N]

Display frame i is compared with source frame frame_offset + i.  ``--maps`` writes, per frame, the error map
(sum over planes of the squared integer errors / (2^b - 1)^2, chroma at (y >> 1, x >> 1) for 4:2:0) and for P / B
frames the alpha, beta and prediction maps.  ``--ms_ssim`` appends MS-SSIM columns (whole frame, in dB, per plane;
``n/a`` for a frame with a plane smaller than 176 x 176) and a mean line, and with ``--maps`` the scale-0 SSIM map of
every plane.  ``--grids`` appends, per frame and per Cool-chic, a table of its latent grids: size, model bits and bpp,
the frame PSNR with the grid alone read as zeros and its change from the decoded frame's, and for the residue the PSNR
with only the synthesis grids from the coarsest down to that one kept (DESIGN §4.7).  The grid analysis decodes the
bitstream a second time, after the quality table.
"""
import argparse

import numpy as np

import coolchic_b200  # noqa: F401  (import alias of the cool-chic_b200/ package)
from coolchic_b200.bitstream.grids import video_grid_analysis
from coolchic_b200.bitstream.quality import video_quality

COLUMNS = ["frame_idx", "frame_type", "psnr_db", "psnr_y_db", "psnr_u_db", "psnr_v_db", "rate_bpp", "alpha_mean",
           "beta_mean", "pred_psnr_db", "dummy_pred_psnr_db"]
MS_SSIM_COLUMNS = ["ms_ssim", "ms_ssim_db", "ms_ssim_y", "ms_ssim_u", "ms_ssim_v"]
GRID_COLUMNS = ["grid", "size", "hyper", "bits", "bpp", "drop_psnr_db", "drop_delta_db", "coarse_psnr_db"]


def _fmt(v):
    return "n/a" if v is None else f"{v:.6f}"


if __name__ == "__main__":
    parser = argparse.ArgumentParser()
    parser.add_argument("--input", "-i", type=str, required=True, help="Bitstream path.")
    parser.add_argument("--original", type=str, required=True, help="Source file (.yuv, .png, .ppm).")
    parser.add_argument("--frame_offset", type=int, default=0, help="Source frame of the first displayed frame.")
    parser.add_argument("--maps", type=str, default=None, help="Write the error / alpha / beta / prediction maps here (.npz).")
    parser.add_argument("--ms_ssim", action="store_true", help="Also report MS-SSIM.")
    parser.add_argument("--grids", action="store_true", help="Also report what each latent grid costs and buys.")
    parser.add_argument("--device", type=int, help="CUDA device ordinal.", default=0)
    args = parser.parse_args()

    with open(args.input, "rb") as f_in:
        frames = video_quality(f_in.read(), args.original, frame_offset=args.frame_offset, device=args.device,
                               want_maps=args.maps is not None, ms_ssim=args.ms_ssim)
    columns = COLUMNS + (MS_SSIM_COLUMNS if args.ms_ssim else [])
    print(" ".join(f"{c:<18}" for c in columns))
    for key, q in frames.items():
        vals = [key, q.frame_type] + [_fmt(getattr(q, c)) for c in columns[2:]]
        print(" ".join(f"{v:<18}" for v in vals))
    n_bits = 8 * sum(q.n_bytes for q in frames.values())
    n_pixels = sum(q.img_size[0] * q.img_size[1] for q in frames.values())
    mean_psnr = sum(q.psnr_db for q in frames.values()) / len(frames)
    print(f"mean psnr_db {mean_psnr:.6f}  total rate_bpp {n_bits / n_pixels:.6f}  ({len(frames)} frames)")
    if args.ms_ssim:
        have = [q.ms_ssim for q in frames.values() if q.ms_ssim is not None]
        print(f"mean ms_ssim {_fmt(sum(have) / len(have) if have else None)}  ({len(have)} of {len(frames)} frames)")
    if args.maps:
        maps = {}
        for key, q in frames.items():
            maps[f"frame{key}_error"] = q.error_map.cpu().numpy()
            for name in ("alpha", "beta", "pred"):
                t = getattr(q, f"{name}_map")
                if t is not None:
                    maps[f"frame{key}_{name}"] = t.cpu().numpy()
            for plane, t in zip("yuv", q.ssim_maps or []):
                maps[f"frame{key}_ssim_{plane}"] = t.cpu().numpy()
        np.savez_compressed(args.maps, **maps)
    if args.grids:
        with open(args.input, "rb") as f_in:
            grids = video_grid_analysis(f_in.read(), args.original, frame_offset=args.frame_offset, device=args.device)
        for key, fg in grids.items():
            for name, rows in fg.coolchics.items():
                print(f"grids frame {key} {fg.frame_type} {name} psnr_db {fg.psnr_db:.6f}")
                print(" ".join(f"{c:<18}" for c in GRID_COLUMNS))
                for r in rows:
                    vals = [r.grid, f"{r.size[0]}x{r.size[1]}", int(r.is_hyper)] + [
                        _fmt(v) for v in (r.bits, r.bpp, r.drop_psnr_db, r.drop_delta_db, r.coarse_psnr_db)]
                    print(" ".join(f"{v:<18}" for v in vals))
