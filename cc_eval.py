"""Quality analysis of a Cool-chic bitstream against its source: PSNR per plane and per frame, rate, and the
prediction statistics of P / B frames, with the reference encoder's column names.

    python cc_eval.py -i <bitstream.cool> --original <src.yuv|png|ppm> [--frame_offset N] [--ms_ssim] [--vif] [--psnr_hvs]
                      [--maps out.npz]
                      [--grids] [--motion] [--device N]

Display frame i is compared with source frame frame_offset + i.  ``--maps`` writes, per frame, the error map
(sum over planes of the squared integer errors / (2^b - 1)^2, chroma at (y >> 1, x >> 1) for 4:2:0) and for P / B
frames the alpha, beta and prediction maps.  ``--ms_ssim`` appends MS-SSIM columns (whole frame, in dB, per plane;
``n/a`` for a frame with a plane smaller than 176 x 176) and a mean line, and with ``--maps`` the scale-0 SSIM map of
every plane.  ``--vif`` appends VIF columns (whole frame and per plane; ``n/a`` for a frame with a plane smaller than
41 x 41 or a flat source plane) and a mean line.  ``--psnr_hvs`` appends PSNR-HVS and PSNR-HVS-M columns (whole
frame, and PSNR-HVS-M per plane; ``n/a`` for a frame with a plane smaller than 8 x 8) and a mean line, and with
``--maps`` each plane's block map of S_hvs_m / 64 / 255^2.  ``--grids`` appends, per frame and per Cool-chic, a table of its latent grids: size, model bits and bpp,
the frame PSNR with the grid alone read as zeros and its change from the decoded frame's, and for the residue the PSNR
with only the synthesis grids from the coarsest down to that one kept (DESIGN §4.7).  The grid analysis decodes the
bitstream a second time, after the quality table.
``--motion`` appends, for every P / B frame, a table of its variants (DESIGN §4.9): the frame with every motion
channel zeroed (no_local_motion), with the global flow zeroed too (no_motion), predicted from one reference only (B:
ref0_only, ref1_only), without the residue (no_residue) and without the prediction (no_prediction), each with its PSNR,
per plane, and its change from the decoded frame's; then one line of flow statistics per reference.  With ``--maps``
it also writes the total displacement of every reference, ``frame<k>_flow<r>`` ([2, H, W]).
"""
import argparse

import numpy as np

import coolchic_b200  # noqa: F401  (import alias of the cool-chic_b200/ package)
from coolchic_b200.bitstream.grids import video_grid_analysis
from coolchic_b200.bitstream.motion import variants_of
from coolchic_b200.bitstream.quality import video_quality

COLUMNS = ["frame_idx", "frame_type", "psnr_db", "psnr_y_db", "psnr_u_db", "psnr_v_db", "rate_bpp", "alpha_mean",
           "beta_mean", "pred_psnr_db", "dummy_pred_psnr_db"]
MS_SSIM_COLUMNS = ["ms_ssim", "ms_ssim_db", "ms_ssim_y", "ms_ssim_u", "ms_ssim_v"]
VIF_COLUMNS = ["vif", "vif_y", "vif_u", "vif_v"]
HVS_COLUMNS = ["psnr_hvs_db", "psnr_hvs_m_db", "psnr_hvs_m_y_db", "psnr_hvs_m_u_db", "psnr_hvs_m_v_db"]
MOTION_COLUMNS = ["variant", "psnr_db", "psnr_y_db", "psnr_u_db", "psnr_v_db", "delta_db"]
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
    parser.add_argument("--vif", action="store_true", help="Also report VIF (visual information fidelity).")
    parser.add_argument("--psnr_hvs", action="store_true", help="Also report PSNR-HVS and PSNR-HVS-M.")
    parser.add_argument("--grids", action="store_true", help="Also report what each latent grid costs and buys.")
    parser.add_argument("--motion", action="store_true", help="Also report what the motion, each reference and the "
                        "residue of every P / B frame buy.")
    parser.add_argument("--device", type=int, help="CUDA device ordinal.", default=0)
    args = parser.parse_args()

    with open(args.input, "rb") as f_in:
        frames = video_quality(f_in.read(), args.original, frame_offset=args.frame_offset, device=args.device,
                               want_maps=args.maps is not None, ms_ssim=args.ms_ssim, motion=args.motion,
                               vif=args.vif, psnr_hvs=args.psnr_hvs)
    columns = (COLUMNS + (MS_SSIM_COLUMNS if args.ms_ssim else []) + (VIF_COLUMNS if args.vif else [])
               + (HVS_COLUMNS if args.psnr_hvs else []))
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
    if args.vif:
        have = [q.vif for q in frames.values() if q.vif is not None]
        print(f"mean vif {_fmt(sum(have) / len(have) if have else None)}  ({len(have)} of {len(frames)} frames)")
    if args.psnr_hvs:
        have = [q for q in frames.values() if q.hvs_planes is not None]
        mean = {c: _fmt(sum(getattr(q, c) for q in have) / len(have) if have else None) for c in HVS_COLUMNS[:2]}
        print(f"mean psnr_hvs_db {mean['psnr_hvs_db']}  psnr_hvs_m_db {mean['psnr_hvs_m_db']}  ({len(have)} of "
              f"{len(frames)} frames)")
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
            for plane, t in zip("yuv", q.hvs_maps or []):
                maps[f"frame{key}_hvs_{plane}"] = t.cpu().numpy()
            for r, ref in enumerate(q.motion.refs if q.motion is not None else []):
                maps[f"frame{key}_flow{r}"] = ref.flow_map.cpu().numpy()
        np.savez_compressed(args.maps, **maps)
    if args.motion:
        for key, q in frames.items():
            m = q.motion
            if m is None:
                continue
            print(f"motion frame {key} {q.frame_type} psnr_db {q.psnr_db:.6f}")
            print(" ".join(f"{c:<18}" for c in MOTION_COLUMNS))
            for v in variants_of(q.frame_type):
                vals = [v] + [_fmt(x) for x in [m.psnr_db(v)] + m.plane_psnr_db(v) + [m.delta_db(v)]]
                print(" ".join(f"{x:<18}" for x in vals))
            for r, ref in enumerate(m.refs):
                print(f"ref{r} global_flow {ref.global_flow[0]} {ref.global_flow[1]}  mean_flow {ref.mean_flow[0]:.6f} "
                      f"{ref.mean_flow[1]:.6f}  mean_local {ref.mean_local:.6f}  max_local {ref.max_local:.6f}  "
                      f"outside {ref.outside} ({100 * ref.outside_fraction:.2f} %)")
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
