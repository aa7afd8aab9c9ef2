"""Whole-stream decode with the CPU oracle (video loop + frame reconstruction), and an
oracle-backed stand-in for the device context so that coolchic_b200.synth can fabricate
streams on a machine without a GPU.   TEST INFRASTRUCTURE ONLY."""
import numpy as np
import torch

import ccoracle


class OracleBackend:
    """Same methods as coolchic_b200._native.Context, computed by the oracle (the raw output only)."""

    def synthesize(self, descs, nn_ints, latents, zero_grids):
        outs = []
        for d, nn, lat, z in zip(descs, nn_ints, latents, zero_grids):
            assert z == 0
            outs.append(torch.from_numpy(ccoracle.synthesize(d, nn, np.asarray(lat.cpu().numpy(), np.int8)))[None])
        return outs

    def decode_nn(self, desc, nn_bytes):
        return ccoracle.decode_nn(desc, nn_bytes)

    def decode_latents(self, desc, nn, payload):
        lat, _ = ccoracle.decode_latents(desc, nn, payload)
        return torch.from_numpy(lat)

    def encode_latents(self, desc, nn, latents=None, seed=None):
        if latents is None:
            lat, payload = ccoracle.sample_latents(desc, nn, seed)
            return torch.from_numpy(lat), payload, 0
        lat = latents.cpu().numpy().astype(np.int8)
        return torch.from_numpy(lat), ccoracle.encode_latents(desc, nn, lat), 0


def decode_coolchic(header, nn_bytes, payload):
    from coolchic_b200._desc import desc_from_header

    d = desc_from_header(header)
    nn = ccoracle.decode_nn(d, nn_bytes)
    lat, _ = ccoracle.decode_latents(d, nn, payload)
    return ccoracle.synthesize(d, nn, lat)


def decode_video(data: bytes):
    """-> {display_index: (frame_data_type, bitdepth, array or dict)} following bitstream/decode.py:26-212."""
    from coolchic_b200.bitstream.header import CoolChicHeader, FrameHeader, VideoHeader

    v = VideoHeader()
    rest = v.read_header(data)
    cs = v.get_coding_structure()
    frames = {}
    for coding_idx in range(cs.get_max_coding_order() + 1):
        f = FrameHeader()
        rest = f.read_header(rest)
        ftype, fmt, bd = f.get_value("frame_type"), f.get_value("frame_data_type"), f.get_value("bitdepth")
        outs = {}
        for name in ["residue"] + (["motion"] if ftype in ("P", "B") else []):
            c = CoolChicHeader()
            rest = c.read_header(rest)
            n_nn, n_lat = c.get_value("nn_n_bytes"), c.get_value("n_bytes_latent")
            outs[name] = decode_coolchic(c, rest[:n_nn], rest[n_nn:n_nn + n_lat])
            rest = rest[n_nn + n_lat:]
        if ftype == "I":
            raw = outs["residue"]
        else:
            refs = []
            for idx in f.get_value("index_references"):
                _, _, rd = frames[idx]
                if fmt == "yuv420":  # convert_420_to_444: nearest x2 (io/format/yuv.py:303-316)
                    u = np.repeat(np.repeat(rd["u"], 2, axis=0), 2, axis=1)
                    vv = np.repeat(np.repeat(rd["v"], 2, axis=0), 2, axis=1)
                    refs.append(np.stack([rd["y"], u, vv]))
                else:
                    refs.append(rd)
            raw = ccoracle.inter_predict(outs["residue"], outs["motion"], refs[0], refs[1] if ftype == "B" else None,
                                         f.get_value("global_flow"), f.get_value("warp_filter_size"))
        frames[f.get_value("display_index")] = (fmt, bd, ccoracle.finish_frame(raw, bd, fmt))
    return frames
