"""Per-Cool-chic decode operator.

Mirror of the reference's ``coolchic/bitstream/component/coolchic.py:29-207``
(``encode_decode_coolchic(mode="decode")``): same signature, same errors, same return value
(raw, un-clamped, un-rounded float32 synthesis output ``[1, C, H, W]``) -- but every stage
(NN parsing, integer ARM + IFCE, range decoding, upsampling, synthesis, final resize) runs in
``libccdec.so`` on the GPU.  ``CoolChicDecoder`` is the module-style wrapper (``load`` /
``forward``) named in BASELINE.json; the reference itself has no such class (SURVEY F2).
"""
from typing import List, Literal, Optional, Sequence, Tuple

import torch
from torch import Tensor

from .. import _native
from .._desc import CcdCoolChicDesc, desc_from_header
from .header import CoolChicHeader


def encode_decode_coolchic(
    header: CoolChicHeader,
    bytes_nn: bytes,
    mode: Literal["encode", "decode"],
    dec_bytes_latent: Optional[bytes] = None,
    enc_quantized_latent: Optional[List[Tensor]] = None,
    verbosity: int = 0,
    device: int = 0,
) -> Tuple[Tensor, Optional[bytes]]:
    """Decode one Cool-chic.  Returns ``(synthesis_output [1, C, H, W] float32 CUDA, None)``."""
    if mode == "encode":
        # the encoder side of the reference operator is out of scope of the decode drop-in;
        # the device range encoder is exposed separately (coolchic_b200.synth)
        if enc_quantized_latent is None:
            raise ValueError(
                "Trying to encode cool_chic latent without indicating the quantized latent value. "
                "Found enc_quantized_latent=None. It should be a list of integer Tensor."
            )
        raise NotImplementedError("mode='encode' is not part of the decode drop-in; see coolchic_b200.synth")
    if mode != "decode":
        raise ValueError(f"Unknown mode {mode}")
    if dec_bytes_latent is None:
        raise ValueError(
            "Trying to encode cool_chic latent with dec_bytes_latent=None. "
            "The argument dec_bytes_latent should represent the bytes of the bitstream."
        )
    dec = CoolChicDecoder(device=device).load(header, bytes_nn, dec_bytes_latent)
    out = dec.forward()
    if verbosity:
        print(header.pretty_string())
    if verbosity >= 2:
        # the reference's per-stage line (component/coolchic.py:199-205): seconds spent on the NN weights, the IFCE
        # contexts, the latents (IFCE included) and upsampling + synthesis.  Here: host parse of the NN payload + staging
        # + H2D | 0 (the IFCE layer is evaluated on the fly inside the entropy kernel) | entropy kernel | float-tail kernels
        t = dec.last_timing
        time_neural_net, time_ifce = t["upload_ms"] / 1e3, 0.0
        time_latent, time_syn = t["entropy_ms"] / 1e3, t["synthesis_ms"] / 1e3
        print(f"{time_neural_net:6.2f} {time_ifce:6.2f} {time_latent:6.2f} {time_syn:6.2f} ")
    return out, None


class CoolChicDecoder:
    """``load(header, bytes_nn, bytes_latent)`` then ``forward() -> Tensor[1, C, H, W]``."""

    def __init__(self, device: int = 0):
        self.device = device
        self.desc: Optional[CcdCoolChicDesc] = None
        self._nn: Optional[bytes] = None
        self._lat: Optional[bytes] = None
        self.latents: Optional[Tensor] = None
        self.last_timing = {}

    def load(self, header: CoolChicHeader, bytes_nn: bytes, bytes_latent: bytes) -> "CoolChicDecoder":
        if bytes_nn is None or bytes_latent is None:
            raise ValueError("CoolChicDecoder.load: bytes_nn and bytes_latent must be bytes objects")
        n_nn, n_lat = header.get_value("nn_n_bytes"), header.get_value("n_bytes_latent")
        if len(bytes_nn) < n_nn or len(bytes_latent) < n_lat:
            raise ValueError(
                f"Cool-chic payload truncated: header announces {n_nn} NN bytes and {n_lat} latent bytes, "
                f"got {len(bytes_nn)} and {len(bytes_latent)}."
            )
        self.desc = desc_from_header(header)
        self._nn = bytes(bytes_nn[:n_nn])
        self._lat = bytes(bytes_latent[:n_lat])
        return self

    @torch.no_grad()
    def forward(self, want_latents: bool = False) -> Tensor:
        if self.desc is None:
            raise RuntimeError("CoolChicDecoder.forward called before load()")
        ctx = _native.get_context(self.device)
        if want_latents:
            out, self.latents = ctx.decode_coolchic(self.desc, self._nn, self._lat, want_latents=True)
        else:
            out = ctx.decode_coolchic(self.desc, self._nn, self._lat)
        self.last_timing = ctx.last_timing()
        return out

    __call__ = forward


def decode_coolchics(headers: Sequence[CoolChicHeader], bytes_nn: Sequence[bytes], bytes_latent: Sequence[bytes],
                     device: int = 0, finish=None) -> List[Tensor]:
    """Decode several independent Cool-chics CONCURRENTLY (one persistent CTA per stream).  ``finish[i]`` =
    (bitdepth, frame_data_type) for the Cool-chic of an I frame: libccdec then returns the finished frame
    (decode.py:191-206 applied) instead of the raw output."""
    ctx = _native.get_context(device)
    descs = [desc_from_header(h) for h in headers]
    outs, _ = ctx.decode_many(descs, [bytes(b) for b in bytes_nn], [bytes(b) for b in bytes_latent], finish=finish)
    return outs
