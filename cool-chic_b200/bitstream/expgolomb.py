"""exp-Golomb(k) coding of the neural-network integers -- host-side mirror of the reference's
``coolchic/bitstream/neuralnet/expgolomb.py`` (``encode_exp_golomb`` :15-71,
``decode_exp_golomb`` :74-130), working on Python ints instead of strings of bits.  The
decoder used on the hot path is the C++ one in libccdec (``ccd_decode_nn``); this module is
the WRITER side (synthetic streams) plus a small pure-Python reader used by the tests."""
from typing import List, Sequence, Tuple


def encode_exp_golomb(data: Sequence[int], count: Sequence[int]) -> Tuple[bytes, int]:
    """Returns (payload, n_padding_bits); the padding bits are a PREFIX (expgolomb.py:64-67)."""
    if len(data) != len(count):
        raise ValueError(
            f"Each data to write must have its exp-golomb count parameter. Found {len(data)} "
            f"data to write and {len(count)} exp-golomb count parameters."
        )
    if len(count) and min(count) < 0:
        raise ValueError(f"Exp-golomb count should be >= 0. Found min(count) = {min(count)}")
    acc, n_bits = 0, 0
    for x, k in zip(data, count):
        x = int(x)
        u = -2 * x if x <= 0 else 2 * x - 1       # sign in the least significant bit
        v = u + (1 << k)                          # order-0 code of u + 2^k - 1, i.e. binary of (u + 2^k)
        length = v.bit_length()
        total = 2 * length - 1 - k                # (length-1) zeros + length bits, minus k leading zeros
        acc = (acc << total) | v
        n_bits += total
    pad = (8 - n_bits % 8) % 8
    return acc.to_bytes((n_bits + pad) // 8, "big"), pad


def exp_golomb_bits(data: Sequence[int], count: Sequence[int]) -> List[int]:
    """Length in bits of the exp-Golomb(k) codeword of each integer (the ``total`` of encode_exp_golomb)."""
    out = []
    for x, k in zip(data, count):
        x = int(x)
        u = -2 * x if x <= 0 else 2 * x - 1
        out.append(2 * (u + (1 << k)).bit_length() - 1 - k)
    return out


def decode_exp_golomb(data_bytes: bytes, n_padding_bits: int, count: Sequence[int]) -> List[int]:
    if isinstance(n_padding_bits, float):
        raise TypeError(f"n_padding_bits must be an int. Found n_padding_bits={n_padding_bits}")
    if len(count) and min(count) < 0:
        raise ValueError(f"Exp-golomb count should be >= 0. Found min(count) = {min(count)}")
    n_bits = 8 * len(data_bytes)
    v = int.from_bytes(data_bytes, "big")
    pos = n_padding_bits

    def take(n: int) -> int:
        nonlocal pos
        if pos + n > n_bits:
            raise ValueError("exp-Golomb payload truncated")
        out = (v >> (n_bits - pos - n)) & ((1 << n) - 1)
        pos += n
        return out

    out = []
    for k in count:
        z = 0
        while take(1) == 0:
            z += 1
        q = ((1 << z) | take(z)) - 1 if z else 0
        r = take(k) if k else 0
        val = (q << k) + r
        out.append((val + 1) // 2 if val & 1 else -(val // 2))
    return out
