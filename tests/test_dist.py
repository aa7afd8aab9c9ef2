"""world_size-2 gloo test (CPU) of the frame-sharding plumbing used by bench.py --gpus N."""
import os
import socket
import sys

import torch.multiprocessing as mp
from conftest import ROOT


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, ret):
    sys.path.insert(0, os.path.abspath(ROOT))
    import torch.distributed as dist

    import coolchic_b200  # noqa: F401
    from coolchic_b200.dist import broadcast_byte_strings, gather_sharded, shard_indices

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    items = [bytes([i]) * (10 + 7 * i) for i in range(5)] if rank == 0 else None
    got = broadcast_byte_strings(items, src=0)
    mine = shard_indices(len(got), rank, world)
    merged = gather_sharded({i: len(got[i]) for i in mine}, world)
    part = broadcast_byte_strings(items, src=0, want=mine)  # only this rank's share is cut out of the buffer
    ok_part = all((part[i] == bytes([i]) * (10 + 7 * i)) if i in mine else part[i] is None for i in range(5))
    empty = broadcast_byte_strings([b"", b"x"] if rank == 0 else None, src=0)
    ret[rank] = (got == [bytes([i]) * (10 + 7 * i) for i in range(5)] and ok_part and empty == [b"", b"x"], mine, merged)
    dist.destroy_process_group()


def test_broadcast_and_shard_two_ranks():
    world, port = 2, _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_worker, args=(world, port, ret), nprocs=world, join=True)
    assert ret[0][0] and ret[1][0]
    assert ret[0][1] == [0, 2, 4] and ret[1][1] == [1, 3]
    assert ret[0][2] == ret[1][2] == {i: 10 + 7 * i for i in range(5)}


def test_shard_indices_cover_everything():
    sys.path.insert(0, os.path.abspath(ROOT))
    import coolchic_b200  # noqa: F401
    from coolchic_b200.dist import shard_indices

    for n in (1, 7, 24, 32):
        for w in (1, 2, 4, 8):
            allidx = sorted(i for r in range(w) for i in shard_indices(n, r, w))
            assert allidx == list(range(n))


def _gop_worker(rank, world, port, ret):
    """decode_video_bytes under a 2-rank gloo group with stand-in decode / reconstruct functions: every rank
    decodes only the Cool-chics of the frames it owns, reconstructs those frames, and ends up with all frames
    after the exchange of the reconstructed ones."""
    sys.path.insert(0, os.path.abspath(ROOT))
    import torch
    import torch.distributed as dist

    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream import decode as dec
    from coolchic_b200.dist import broadcast_byte_strings
    from coolchic_b200.io.framedata import FrameData

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    data = open(os.path.join(ROOT, "tests", "golden", "gop5_64x96_yuv420.cool"), "rb").read() if rank == 0 else None
    data = broadcast_byte_strings([data] if rank == 0 else None, src=0)[0]
    decoded_here = []

    def fake_decode(headers, nn, lat, device=0, finish=None):
        outs = []
        for h, b in zip(headers, lat):
            decoded_here.append(len(b))
            outs.append(torch.full(dec.output_shape(h), float(len(b) % 251), dtype=torch.float32))
        return outs

    def fake_reconstruct(frame_header, cc_out, refs, device):
        v = sum(float(t.mean()) for t in cc_out.values()) + sum(float(r.data.mean()) for r in refs)
        return FrameData(8, "rgb", torch.full((1, 3, 2, 2), v))

    frames = dec.decode_video_bytes(data, decode_fn=fake_decode, reconstruct_fn=fake_reconstruct)
    ret[rank] = (sorted(decoded_here), {k: float(f.data.mean()) for k, f in frames.items()})
    dist.destroy_process_group()


def test_gop_frames_are_owned_and_exchanged():
    import io
    from contextlib import redirect_stdout

    world, port = 2, _free_port()
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_gop_worker, args=(world, port, ret), nprocs=world, join=True)
    # 5 frames: I (1 Cool-chic) + 4 inter frames (2 each) = 9 Cool-chics; frame ownership by coding index:
    # rank 0 owns frames 0, 2, 4 (1 + 2 + 2 Cool-chics), rank 1 frames 1, 3 (2 + 2), no overlap
    assert len(ret[0][0]) == 5 and len(ret[1][0]) == 4
    assert ret[0][1] == ret[1][1] and len(ret[0][1]) == 5  # both ranks reconstructed the same 5 frames
    # and the same values as a single-process run of the same stand-ins
    sys.path.insert(0, os.path.abspath(ROOT))
    import torch

    import coolchic_b200  # noqa: F401
    from coolchic_b200.bitstream import decode as dec
    from coolchic_b200.io.framedata import FrameData

    data = open(os.path.join(ROOT, "tests", "golden", "gop5_64x96_yuv420.cool"), "rb").read()
    all_lens = []

    def fake_decode(headers, nn, lat, device=0, finish=None):
        all_lens.extend(len(b) for b in lat)
        return [torch.full(dec.output_shape(h), float(len(b) % 251), dtype=torch.float32) for h, b in zip(headers, lat)]

    def fake_reconstruct(frame_header, cc_out, refs, device):
        v = sum(float(t.mean()) for t in cc_out.values()) + sum(float(r.data.mean()) for r in refs)
        return FrameData(8, "rgb", torch.full((1, 3, 2, 2), v))

    with redirect_stdout(io.StringIO()):
        single = dec.decode_video_bytes(data, decode_fn=fake_decode, reconstruct_fn=fake_reconstruct)
    assert sorted(all_lens) == sorted(ret[0][0] + ret[1][0])
    assert {k: float(f.data.mean()) for k, f in single.items()} == ret[0][1]
