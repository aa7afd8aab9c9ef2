"""Data movement of the job calls: a call stages its inputs with one host->device copy and brings its results back
with one device->host copy, whatever the number of jobs (copies counted in a torch.profiler trace of CUDA activities)."""
import time

import pytest


def _copies(fn):
    """(host->device, device->host) copies of one fn() call, after a warm-up call.  The profiler drops device activities
    whose timestamps fall outside its capture window, so the call runs 50 ms inside both ends of it."""
    import torch

    fn()
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        time.sleep(0.05)
        fn()
        torch.cuda.synchronize()
        time.sleep(0.05)
    names = [e.name for e in prof.events()]
    assert any("k_" in n for n in names), f"the trace holds none of the call's kernels: {sorted(set(names))}"
    return sum(n.startswith("Memcpy HtoD") for n in names), sum(n.startswith("Memcpy DtoH") for n in names)


@pytest.mark.gpu
def test_one_copy_each_way_per_call(ctx, kodim14):
    import torch

    from coolchic_b200 import _native
    from coolchic_b200.io.framedata import FrameData

    dev = ctx.torch_device
    n = 132
    d, nb, lb = kodim14["desc"], kodim14["nn_bytes"], kodim14["lat_bytes"]
    assert _copies(lambda: ctx.decode_many([d] * n, [nb] * n, [lb] * n)) == (1, 1)

    _, lats = ctx.decode_many([d] * n, [nb] * n, [lb] * n, want_latents=True)
    nn = _native.decode_nn(d, nb)
    assert _copies(lambda: ctx.latent_rate([d] * n, [nn] * n, lats, want_spatial=True)) == (1, 1)

    # 32 frames of 1080p 4:2:0, the size of the frames of bench.py's gop32_1080p_yuv420 workload
    h, w = 1080, 1920
    g = torch.Generator(device=dev).manual_seed(0)
    frames, srcs = [], []
    for _ in range(32):
        k = torch.randint(0, 256, (h * w * 3 // 2,), generator=g, device=dev, dtype=torch.int32)
        y, u, v = (k.float() / 255).split([h * w, h * w // 4, h * w // 4])
        frames.append(FrameData(8, "yuv420", {"y": y.view(1, 1, h, w), "u": u.view(1, 1, h // 2, w // 2),
                                              "v": v.view(1, 1, h // 2, w // 2)}))
        srcs.append(k.to(torch.uint8))
    assert _copies(lambda: ctx.frame_distortion(frames, srcs, ["planar"] * 32)) == (1, 1)

    # one P frame: the statistics come back in one copy, and nothing goes up
    h, w = 128, 192
    residue = torch.rand((1, 4, h, w), generator=g, device=dev) - 0.5
    motion = 4 * torch.rand((1, 2, h, w), generator=g, device=dev) - 2
    ref = FrameData(8, "rgb", torch.randint(0, 256, (1, 3, h, w), generator=g, device=dev).float() / 255)
    src = torch.randint(0, 256, (3 * h * w,), generator=g, device=dev, dtype=torch.int32).to(torch.uint8)
    assert _copies(lambda: ctx.inter_stats(residue, motion, [ref], False, "rgb", 8, [0, 0], 8, source=src)) == (0, 1)
