#!/usr/bin/env python
"""Timing of the multi-token cross-attention path on one GPU:

  * v3d_attention_cross at the V3D_512 spatial shapes (B = 36 frames, N = 4096 / 1024 / 256 queries, 5 / 10 / 20 heads)
    for M = 2, 4, 77 and 257 context tokens, with TFLOP/s of the useful work 4 * rows * M * 64 * heads;
  * one V3D_512 UNet forward (width 320, T = 18, latent 64x64, CFG batch 36, random weights, CUDA graphs) with a
    4-token context against the single-token context, alternated in this process.

CUDA events around many launches, every shape warmed first, the two forwards alternated; the GPU name, power limit and
SM clock are read in the same run.  Prints one line per case and a JSON summary.  Needs a CUDA device.
Usage: python tools/cross_attention_timing.py [--rounds 3] [--iters 20]"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from sampler_timing import gpu_info  # noqa: E402
from v3d_b200 import ops  # noqa: E402

DEV = "cuda"


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_kernel(res, iters):
    B = 36
    for lvl, n, heads in (("L0", 4096, 5), ("L1", 1024, 10), ("L2", 256, 20)):
        c = heads * 64
        q = torch.randn(B * n, c, device=DEV).to(torch.bfloat16)
        o = torch.empty_like(q)
        for M in (2, 4, 77, 257):
            kv = torch.randn(B * M, 2 * c, device=DEV).to(torch.bfloat16)
            fn = lambda: ops.attention_cross(q, kv, o, B, n, M, heads, 0.125)  # noqa: E731
            timed(fn, 3)
            ms = timed(fn, iters)
            tf = 4.0 * B * n * M * 64 * heads / ms / 1e9
            gb = (q.numel() + o.numel() + kv.numel()) * 2 / ms / 1e6
            print(f"cross {lvl} N={n} heads={heads} M={M:3d}  {ms:8.4f} ms  {tf:7.2f} TF/s  {gb:7.1f} GB/s")
            res.append(dict(kind="attention_cross", level=lvl, n=n, heads=heads, tokens=M, ms=ms, tflops=tf, gbs=gb))


def bench_unet(res, rounds, iters):
    from v3d_b200 import engine
    from v3d_b200.unet import VideoUNet

    T, hw = 18, 64
    kw = dict(engine.v3d_512_config(num_frames=T, num_steps=1)["network_config"]["params"])
    with torch.device("meta"):
        net = VideoUNet(**kw)
    net.init_random_(DEV, seed=0)
    net.eval()
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(2 * T, 8, hw, hw, device=DEV, generator=g)
    ts = torch.full((2 * T,), 0.3, device=DEV)
    y = torch.randn(2 * T, 768, device=DEV, generator=g)
    ind = torch.zeros(2, T, device=DEV)
    ctx = {M: torch.randn(2 * T, M, 1024, device=DEV, generator=g) for M in (1, 4)}
    run = {M: (lambda M=M: net(x, ts, ctx[M], y, None, T, ind)) for M in ctx}
    with torch.no_grad():
        for M in ctx:                       # eager, capture, replay
            for _ in range(3):
                run[M]()
        torch.cuda.synchronize()
        times = {M: [] for M in ctx}
        for _ in range(rounds):
            for M in (1, 4):
                times[M].append(timed(run[M], iters))
    for M, ts_ in times.items():
        print(f"unet V3D_512 forward M={M}: " + " ".join(f"{t:.2f}" for t in ts_) + " ms")
    r = min(times[4]) / min(times[1])
    print(f"M=4 / M=1 (best of {rounds}): {r:.4f}")
    res.append(dict(kind="unet_forward", ms_m1=times[1], ms_m4=times[4], ratio_best=r))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--skip-unet", action="store_true")
    a = ap.parse_args()
    info = gpu_info(torch.cuda.current_device())
    print(info)
    res = [dict(kind="gpu", **info)]
    bench_kernel(res, max(a.iters, 50))
    if not a.skip_unet:
        bench_unet(res, a.rounds, a.iters)
    res.append(dict(kind="gpu_after", **gpu_info(torch.cuda.current_device())))
    print("JSON " + json.dumps(res))


if __name__ == "__main__":
    main()
