#!/usr/bin/env python
"""Timing of the temporal self-attention on one GPU, across the boundary between its two kernels:

  * v3d_attention_temporal at the V3D_512 shapes (2 CFG halves x 4096 / 1024 / 256 / 64 pixels, 5 / 10 / 20 / 20 heads)
    for T = 18 and 32 (attn_temporal_kernel) and T = 33, 48, 64 and 128 (attn_temporal_long_kernel), the whole set
    alternated `--rounds` times in this process.  The kernel is HBM-bound: it reads q, k, v and writes o once, 4 * M * C
    bf16 = 8 * M * C bytes for M = 2 * T * pixels rows; reported are ms, ns per row, achieved GB/s over those bytes and
    their share of the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s, a figure for a 700 W card);
  * one UNet forward (width 320, latent 64x64, CFG, random weights, CUDA graphs) at T = 18 and T = 36, alternated, as ms
    per forward and per view-frame.

CUDA events around >= 50 launches, every shape warmed first; the GPU name, power limit and SM clock are read in the
same run.  Prints one line per case and a JSON summary.  Needs a CUDA device; there is no fallback.
Usage: python tools/temporal_attention_timing.py [--rounds 3] [--iters 50] [--skip-unet]"""
import argparse
import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

from sampler_timing import gpu_info  # noqa: E402

DEV = "cuda"
HBM_PEAK_GBS = 3350.0                      # H100 SXM data sheet, HBM3
LEVELS = (("L0", 4096, 5), ("L1", 1024, 10), ("L2", 256, 20), ("mid", 64, 20))
FRAMES = (18, 32, 33, 48, 64, 128)
NB = 2


def kernel_of(T: int) -> str:
    return "attn_temporal_kernel" if T <= 32 else "attn_temporal_long_kernel"


def algorithmic_bytes(T: int, pixels: int, heads: int, nb: int = NB) -> int:
    """q, k, v read and o written once: 4 matrices of M = nb * T * pixels rows by C = 64 * heads bf16 columns."""
    return 4 * (nb * T * pixels) * (64 * heads) * 2


def timed(fn, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bench_kernel(res, rounds, iters):
    from v3d_b200 import ops

    cases = {}
    for lvl, pixels, heads in LEVELS:
        c = heads * 64
        for T in FRAMES:
            rows = NB * T * pixels
            qkv = torch.randn(rows, 3 * c, device=DEV).to(torch.bfloat16)
            o = torch.empty(rows, c, device=DEV, dtype=torch.bfloat16)
            fn = lambda qkv=qkv, o=o, T=T, pixels=pixels, heads=heads: ops.attention_temporal(  # noqa: E731
                qkv, o, NB, T, pixels, heads, 0.125)
            timed(fn, 3)
            cases[(lvl, pixels, heads, T)] = (fn, [])
    for _ in range(rounds):
        for fn, ms in cases.values():
            ms.append(timed(fn, iters))
    for (lvl, pixels, heads, T), (_, ms) in cases.items():
        best = min(ms)
        nbytes = algorithmic_bytes(T, pixels, heads)
        gbs = nbytes / best / 1e6
        ns_row = best * 1e6 / (NB * T * pixels)
        print(f"temporal {lvl:3s} pixels={pixels:4d} heads={heads:2d} T={T:3d} {kernel_of(T):26s} "
              + " ".join(f"{m:8.4f}" for m in ms) + f" ms  {ns_row:7.3f} ns/row  {gbs:7.1f} GB/s  "
              f"{100 * gbs / HBM_PEAK_GBS:5.1f} % of 3.35 TB/s (HBM-bound)")
        res.append(dict(kind="attention_temporal", level=lvl, pixels=pixels, heads=heads, T=T, kernel=kernel_of(T),
                        ms=ms, ms_best=best, ns_per_row=ns_row, bytes=nbytes, gbs=gbs,
                        hbm_share=gbs / HBM_PEAK_GBS))


def bench_unet(res, rounds, iters):
    from v3d_b200 import engine
    from v3d_b200.unet import VideoUNet

    hw = 64
    kw = dict(engine.v3d_512_config(num_frames=18, num_steps=1)["network_config"]["params"])
    with torch.device("meta"):
        net = VideoUNet(**kw)
    net.init_random_(DEV, seed=0)
    net.eval()
    g = torch.Generator(device=DEV).manual_seed(0)
    run = {}
    for T in (18, 36):
        x = torch.randn(2 * T, 8, hw, hw, device=DEV, generator=g)
        ts = torch.full((2 * T,), 0.3, device=DEV)
        y = torch.randn(2 * T, 768, device=DEV, generator=g)
        ind = torch.zeros(2, T, device=DEV)
        ctx = torch.randn(2 * T, 1, 1024, device=DEV, generator=g)
        run[T] = lambda x=x, ts=ts, ctx=ctx, y=y, T=T, ind=ind: net(x, ts, ctx, y, None, T, ind)  # noqa: E731
    with torch.no_grad():
        for T in run:                       # eager, capture, replay
            for _ in range(3):
                run[T]()
        torch.cuda.synchronize()
        times = {T: [] for T in run}
        for _ in range(rounds):
            for T in run:
                times[T].append(timed(run[T], iters))
    per_frame = {T: min(ms) / T for T, ms in times.items()}
    for T, ms in times.items():
        print(f"unet width 320 latent 64x64 CFG forward T={T}: " + " ".join(f"{t:.2f}" for t in ms)
              + f" ms  {per_frame[T]:.3f} ms per view-frame")
    print(f"ms per view-frame, T=36 / T=18 (best of {rounds}): {per_frame[36] / per_frame[18]:.4f}")
    res.append(dict(kind="unet_forward", ms_t18=times[18], ms_t36=times[36], ms_per_frame_t18=per_frame[18],
                    ms_per_frame_t36=per_frame[36]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--unet-iters", type=int, default=10)
    ap.add_argument("--skip-unet", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("temporal_attention_timing needs a CUDA device; there is nothing to time without one")
    info = gpu_info(torch.cuda.current_device())
    print(info)
    res = [dict(kind="gpu", **info)]
    bench_kernel(res, a.rounds, max(a.iters, 50))
    if not a.skip_unet:
        bench_unet(res, a.rounds, a.unet_iters)
    res.append(dict(kind="gpu_after", **gpu_info(torch.cuda.current_device())))
    print("JSON " + json.dumps(res))


if __name__ == "__main__":
    main()
