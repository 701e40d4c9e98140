"""Time the native PixelNeRF render (rays + fused render + decoder, csrc/pixelnerf.cu) against the oracle's torch
restatement of the reference (oracle/ref_pixelnerf.py, fp32, on the same GPU).

    python tools/pixelnerf_timing.py [--rounds 3] [--iters 3] [--json out.json]

Both columns are timed the same way: one warm-up call, then CUDA events over `iters` back-to-back calls, best of
`rounds`.  Peak memory is torch.cuda.max_memory_allocated over one call after a reset, above what was allocated
before it.  The MLP rate counts the real work, 2 (d_in 128 + 128 128 + 128 129) FLOP per sample, not the padded
tiles the kernel runs.  The card's name, power limit and SM clock are printed with the table.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from oracle import ref_pixelnerf as R  # noqa: E402
from oracle.make_golden_scene import look_at_cams  # noqa: E402


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # pragma: no cover
        return f"nvidia-smi unavailable: {e}"


def timed(fn, rounds: int, iters: int):
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b) / iters)
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return best, (torch.cuda.max_memory_allocated() - base) / 2**20


def render_case(T, rs, ns, S, C, src, rounds, iters, with_oracle=True):
    from v3d_b200.pixelnerf import PixelNeRF

    dev = torch.device("cuda")
    m = PixelNeRF(num_samples_per_ray=ns, feature_dim=C, use_feats_std=True, use_pos_emb=True).to(dev)
    sd = {k: v.to(dev) for k, v in R.state_dict(m.d_in, 0).items()}
    m.load_state_dict(sd)
    cams = look_at_cams(T, 0.2)[None].to(dev)
    scams = look_at_cams(S, 1.0, 2.3)[None].to(dev)
    img = torch.rand(1, S, C, src, src, device=dev) * 2 - 1
    sc2w, sk = scams[..., :16].reshape(1, S, 4, 4), scams[..., 16:].reshape(1, S, 3, 3)
    tc2w, tk = cams[..., :16].reshape(1, T, 4, 4), cams[..., 16:].reshape(1, T, 3, 3)
    u = torch.rand(ns, T, rs * rs, 1, device=dev)
    m.jitter_sampler = lambda shape, d: u
    with torch.no_grad():
        nat = timed(lambda: m(img, sc2w, sk, tc2w, tk, rs), rounds, iters)
        flop = 2.0 * (m.d_in * 128 + 128 * 128 + 128 * 129) * T * rs * rs * ns
        row = {"T": T, "render": rs, "ns": ns, "S": S, "C": C, "src": src, "native_ms": nat[0], "native_mib": nat[1],
               "mlp_tflop": flop / 1e12, "native_mlp_tflops": flop / nat[0] / 1e9}
        if with_oracle:
            try:
                ref = timed(lambda: R.pixelnerf(sd, img, sc2w, sk, cams, rs, u.reshape(ns, -1), ns, use_std=True,
                                                use_pe=True), rounds, iters)
                row.update(torch_ms=ref[0], torch_mib=ref[1])
            except torch.OutOfMemoryError:
                row.update(torch_ms=None, torch_mib="out of memory")
            torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=3)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "pixelnerf_timing measures on the GPU; there is no CPU fallback"
    info = gpu_info()
    print(f"# {info}")
    rows = []
    for rs in (32, 64):
        for S in (1, 4):
            for src in (256, 512):
                r = render_case(24, rs, 128, S, 3, src, a.rounds, a.iters)
                rows.append(r)
                print(json.dumps(r))
    if a.json:
        Path(a.json).parent.mkdir(parents=True, exist_ok=True)
        Path(a.json).write_text(json.dumps({"gpu": info, "render": rows}, indent=1))


if __name__ == "__main__":
    main()
