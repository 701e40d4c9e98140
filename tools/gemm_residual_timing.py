#!/usr/bin/env python
"""Residual GEMMs at the UNet (V3D_512, B = 36) and decoder shapes: R1 / R2 staged by TMA against R1 / R2 read by the
epilogue (__ldg).  The second arm passes copies of the residuals with a row pitch of N + 2 elements, which TMA cannot
address, so the same launch takes the __ldg path on the same values.  The two arms alternate in one process, inputs
larger than L2 are cycled so no launch re-reads an L2-resident operand set, and each line reports the median of the
rounds.  Prints the card, its power limit and one JSON summary line.  `--arms staged` times the contiguous launches
only, which any build of the library accepts (to compare two builds at the same shapes).
Usage: python tools/gemm_residual_timing.py [--rounds 5] [--iters 10] [--arms both|staged]"""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from v3d_b200 import ops  # noqa: E402

DEV = "cuda"
L2_CYCLE_BYTES = 256 << 20  # operand sets cycled per arm: several times the H100's 50 MB L2


def bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).to(torch.bfloat16)


def pitched(t):
    buf = torch.empty(t.shape[0], t.shape[1] + 2, device=DEV, dtype=t.dtype)
    buf[:, : t.shape[1]].copy_(t)
    return buf[:, : t.shape[1]]


# (name, kind, geometry, K, N, residuals): UNet levels L0-L3 at 64^2 / 32^2 / 16^2 / 8^2 latents, decoder at 18 frames
B, T = 36, 18
HW = {0: 4096, 1: 1024, 2: 256, 3: 64}
CS = {0: 320, 1: 640, 2: 1280, 3: 1280}
SIDE = {0: 64, 1: 32, 2: 16, 3: 8}


def cases():
    out = []
    for lvl in (0, 1, 2, 3):
        M, C, s = B * HW[lvl], CS[lvl], SIDE[lvl]
        out.append((f"unet L{lvl} conv3x3 +r1", "conv", (B, s, s), C, C, 1))
        out.append((f"unet L{lvl} to_out/proj_out +r1", "linear", M, C, C, 1))
        out.append((f"unet L{lvl} ff.net.2 +r1", "linear", M, 4 * C, C, 1))
        out.append((f"unet L{lvl} temporal ff +r1+r2", "linear", M, 4 * C, C, 2))
        out.append((f"unet L{lvl} time_stack (3,1,1) +r1", "tconv", (2, T * HW[lvl] // 2, HW[lvl]), C, C, 1))
    for side, c in ((64, 512), (128, 512), (256, 256), (512, 128)):
        out.append((f"dec {side}^2 conv3x3 +r1", "conv", (T, side, side), c, c, 1))
    return out


def build(kind, geom, K, N, nres):
    """One operand set, and the two launch closures (staged, __ldg) over it."""
    if kind == "conv":
        n, h, w = geom
        rows = n * h * w
        a, wt = bf(rows, K), bf(N, 9 * K, scale=(9 * K) ** -0.5)
        kw = dict(K=K, N=N, rows_per_batch=rows, conv=(n, h, w))
        flops = 2.0 * rows * N * 9 * K
    elif kind == "tconv":
        batch, rpb, hw = geom
        rows = batch * rpb
        a, wt = bf(rows, K), bf(N, 3 * K, scale=(3 * K) ** -0.5)
        kw = dict(K=K, N=N, rows_per_batch=rpb, batch=batch, a_batch_stride=rpb * K, ntaps=3, tap_shift=hw)
        flops = 2.0 * rows * N * 3 * K
    else:
        rows = geom
        a, wt = bf(rows, K), bf(N, K, scale=K ** -0.5)
        kw = dict(K=K, N=N, rows_per_batch=rows)
        flops = 2.0 * rows * N * K
    bias = torch.randn(N, device=DEV)
    o = torch.empty(rows, N, device=DEV, dtype=torch.bfloat16)
    r1 = bf(rows, N)
    r2 = bf(rows, N) if nres == 2 else None
    r1p, r2p = pitched(r1), (pitched(r2) if r2 is not None else None)
    kw.update(bias=bias, s0=0.5, s1=1.0, s2=0.5)
    nbytes = a.numel() * 2 + o.numel() * 2 * (1 + nres)

    def staged():
        ops.gemm(a, wt, o, r1=r1, r2=r2, **kw)

    def loaded():
        ops.gemm(a, wt, o, r1=r1p, ldr1=N + 2, r2=r2p, ldr2=N + 2 if r2p is not None else 0, **kw)

    return staged, loaded, flops, nbytes


def time_cycle(fns, iters):
    for f in fns:
        f()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(iters):
        fns[i % len(fns)]()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def card():
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        q = "unknown"
    return name, q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--arms", choices=["both", "staged"], default="both")
    args = ap.parse_args()
    both = args.arms == "both"
    name, q = card()
    print(f"card: {name}; power limit, max SM clock: {q}")
    results = []
    for label, kind, geom, K, N, nres in cases():
        first = build(kind, geom, K, N, nres)
        copies = max(1, min(8, -(-L2_CYCLE_BYTES // first[3])))
        sets = [first] + [build(kind, geom, K, N, nres) for _ in range(copies - 1)]
        st_fns, ld_fns = [s[0] for s in sets], [s[1] for s in sets]
        t_st, t_ld = [], []
        for _ in range(args.rounds):
            t_st.append(time_cycle(st_fns, args.iters))
            if both:
                t_ld.append(time_cycle(ld_fns, args.iters))
        ms_st = statistics.median(t_st)
        tf_st = first[2] / ms_st / 1e9
        line = f"{label:34s} K={K:5d} N={N:5d}  staged {ms_st:8.3f} ms {tf_st:6.1f} TF/s"
        res = dict(name=label, K=K, N=N, staged_ms=ms_st, staged_tflops=tf_st)
        if both:
            ms_ld = statistics.median(t_ld)
            tf_ld = first[2] / ms_ld / 1e9
            line += f"   __ldg {ms_ld:8.3f} ms {tf_ld:6.1f} TF/s   {100 * (ms_ld / ms_st - 1):+6.1f}%"
            res.update(ldg_ms=ms_ld, ldg_tflops=tf_ld)
        print(line)
        results.append(res)
        del sets, first
        torch.cuda.empty_cache()
    print(json.dumps(dict(card=name, power_limit_and_max_sm_clock=q, results=results)))


if __name__ == "__main__":
    main()
