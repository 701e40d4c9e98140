#!/usr/bin/env python
"""Per-shape kernel timings at the V3D_512 shapes (B=36, T=18, latent 64x64): CUDA-event timed, inputs larger
than L2 are cycled so no launch re-reads an L2-resident operand set. Prints one line per shape and a JSON summary.
Usage: python tools/microbench.py [gemm] [conv] [attn] [norm] [small]"""
import json
import sys
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parent.parent))
from v3d_b200 import ops  # noqa: E402

DEV = "cuda"
# NVIDIA's H100 SXM data sheet (dense BF16, HBM3); percentages below are of these, not of measured peaks
PEAK_TF, PEAK_GB = 989.0, 3350.0


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def bf(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).to(torch.bfloat16)


def bench_gemm(out):
    B, T = 36, 18
    rows = {0: B * 4096, 1: B * 1024, 2: B * 256, 3: B * 64}
    Cs = {0: 320, 1: 640, 2: 1280, 3: 1280}
    cases = []
    for lvl in (0, 1, 2, 3):
        M, C = rows[lvl], Cs[lvl]
        cases += [(f"L{lvl} qkv", M, C, 3 * C, {}), (f"L{lvl} proj+res", M, C, C, {"res": 1}),
                  (f"L{lvl} geglu", M, C, 8 * C, {"geglu": 1}), (f"L{lvl} ff_out+res", M, 4 * C, C, {"res": 1}),
                  (f"L{lvl} ff_out+blend", M, 4 * C, C, {"res": 2})]
    if "ksweep" in sys.argv:
        cases = [(f"ksweep N={n} K={k}", 147456, k, n, o) for n, o in ((960, {}), (320, {"res": 1}), (2560, {"geglu": 1}))
                 for k in (64, 128, 320, 640, 1280)]
    for name, M, K, N, opt in cases:
        a, w = bf(M, K), bf(N, K, scale=K ** -0.5)
        bias = torch.randn(N, device=DEV)
        n_out = N // 2 if opt.get("geglu") else N
        o = torch.empty(M, n_out, device=DEV, dtype=torch.bfloat16)
        kw = dict(K=K, N=N, rows_per_batch=M, bias=bias)
        if opt.get("geglu"):
            kw["act"] = ops.ACT_GEGLU
        if opt.get("res", 0) >= 1:
            kw.update(r1=bf(M, n_out), s1=1.0)
        if opt.get("res", 0) >= 2:
            kw.update(r2=bf(M, n_out), s2=0.5)
        ms = timeit(lambda: ops.gemm(a, w, o, **kw))
        tf = 2.0 * M * N * K / ms / 1e9
        print(f"gemm {name:18s} M={M:7d} K={K:5d} N={N:5d}  {ms:8.3f} ms  {tf:7.1f} TF/s  {100 * tf / PEAK_TF:5.1f}%")
        out.append(dict(kind="gemm", name=name, M=M, K=K, N=N, ms=ms, tflops=tf))
    # temporal conv
    for lvl in (0, 1, 2, 3):
        hw, C = rows[lvl] // B, Cs[lvl]
        x, w = bf(2 * T * hw, C), bf(C, 3 * C, scale=(3 * C) ** -0.5)
        o = torch.empty(2 * T * hw, C, device=DEV, dtype=torch.bfloat16)
        r1 = bf(2 * T * hw, C)
        ms = timeit(lambda: ops.gemm(x, w, o, K=C, N=C, rows_per_batch=T * hw, batch=2, a_batch_stride=T * hw * C,
                                     ntaps=3, tap_shift=hw, r1=r1, s1=1.0, s0=0.5))
        tf = 2.0 * 2 * T * hw * C * 3 * C / ms / 1e9
        print(f"tconv L{lvl} rows={2 * T * hw} C={C}  {ms:8.3f} ms  {tf:7.1f} TF/s  {100 * tf / PEAK_TF:5.1f}%")
        out.append(dict(kind="tconv", name=f"L{lvl}", ms=ms, tflops=tf))


def bench_conv(out):
    cases = [("unet L0 320->320", 36, 64, 64, 320, 320), ("unet L0 960->320", 36, 64, 64, 960, 320),
             ("unet L1 640->640", 36, 32, 32, 640, 640), ("unet L2 1280->1280", 36, 16, 16, 1280, 1280),
             ("unet L3 1280->1280", 36, 8, 8, 1280, 1280), ("unet L3 2560->1280", 36, 8, 8, 2560, 1280),
             ("dec 64 512->512", 18, 64, 64, 512, 512), ("dec 128 512->512", 18, 128, 128, 512, 512),
             ("dec 256 256->256", 18, 256, 256, 256, 256), ("dec 512 128->128", 18, 512, 512, 128, 128)]
    for name, n, h, w, ci, co in cases:
        x, wt = bf(n * h * w, ci), bf(co, 9 * ci, scale=(9 * ci) ** -0.5)
        bias = torch.randn(co, device=DEV)
        o = torch.empty(n * h * w, co, device=DEV, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.gemm(x, wt, o, K=ci, N=co, rows_per_batch=n * h * w, bias=bias, conv=(n, h, w)),
                    iters=5)
        tf = 2.0 * n * h * w * co * 9 * ci / ms / 1e9
        print(f"conv {name:20s} {ms:8.3f} ms  {tf:7.1f} TF/s  {100 * tf / PEAK_TF:5.1f}%")
        out.append(dict(kind="conv", name=name, ms=ms, tflops=tf))


def bench_attn(out):
    for name, nb, ntok, heads in [("L0", 36, 4096, 5), ("L1", 36, 1024, 10), ("L2", 36, 256, 20), ("L3", 36, 64, 20)]:
        c = heads * 64
        qkv = bf(nb * ntok, 3 * c)
        o = torch.empty(nb * ntok, c, device=DEV, dtype=torch.bfloat16)
        for impl, fn in (("wgmma", ops.attention_spatial), ("mma", ops.attention_spatial_mma)):
            ms = timeit(lambda: fn(qkv, o, nb, ntok, heads, 0.125), iters=5)
            tf = 4.0 * nb * heads * ntok * ntok * 64 / ms / 1e9
            print(f"attn {name} {impl:8s} ntok={ntok} heads={heads}  {ms:8.3f} ms  {tf:7.1f} TF/s  {100 * tf / PEAK_TF:5.1f}%")
            out.append(dict(kind="attn", name=name, impl=impl, ms=ms, tflops=tf))
    for name, s, heads in [("L0", 4096, 5), ("L1", 1024, 10), ("L2", 256, 20), ("L3", 64, 20)]:
        c = heads * 64
        qkv = bf(2 * 18 * s, 3 * c)
        o = torch.empty(2 * 18 * s, c, device=DEV, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.attention_temporal(qkv, o, 2, 18, s, heads, 0.125), iters=5)
        gb = (qkv.numel() + o.numel()) * 2 / ms / 1e6
        print(f"tattn {name} S={s} heads={heads}  {ms:8.3f} ms  {gb:7.1f} GB/s  {100 * gb / PEAK_GB:5.1f}%")
        out.append(dict(kind="tattn", name=name, ms=ms, gbs=gb))


def bench_norm(out):
    for name, ns, rows, c in [("gn2d L0 320", 36, 4096, 320), ("gn3d L0 320", 2, 18 * 4096, 320),
                              ("gn2d L0 640", 36, 4096, 640), ("gn2d L0 960", 36, 4096, 960),
                              ("gn2d L1 640", 36, 1024, 640), ("gn2d dec256 256", 18, 65536, 256),
                              ("gn2d L2 1280", 36, 256, 1280), ("gn2d L3 1280", 36, 64, 1280),
                              ("gn3d L3 1280", 2, 18 * 64, 1280), ("gn2d dec512 128", 18, 262144, 128),
                              ("gn3d dec512 128", 1, 18 * 262144, 128)]:
        x = bf(ns * rows, c)
        y = torch.empty_like(x)
        g, b = torch.ones(c, device=DEV), torch.zeros(c, device=DEV)
        st = torch.empty(ns, 32, 2, device=DEV, dtype=torch.float64)
        ms1 = timeit(lambda: ops.groupnorm_stats(x, st, rows, ns, c), iters=5)
        ms2 = timeit(lambda: ops.groupnorm_apply(x, y, st, g, b, rows, ns, c, 1e-5, True), iters=5)
        ws = ops.groupnorm_workspace(DEV)
        ms3 = timeit(lambda: ops.groupnorm(x, y, g, b, rows, ns, c, 1e-5, True, ws), iters=5)
        gb1 = x.numel() * 2 / ms1 / 1e6
        gb2 = x.numel() * 4 / ms2 / 1e6
        gb3 = x.numel() * 4 / ms3 / 1e6
        print(f"{name:18s} stats {ms1:7.3f} ms {gb1:7.0f} GB/s ({100 * gb1 / PEAK_GB:4.1f}%)  apply {ms2:7.3f} ms {gb2:7.0f} GB/s ({100 * gb2 / PEAK_GB:4.1f}%)"
              f"  one-launch {ms3:7.3f} ms {gb3:7.0f} GB/s ({100 * gb3 / PEAK_GB:4.1f}% of peak on read-once + write-once bytes; pair {ms1 + ms2:7.3f} ms)")
        out.append(dict(kind="gn", name=name, stats_ms=ms1, apply_ms=ms2, fused_ms=ms3, stats_gbs=gb1, apply_gbs=gb2, fused_gbs=gb3))
    for name, rows, c in [("ln L0", 36 * 4096, 320), ("ln L1", 36 * 1024, 640), ("ln L2", 36 * 256, 1280)]:
        x = bf(rows, c)
        y = torch.empty_like(x)
        g, b = torch.ones(c, device=DEV), torch.zeros(c, device=DEV)
        ms = timeit(lambda: ops.layernorm(x, y, g, b, rows, c), iters=5)
        gb = x.numel() * 4 / ms / 1e6
        print(f"{name:18s} {ms:7.3f} ms {gb:7.0f} GB/s ({100 * gb / PEAK_GB:4.1f}%)")
        out.append(dict(kind="ln", name=name, ms=ms, gbs=gb))


def bench_small(out):
    for name, m, k, n, ai in [("emb_all", 36, 1280, 38400, 1), ("cv_all", 36, 1024, 25600, 0),
                              ("time_embed.2", 36, 1280, 1280, 0), ("to_out 320", 36, 320, 320, 0),
                              ("to_out 1280", 36, 1280, 1280, 0), ("pos.0 1280", 36, 1280, 5120, 0)]:
        x = torch.randn(m, k, device=DEV)
        w = bf(n, k, scale=k ** -0.5)
        b = torch.randn(n, device=DEV)
        y = torch.empty(m, n, device=DEV)
        ms = timeit(lambda: ops.small_linear(x, w, b, y, act_in=ai), iters=5)
        gb = n * k * 2 / ms / 1e6
        print(f"small {name:14s} M={m} K={k} N={n}  {ms:7.3f} ms  weights {gb:7.0f} GB/s")
        out.append(dict(kind="small", name=name, ms=ms, gbs=gb))


def one_gemm(M=147456, K=320, N=2560, geglu=True, iters=6):
    """single shape, few launches: the target of `ncu --set full -k regex:gemm_tc`"""
    a, w = bf(M, K), bf(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    o = torch.empty(M, N // 2 if geglu else N, device=DEV, dtype=torch.bfloat16)
    kw = dict(K=K, N=N, rows_per_batch=M, bias=bias)
    if geglu:
        kw["act"] = ops.ACT_GEGLU
    if "res" in sys.argv:
        kw.update(r1=bf(M, N), s1=1.0)
    for _ in range(iters):
        ops.gemm(a, w, o, **kw)
    torch.cuda.synchronize()


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "one_gemm":
        nums = [int(a) for a in sys.argv[2:] if a.isdigit()]
        if len(nums) == 3:
            one_gemm(nums[0], nums[1], nums[2], geglu="geglu" in sys.argv)
        else:
            one_gemm(geglu="nogeglu" not in sys.argv)
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "time":
        M, K, N = [int(a) for a in sys.argv[2:5]]
        a, w = bf(M, K), bf(N, K, scale=K ** -0.5)
        o = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
        ms = timeit(lambda: ops.gemm(a, w, o, K=K, N=N, rows_per_batch=M))
        print(f"time M={M} K={K} N={N}: {ms * 1e3:.1f} us  {2 * M * K * N / ms / 1e9:.0f} TF/s")
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "ncu_set":
        # one process, two launches of every kernel family at its V3D_512 top-level shape: the target of ONE
        # `ncu --set full -k regex:"gn_|layernorm|attn_|gemm_tc|softmax_rows"` run (profiles/: one capture per kernel)
        ns, rows, c = 36, 4096, 320
        x = bf(ns * rows, c)
        y = torch.empty_like(x)
        g, b = torch.ones(c, device=DEV), torch.zeros(c, device=DEV)
        st = torch.zeros(ns, 32, 2, device=DEV, dtype=torch.float64)
        qkv = bf(ns * rows, 3 * c)
        o = torch.empty(ns * rows, c, device=DEV, dtype=torch.bfloat16)
        wt = bf(c, 9 * c, scale=(9 * c) ** -0.5)
        wl = bf(c, c, scale=c ** -0.5)
        wg = bf(8 * c, c, scale=c ** -0.5)
        og = torch.empty(ns * rows, 4 * c, device=DEV, dtype=torch.bfloat16)
        bias, bias8 = torch.randn(c, device=DEV), torch.randn(8 * c, device=DEV)
        sc = torch.randn(4 * 4096, 4096, device=DEV)
        pr = torch.empty(4 * 4096, 4096, device=DEV, dtype=torch.bfloat16)
        gws = ops.groupnorm_workspace(DEV)
        for _ in range(2):
            ops.groupnorm_stats(x, st, rows, ns, c)
            ops.groupnorm_apply(x, y, st, g, b, rows, ns, c, 1e-5, True)
            ops.groupnorm_stats(x, st[:2], 18 * rows, 2, c)
            ops.groupnorm_apply(x, y, st[:2], g, b, 18 * rows, 2, c, 1e-5, True)
            ops.groupnorm(x, y, g, b, rows, ns, c, 1e-5, True, gws)
            ops.groupnorm(x, y, g, b, 18 * rows, 2, c, 1e-5, True, gws)
            ops.layernorm(x, y, g, b, ns * rows, c)
            ops.attention_temporal(qkv, o, 2, 18, rows, 5, 0.125)
            ops.attention_spatial(qkv, o, ns, rows, 5, 0.125)
            ops.gemm(x, wt, o, K=c, N=c, rows_per_batch=ns * rows, bias=bias, conv=(ns, 64, 64))
            ops.gemm(x, wl, o, K=c, N=c, rows_per_batch=ns * rows, bias=bias, r1=y, s1=1.0)
            ops.gemm(x, wg, og, K=c, N=8 * c, rows_per_batch=ns * rows, bias=bias8, act=ops.ACT_GEGLU)
            ops.softmax_rows_f32(sc, pr, 4 * 4096, 4096)
        torch.cuda.synchronize()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "one_conv":
        n, h, w, ci, co = 36, 64, 64, 320, 320
        x, wt = bf(n * h * w, ci), bf(co, 9 * ci, scale=(9 * ci) ** -0.5)
        bias = torch.randn(co, device=DEV)
        o = torch.empty(n * h * w, co, device=DEV, dtype=torch.bfloat16)
        for _ in range(6):
            ops.gemm(x, wt, o, K=ci, N=co, rows_per_batch=n * h * w, bias=bias, conv=(n, h, w))
        torch.cuda.synchronize()
        sys.exit(0)
    if len(sys.argv) > 1 and sys.argv[1] == "one_attn":
        qkv = bf(36 * 4096, 960)
        o = torch.empty(36 * 4096, 320, device=DEV, dtype=torch.bfloat16)
        for _ in range(4):
            ops.attention_spatial(qkv, o, 36, 4096, 5, 0.125)
        torch.cuda.synchronize()
        sys.exit(0)
    sel = (set(sys.argv[1:]) - {"ksweep"}) or {"gemm", "conv", "attn", "norm", "small"}
    res = []
    if "gemm" in sel:
        bench_gemm(res)
    if "conv" in sel:
        bench_conv(res)
    if "attn" in sel:
        bench_attn(res)
    if "norm" in sel:
        bench_norm(res)
    if "small" in sel:
        bench_small(res)
    print("JSON " + json.dumps(res))
