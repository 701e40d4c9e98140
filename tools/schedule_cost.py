#!/usr/bin/env python
"""Exact algorithmic work of the hot path's launch schedules, without a GPU: the drop-in VideoUNet / VideoDecoder run
on torch's `meta` device (shapes only) with every `v3d_b200.ops` entry point replaced by a counter that books, per
kernel family, launches, algorithmic FLOPs and algorithmic HBM bytes (each operand read once, each result written
once - the "per unit" figures of DESIGN.md section 3 and of bench.py's roofline), and every ViewShard / CfgSplit
exchange replaced by a byte counter.  Nothing is computed; this is bookkeeping of what the host schedule launches.

    python tools/schedule_cost.py                      # V3D_512: one UNet forward (B=36) + one decode, per family
    python tools/schedule_cost.py --plan views --world 8 --rank 0      # this rank's share when frame-sharded
    python tools/schedule_cost.py --frames 24 --json out.json
    python tools/schedule_cost.py --tokens 4                   # a 4-token cross-attention context (default 1)
"""
from __future__ import annotations

import argparse
import contextlib
import json
import sys
from collections import OrderedDict
from pathlib import Path

import torch
import torch.nn as nn

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

from v3d_b200 import engine, ops as real_ops  # noqa: E402
from v3d_b200.viewshard import ViewShard, partition_frames  # noqa: E402

META = torch.device("meta")
BOOK: "OrderedDict[str, list]" = OrderedDict()     # family -> [launches, flops, bytes]
COMM: "OrderedDict[str, list]" = OrderedDict()     # exchange -> [calls, bytes sent by this rank]


def book(fam, flops=0.0, nbytes=0.0):
    e = BOOK.setdefault(fam, [0, 0.0, 0.0])
    e[0] += 1
    e[1] += flops
    e[2] += nbytes


def _nb(t):
    return t.element_size()


# ---- counters standing in for v3d_b200.ops ---------------------------------------------------------------------------
def gemm(a, w, out, *, K, N, rows_per_batch, batch=1, bias=None, fbias=None, r1=None, r2=None, act=0, ntaps=1,
         conv=None, a_rows=0, **kw):
    taps = 9 if conv is not None else ntaps
    rows = conv[0] * conv[1] * conv[2] if conv is not None else batch * rows_per_batch
    n_out = N // 2 if act == real_ops.ACT_GEGLU else N
    a_read = (batch * a_rows if a_rows else rows) * K * 2           # the taps re-read A from L2, not from HBM
    b_read = (batch if kw.get("b_batch_stride") else 1) * N * taps * K * 2
    nbytes = a_read + b_read + rows * n_out * _nb(out) + sum(rows * n_out * 2 for r in (r1, r2) if r is not None)
    fam = "gemm.conv3x3" if conv is not None else ("gemm.temporal" if taps == 3 else "gemm.linear")
    book(fam, 2.0 * rows * N * K * taps, nbytes)
    return out


def groupnorm_stats(x, stats, rows_per_sample, nsamples, c, **kw):
    book("groupnorm_stats", 0, rows_per_sample * nsamples * c * 2)
    return stats


def groupnorm_workspace(device):
    return None


def groupnorm(x, y, gamma, beta, rows_per_sample, nsamples, c, eps, silu, workspace, **kw):
    # one launch: x read (HBM), re-read (L2 when it fits), y written -- algorithmic bytes = read once + write once
    book("groupnorm", 0, 2 * rows_per_sample * nsamples * c * 2)
    return y


def groupnorm_apply(x, y, stats, gamma, beta, rows_per_sample, nsamples, c, eps, silu, **kw):
    book("groupnorm_apply", 0, 2 * rows_per_sample * nsamples * c * 2)
    return y


def layernorm(x, y, gamma, beta, rows, c, eps=1e-5, add=None, ysum=None, rows_per_frame=1):
    book("layernorm", 0, (3 if ysum is not None else 2) * rows * c * 2)
    return y


def softmax_rows_f32(x, y, rows, n, scale=1.0):
    book("softmax_rows_f32", 0, rows * n * 6)
    return y


def attention_spatial(qkv, out, nbatch, ntok, nheads, scale):
    book("attention_spatial", 4.0 * nbatch * nheads * ntok * ntok * 64, 4 * nbatch * ntok * nheads * 64 * 2)
    return out


def attention_temporal(qkv, out, nb, t, s, nheads, scale):
    book("attention_temporal", 4.0 * nb * s * nheads * t * t * 64, 4 * nb * t * s * nheads * 64 * 2)
    return out


def attention_temporal_kv(q, kv, out, nb, tq, s, nheads, kv_row, kv_bstride, scale):
    tk = len(kv_row)
    book("attention_temporal", 4.0 * nb * s * nheads * tq * tk * 64, (2 * tq + 2 * tk) * nb * s * nheads * 64 * 2)
    return out


def attention_cross(q, kv, out, nbatch, nq, nk, nheads, scale, kv_bstride=None):
    # Q read and O written once per query row, the item's K / V once per (item, query tile) -- counted once here
    book("attention_cross", 4.0 * nbatch * nq * nk * nheads * 64, (2 * nq + 2 * nk) * nbatch * nheads * 64 * 2)
    return out


def upsample_nearest2x(x, y, n, h, w, c):
    book("upsample_nearest2x", 0, 5 * n * h * w * c * 2)
    return y


def copy_channels(src, ld_src, dst, ld_dst, rows, ncols):
    book("copy_channels", 0, 2 * rows * ncols * 2)


def im2col3x3(x, y, n, h, w, c, stride, pad, hout, wout, kpad):
    book("im2col3x3", 0, n * h * w * c * 2 + n * hout * wout * kpad * 2)
    return y


def nchw_f32_to_nhwc_bf16(x, y, scale=1.0):
    book("layout", 0, x.numel() * 6)
    return y


def nhwc_to_nchw_f32(x, y, n, c, hw, ldx, scale=1.0):
    book("layout", 0, n * c * hw * (_nb(x) + 4))
    return y


def small_linear(x, w, bias, y, **kw):
    book("small_linear", 2.0 * x.shape[0] * w.shape[0] * w.shape[1], w.numel() * 2 + (x.numel() + y.numel()) * 4)
    return y


def timestep_embedding(t, out, dim, max_period=10000.0):
    book("timestep_embedding", 0, out.numel() * 4)
    return out


def time_mix_conv(x, ldx, w, bias, y, nb, t, hw, c):
    book("time_mix_conv", 2.0 * nb * t * hw * c * c * 3, nb * t * hw * (ldx * 4 + c * 4))
    return y


COUNTERS = ["gemm", "groupnorm_stats", "groupnorm_apply", "groupnorm", "groupnorm_workspace", "layernorm", "softmax_rows_f32", "attention_spatial",
            "attention_temporal", "attention_temporal_kv", "attention_cross", "upsample_nearest2x", "copy_channels", "im2col3x3",
            "nchw_f32_to_nhwc_bf16", "nhwc_to_nchw_f32", "small_linear", "timestep_embedding", "time_mix_conv"]


@contextlib.contextmanager
def counting():
    saved = {n: getattr(real_ops, n) for n in COUNTERS}
    try:
        for n in COUNTERS:
            setattr(real_ops, n, globals()[n])
        yield
    finally:
        for n, f in saved.items():
            setattr(real_ops, n, f)


class DryShard(ViewShard):
    """ViewShard whose exchanges only count the bytes this rank sends."""

    def _comm(self, kind, nbytes):
        e = COMM.setdefault(kind, [0, 0.0])
        e[0] += 1
        e[1] += nbytes

    def allreduce_stats_(self, stats):
        self._comm("gn_allreduce", stats.numel() * 8 if self.world > 1 else 0)
        return stats

    def exchange_halos(self, pad):
        nb = pad.shape[0]
        frame = pad[0, 0].numel() * pad.element_size()
        neighbours = (self.rank > 0) + (self.rank < self.world - 1)
        self._comm("halo", nb * neighbours * frame)
        return pad

    def gather_rows(self, send, buf=None, filled_rows=None):
        self._comm("kv_allgather", send.numel() * send.element_size() * (self.world > 1))
        return send.new_empty((self.world * send.shape[0],) + tuple(send.shape[1:]))


def _realise_mix_factors(mod: nn.Module) -> None:
    """_pack reads the (scalar) mix factors on the host; give them real storage, everything else stays on meta."""
    for name, p in list(mod.named_parameters()):
        if name.endswith("mix_factor"):
            owner = mod
            for part in name.split(".")[:-1]:
                owner = owner._modules[part]
            owner._parameters[name.split(".")[-1]] = nn.Parameter(torch.zeros(p.shape), requires_grad=False)


def run(frames: int, latent: int, plan: str, world: int, rank: int, edm_steps: int, tokens: int = 1):
    cfg = engine.v3d_512_config(num_frames=frames)
    with torch.device("meta"):
        eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    for m in (unet, dec):
        _realise_mix_factors(m)
    vs = None
    nb, tl = 2, frames
    if plan in ("views", "cfg+views"):
        pv = world if plan == "views" else world // 2
        vs = DryShard(frames, rank if plan == "views" else rank // 2, pv, None, partition_frames(frames, pv))
        tl = vs.tl
    if plan in ("cfg", "cfg+views"):
        nb = 1
    B = nb * tl
    with counting(), torch.no_grad():
        Pu = unet._pack(META)
        x = torch.empty(B, 8, latent, latent, device=META)
        ctx = torch.empty(B + (nb if vs is not None else 0), tokens * 1024, device=META)
        unet.view_shard = vs
        unet._run(Pu, x, torch.empty(B, device=META), ctx, torch.empty(B, 768, device=META), B, tl, nb, latent, latent,
                  META)
        unet_book = {k: list(v) for k, v in BOOK.items()}
        unet_comm = {k: list(v) for k, v in COMM.items()}
        BOOK.clear()
        COMM.clear()
        # decode: frame blocks whenever the image is spread over ranks
        if plan == "none":
            dvs, dtl = None, frames
        else:
            blocks = partition_frames(frames, world) if plan != "cfg+views" else None
            if blocks is None:
                blocks = []
                for t0, n in partition_frames(frames, world // 2):
                    blocks += [(t0, (n + 1) // 2), (t0 + (n + 1) // 2, n // 2)]
            dvs = DryShard(frames, rank, world, None, blocks)
            dtl = dvs.tl
        Pd = dec._pack(META)
        dec.view_shard = dvs
        dec._run(Pd, torch.empty(dtl, 4, latent, latent, device=META), dtl, dtl, 1, latent, latent)
        dec_book = {k: list(v) for k, v in BOOK.items()}
        dec_comm = {k: list(v) for k, v in COMM.items()}
        BOOK.clear()
        COMM.clear()
    cfg_bytes = tl * 4 * latent * latent * 4 if nb == 1 else 0      # one denoised half per network evaluation
    return {"config": {"frames": frames, "latent": latent, "plan": plan, "world": world, "rank": rank,
                       "unet_batch": B, "frames_local": tl, "edm_steps": edm_steps, "context_tokens": tokens},
            "unet_forward": unet_book, "decode": dec_book,
            "comm_per_unet_forward": dict(unet_comm, cfg_gather=[1 if nb == 1 else 0, cfg_bytes]),
            "comm_per_decode": dec_comm}


def table(title, bookd):
    print(f"\n**{title}**\n\n| family | launches | GFLOP | algorithmic GB |\n|---|---|---|---|")
    tot = [0, 0.0, 0.0]
    for k, (n, f, b) in sorted(bookd.items(), key=lambda kv: -(kv[1][1] + kv[1][2])):
        print(f"| {k} | {n} | {f / 1e9:.1f} | {b / 1e9:.3f} |")
        tot = [tot[0] + n, tot[1] + f, tot[2] + b]
    print(f"| **total** | {tot[0]} | {tot[1] / 1e9:.1f} | {tot[2] / 1e9:.2f} |")
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=18)
    ap.add_argument("--latent", type=int, default=64)
    ap.add_argument("--edm-steps", type=int, default=25)
    ap.add_argument("--plan", choices=["none", "views", "cfg", "cfg+views"], default="none")
    ap.add_argument("--world", type=int, default=1)
    ap.add_argument("--rank", type=int, default=0)
    ap.add_argument("--tokens", type=int, default=1, help="cross-attention context tokens per frame")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    res = run(a.frames, a.latent, a.plan, a.world, a.rank, a.edm_steps, a.tokens)
    c = res["config"]
    print(f"schedule cost: T={c['frames']} latent {c['latent']}^2, plan {c['plan']} (world {c['world']}, rank {c['rank']}): "
          f"UNet batch {c['unet_batch']}, {c['frames_local']} local frames, {c['context_tokens']} context token(s)")
    tu = table("one UNet forward", res["unet_forward"])
    td = table("one first-stage decode", res["decode"])
    S = a.edm_steps
    print(f"\nper image ({S} EDM steps): {S * tu[0] + td[0]} launches, {(S * tu[1] + td[1]) / 1e12:.1f} TFLOP, "
          f"{(S * tu[2] + td[2]) / 1e9:.0f} GB algorithmic traffic")
    if a.plan != "none":
        print("\n**exchanges of this rank**\n\n| exchange | per UNet forward: calls | MB sent | per decode: calls | MB sent |\n|---|---|---|---|---|")
        keys = list(OrderedDict.fromkeys(list(res["comm_per_unet_forward"]) + list(res["comm_per_decode"])))
        for k in keys:
            u = res["comm_per_unet_forward"].get(k, [0, 0])
            d = res["comm_per_decode"].get(k, [0, 0])
            print(f"| {k} | {u[0]} | {u[1] / 1e6:.2f} | {d[0]} | {d[1] / 1e6:.2f} |")
    if a.json:
        Path(a.json).write_text(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
