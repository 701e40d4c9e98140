"""TEST INFRASTRUCTURE: CPU stand-ins for the deterministic GroupNorm entry points (v3d_groupnorm_det_blocks,
v3d_groupnorm_partials, v3d_groupnorm_fold_apply, v3d_groupnorm_det), layered on tests/emu_ops.py.

Each restates the contract of include/v3d_b200.h in torch: a sample's rows are cut into blocks of min(256, hw) rows that
never straddle a frame; a block's (sum, sumsq) per group is summed in fp64 and stored as fp32 (the kernel's fp32 tree
rounds differently, so the stand-in matches it to fp32 rounding, not bit for bit); the per-sample fold adds the pairs
in fp64 in the kernel's order (lane l of 32 adds blocks l, l + 32, ... in turn, then an xor-shuffle tree).  What the
stand-ins share with the kernels is the property the host schedules rely on: a block's pair depends on that block's
rows only, so a frame-sharded schedule that gathers the pairs correctly reproduces the unsharded one BIT FOR BIT.
"""
from __future__ import annotations

import contextlib

import torch
import torch.nn.functional as F

import emu_ops
from emu_ops import BF, _store, _strided, _tick
from v3d_b200 import ops as real_ops


def groupnorm_det_blocks(rows_per_sample, hw):
    if hw <= 0 or rows_per_sample % hw:
        raise RuntimeError(f"groupnorm_det_blocks: hw={hw} does not divide rows_per_sample={rows_per_sample}")
    r = min(256, hw)
    return rows_per_sample // hw * ((hw + r - 1) // r)


def groupnorm_det_workspace_bytes(rows_per_sample, hw, nsamples, groups=32):
    return 256 + 8 * groupnorm_det_blocks(rows_per_sample, hw) * nsamples * groups


def groupnorm_det_workspace(device, nbytes):
    return torch.zeros(8, dtype=torch.uint8)


def block_pairs(x, rows_per_sample, hw, nsamples, c, ldx=None, groups=32):
    """-> fp32 [nsamples, blocks, groups, 2]: each block's (sum, sumsq) per group, summed in fp64"""
    ldx = c if ldx is None else ldx
    cpg = c // groups
    frames = rows_per_sample // hw
    r = min(256, hw)
    nbf = (hw + r - 1) // r
    v = _strided(x, (nsamples, frames, hw, c), (rows_per_sample * ldx, hw * ldx, ldx, 1)).double()
    v = F.pad(v, (0, 0, 0, nbf * r - hw))                                       # the short last block: zero rows
    v = v.reshape(nsamples, frames * nbf, r, groups, cpg).permute(0, 1, 3, 2, 4)
    v = v.reshape(nsamples, frames * nbf, groups, r * cpg).contiguous()        # one contiguous row per (block, group)
    return torch.stack([v.sum(-1), (v * v).sum(-1)], dim=-1).float()


def fold(pairs):
    """fp32 [nsamples, blocks, groups, 2] -> fp64 [nsamples, groups, 2], in the kernel's order"""
    ns, nblk, g, _ = pairs.shape
    k = (nblk + 31) // 32
    p = F.pad(pairs.double(), (0, 0, 0, 0, 0, 32 * k - nblk)).reshape(ns, k, 32, g, 2)
    acc = torch.zeros(ns, 32, g, 2, dtype=torch.float64, device=pairs.device)
    for i in range(k):                                                          # lane l: blocks l, l + 32, ...
        acc = acc + p[:, i]
    lanes = torch.arange(32, device=pairs.device)
    for o in (16, 8, 4, 2, 1):                                                  # xor-shuffle tree
        acc = acc + acc[:, lanes ^ o]
    return acc[:, 0]


def groupnorm_partials(x, partials, rows_per_sample, hw, nsamples, c, ldx=None, groups=32, ldp=None):
    assert x.dtype == BF and partials.dtype == torch.float32
    _tick()
    pairs = block_pairs(x, rows_per_sample, hw, nsamples, c, ldx=ldx, groups=groups)
    nblk = pairs.shape[1]
    ldp = nblk if ldp is None else ldp
    _strided(partials, (nsamples, nblk, groups, 2), (ldp * groups * 2, groups * 2, 2, 1)).copy_(pairs)
    return partials


def groupnorm_fold_apply(x, y, partials, gamma, beta, rows_per_sample, nsamples, c, eps, silu, nblocks,
                         count_rows=None, ldx=None, groups=32):
    _tick()
    ldx = c if ldx is None else ldx
    cpg = c // groups
    count_rows = rows_per_sample if count_rows is None else count_rows
    st = fold(_strided(partials, (nsamples, nblocks, groups, 2), (nblocks * groups * 2, groups * 2, 2, 1)))
    n = float(count_rows * cpg)
    mean = st[..., 0] / n
    var = (st[..., 1] / n - mean * mean).clamp_min(0.0)
    mean_f = mean.float().double()
    rstd_f = (1.0 / torch.sqrt(var + eps)).float().double()
    v = _strided(x, (nsamples, rows_per_sample, groups, cpg), (rows_per_sample * ldx, ldx, cpg, 1)).double()
    v = (v - mean_f[:, None, :, None]) * rstd_f[:, None, :, None]
    v = v.reshape(nsamples, rows_per_sample, c) * gamma.double() + beta.double()
    if silu:
        v = F.silu(v)
    _store(_strided(y, (nsamples * rows_per_sample, c), (c, 1)), v.reshape(-1, c))
    return y


def groupnorm_det(x, y, gamma, beta, rows_per_sample, hw, nsamples, c, eps, silu, workspace, ldx=None, groups=32):
    """single launch = partials + fold/apply (one tick)"""
    nblk = groupnorm_det_blocks(rows_per_sample, hw)
    part = torch.empty(nsamples, nblk, groups, 2, dtype=torch.float32, device=x.device)
    groupnorm_partials(x, part, rows_per_sample, hw, nsamples, c, ldx=ldx, groups=groups)
    groupnorm_fold_apply(x, y, part, gamma, beta, rows_per_sample, nsamples, c, eps, silu, nblk, ldx=ldx,
                         groups=groups)
    _tick(-1)
    return y


_EMULATED = ["groupnorm_det_blocks", "groupnorm_det_workspace_bytes", "groupnorm_det_workspace", "groupnorm_partials",
             "groupnorm_fold_apply", "groupnorm_det"]


@contextlib.contextmanager
def patched():
    """emu_ops.patched() plus the deterministic GroupNorm stand-ins."""
    saved = {n: getattr(real_ops, n) for n in _EMULATED}
    try:
        with emu_ops.patched():
            for n in _EMULATED:
                setattr(real_ops, n, globals()[n])
            yield
    finally:
        for n, f in saved.items():
            setattr(real_ops, n, f)
