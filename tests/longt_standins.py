"""TEST INFRASTRUCTURE: torch stand-ins of v3d_attention_temporal and v3d_attention_temporal_kv over the whole range the
kernels take (1..128 view-frames), next to those of tests/emu_ops.py, whose frame-sharded stand-in stops at 32 frames.

Same conventions as emu_ops: the contract of include/v3d_b200.h restated in torch, bf16 storage, fp64 arithmetic, one
bf16 rounding at the store, device-agnostic (tests/test_long_video_gpu.py holds both against the kernels on the same
CUDA tensors).  The dense and the frame-sharded form share one `_attend`, so a sharded run equals the unsharded one to
the last bit wherever the schedule and the row table are right.  `patched()` installs them on `v3d_b200.ops` together
with every stand-in of cross_standins.patched().
"""
from __future__ import annotations

import contextlib

import torch

import cross_standins
from emu_ops import _store, _strided, _tick
from v3d_b200 import ops as real_ops

MAX_FRAMES = 128


def _attend(q, k, v, scale):
    """softmax(q k^T scale) v in fp64, written out: q [..., tq, 64], k / v [..., tk, 64]."""
    s = torch.einsum("...qd,...kd->...qk", q, k) * scale
    p = torch.exp(s - s.amax(dim=-1, keepdim=True))
    return torch.einsum("...qk,...kd->...qd", p / p.sum(dim=-1, keepdim=True), v)


def attention_temporal(qkv, out, nb, t, s, nheads, scale):
    _tick()
    assert 0 < t <= MAX_FRAMES
    c, ld = nheads * 64, qkv.stride(0)
    rows = nb * t * s

    def seq(i):  # rows (b, t, s) -> sequences [b, s, h, t, 64]
        m = _strided(qkv[:, i * c:], (rows, c), (ld, 1)).double().reshape(nb, t, s, nheads, 64)
        return m.permute(0, 2, 3, 1, 4)

    o = _attend(seq(0), seq(1), seq(2), scale)
    _store(_strided(out, (rows, c), (out.stride(0), 1)), o.permute(0, 3, 1, 2, 4).reshape(rows, c))
    return out


def attention_temporal_kv(q, kv, out, nb, tq, s, nheads, kv_row, kv_bstride, scale):
    _tick()
    c = nheads * 64
    tk = len(kv_row)
    assert 0 < tq <= tk <= MAX_FRAMES
    rows = nb * tq * s
    qm = _strided(q, (rows, c), (q.stride(0), 1)).double().reshape(nb, tq, s, nheads, 64).permute(0, 2, 3, 1, 4)
    row = torch.tensor(kv_row, device=kv.device)
    bstride = torch.tensor(kv_bstride, device=kv.device)
    idx = (row[None, None, :] + torch.arange(nb, device=kv.device)[:, None, None] * bstride[None, None, :]
           + torch.arange(s, device=kv.device)[None, :, None])                             # [b, s, tk] buffer rows
    kvm = _strided(kv, (kv.shape[0], 2 * c), (kv.stride(0), 1))[idx].double()              # [b, s, tk, 2c]
    km = kvm[..., :c].reshape(nb, s, tk, nheads, 64).permute(0, 1, 3, 2, 4)
    vm = kvm[..., c:].reshape(nb, s, tk, nheads, 64).permute(0, 1, 3, 2, 4)
    o = _attend(qm, km, vm, scale)                                                          # [b, s, h, tq, 64]
    _store(_strided(out, (rows, c), (out.stride(0), 1)), o.permute(0, 3, 1, 2, 4).reshape(rows, c))
    return out


@contextlib.contextmanager
def patched():
    """cross_standins.patched() with the two temporal attention stand-ins of this module, for the duration of a test."""
    saved = real_ops.attention_temporal, real_ops.attention_temporal_kv
    with cross_standins.patched():
        try:
            real_ops.attention_temporal, real_ops.attention_temporal_kv = attention_temporal, attention_temporal_kv
            yield
        finally:
            real_ops.attention_temporal, real_ops.attention_temporal_kv = saved
