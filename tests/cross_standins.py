"""TEST INFRASTRUCTURE: the torch stand-in of v3d_attention_cross, next to those of tests/emu_ops.py.

Same conventions as emu_ops: the contract of include/v3d_b200.h restated in torch, bf16 storage, fp64 arithmetic, one
bf16 rounding at the store, device-agnostic (tests/test_cross_attention_gpu.py holds it against the kernel on the
same CUDA tensors).  `patched()` installs it on `v3d_b200.ops` together with every stand-in of emu_ops.patched().
"""
from __future__ import annotations

import contextlib

import torch.nn.functional as F

import emu_ops
from emu_ops import _store, _strided, _tick
from v3d_b200 import ops as real_ops


def attention_cross(q, kv, out, nbatch, nq, nk, nheads, scale, kv_bstride=None):
    _tick()
    c = nheads * 64
    bs = nk if kv_bstride is None else kv_bstride
    assert nk >= 1 and bs >= nk
    qm = _strided(q, (nbatch, nq, nheads, 64), (nq * q.stride(0), q.stride(0), 64, 1)).double().transpose(1, 2)
    km, vm = (_strided(kv[:, i * c:] if i else kv, (nbatch, nk, nheads, 64), (bs * kv.stride(0), kv.stride(0), 64, 1))
              .double().transpose(1, 2) for i in range(2))
    o = F.scaled_dot_product_attention(qm, km, vm, scale=scale)                            # [b, h, nq, 64]
    _store(_strided(out, (nbatch * nq, c), (out.stride(0), 1)), o.transpose(1, 2).reshape(nbatch * nq, c))
    return out


EMULATED = emu_ops._EMULATED + ["attention_cross"]


@contextlib.contextmanager
def patched():
    """emu_ops.patched() plus attention_cross, for the duration of a test."""
    saved = real_ops.attention_cross
    with emu_ops.patched():
        try:
            real_ops.attention_cross = attention_cross
            yield
        finally:
            real_ops.attention_cross = saved
