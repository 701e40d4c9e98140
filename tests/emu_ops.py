"""TEST INFRASTRUCTURE: a torch-on-CPU stand-in for the `v3d_b200.ops` API (the C-ABI wrappers).

The product path has no CPU implementation and must not get one; this module exists so that the HOST SCHEDULES of
the drop-in modules (`VideoUNet._run`, `VideoDecoder._run`, the samplers, the shard plans, PixelNeRF: which kernel runs
on which buffer with which strides, offsets, fused-epilogue operands, halo buffers and exchanges) can be executed and
checked on a box without a GPU:
  * against the oracle and the real reference's fixtures (tests/test_host_schedule_cpu.py and the other *_cpu.py
    files): a wrong leading dimension, bias row, residual, packing permutation or layout convention in the schedule
    shows up as a parity failure;
  * frame-sharded against unsharded over gloo.
Each function restates the CONTRACT documented in include/v3d_b200.h for one entry point, in plain torch: bf16 storage,
arithmetic in fp64 (so that results do not depend on how a CPU BLAS blocks a given shape: a frame-sharded run and an
unsharded run then agree to the last bit wherever the schedule is right), one rounding at the store.  The sampler steps
and the PixelNeRF entry points compute in fp32; their sections say how.  The stand-ins are only ever installed by
`patched()` inside tests, which also counts and can record their launches; nothing under v3d_b200/ imports this module.
The functions are device-agnostic, so tests/test_standins_gpu.py and the other GPU tests can hold them against the real
kernels on the same CUDA tensors.
"""
from __future__ import annotations

import contextlib
import hashlib
import math
from collections import Counter

import torch
import torch.nn.functional as F

from oracle import ref_pixelnerf
from v3d_b200 import ops as real_ops

ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2
BF = torch.bfloat16
MAX_FRAMES = 128
_launches: Counter = Counter()          # calls per launch entry point, counted by patched() and never reset


def _strided(t: torch.Tensor, size, stride) -> torch.Tensor:
    """Typed window into t's storage starting at t's first element (what a kernel sees through a raw pointer)."""
    return torch.as_strided(t, size, stride, t.storage_offset())


def _store(dst: torch.Tensor, val: torch.Tensor) -> None:
    dst.copy_(val.to(dst.dtype))


def launch_count() -> int:
    return sum(_launches.values())


pick_block_n = real_ops.pick_block_n      # host functions of the library (no GPU involved)
geglu_perm = real_ops.geglu_perm
_require_cuda_current_device = real_ops.require_current_device


def require_current_device(t, who):
    """The entry points' CUDA gate with CPU tensors let through, so that `patched()` alone runs any module, sampler or
    engine on CPU; a CUDA tensor gets the real check."""
    if t.is_cuda:
        _require_cuda_current_device(t, who)


def digest(record: list) -> tuple:
    """(launches, sha256) of a launch record of `patched(record)`: pins a whole schedule's kernels, arguments and order."""
    return len(record), hashlib.sha256(repr(record).encode()).hexdigest()


# ---------------------------------------------------------------------------------------------------------------
# v3d_gemm_bf16
# ---------------------------------------------------------------------------------------------------------------
def gemm(a, w, out, *, K, N, rows_per_batch, batch=1, lda=None, ldb=None, ldd=None, a_batch_stride=0,
         b_batch_stride=0, bias=None, fbias=None, rows_per_frame=1, ldfb=0, r1=None, ldr1=0, r2=None, ldr2=0, s0=1.0,
         s1=1.0, s2=1.0, act=ACT_NONE, ntaps=1, tap_shift=0, conv=None, block_n=0, transposed=False, valid_cols=0,
         accumulate=False, a_rows=0, a_row0=0):
    assert a.dtype == BF and w.dtype == BF and not transposed and not accumulate
    assert K % 64 == 0 and N % 16 == 0, (K, N)
    taps = 9 if conv is not None else ntaps
    lda = K if lda is None else lda
    ldb = taps * K if ldb is None else ldb
    n_out = N // 2 if act == ACT_GEGLU else N
    ldd = n_out if ldd is None else ldd
    if conv is not None:
        n, h, wd = conv
        rows = n * h * wd
        x = _strided(a, (n, h, wd, K), (h * wd * lda, wd * lda, lda, 1)).double().permute(0, 3, 1, 2)
        wt = _strided(w, (N, 9 * K), (ldb, 1)).double().reshape(N, 3, 3, K).permute(0, 3, 1, 2)   # (ky, kx, ci)
        acc = F.conv2d(x, wt, padding=1).permute(0, 2, 3, 1).reshape(rows, N)
    else:
        rows = batch * rows_per_batch
        arows = a_rows if a_rows > 0 else rows_per_batch + a_row0
        abs_ = a_batch_stride if batch > 1 else arows * lda
        A = _strided(a, (batch, arows, K), (abs_, lda, 1)).double()
        nbb = batch if b_batch_stride else 1
        Bm = _strided(w, (nbb, N, taps * K), (b_batch_stride, ldb, 1)).double()
        acc = torch.zeros(batch, rows_per_batch, N, dtype=torch.float64, device=a.device)
        for tap in range(taps):
            first = a_row0 + (tap - taps // 2) * tap_shift           # A row read by output row 0
            lo, hi = max(0, -first), min(rows_per_batch, arows - first)
            if hi <= lo:
                continue
            At = torch.zeros(batch, rows_per_batch, K, dtype=torch.float64, device=a.device)
            At[:, lo:hi] = A[:, first + lo: first + hi]               # rows outside [0, a_rows) read as zero
            acc += At @ Bm[:, :, tap * K:(tap + 1) * K].transpose(1, 2)
        acc = acc.reshape(rows, N)
    if bias is not None:
        acc = acc + bias.double()[:N]
    if fbias is not None:
        ldfb_ = ldfb if ldfb > 0 else N
        frames = (rows + rows_per_frame - 1) // rows_per_frame
        fb = _strided(fbias, (frames, N), (ldfb_, 1)).double()
        acc = acc + fb.repeat_interleave(rows_per_frame, dim=0)[:rows]
    if act == ACT_GEGLU:
        bn = block_n or pick_block_n(N, act)
        half = bn // 2
        t = acc.reshape(rows, N // bn, bn)
        acc = (t[..., :half] * F.gelu(t[..., half:])).reshape(rows, n_out)       # value * gelu_erf(gate)
    elif act == ACT_SILU:
        acc = F.silu(acc)
    res = s0 * acc
    if r1 is not None:
        res = res + s1 * _strided(r1, (rows, n_out), (ldr1 or n_out, 1)).double()
    if r2 is not None:
        res = res + s2 * _strided(r2, (rows, n_out), (ldr2 or n_out, 1)).double()
    _store(_strided(out, (rows, n_out), (ldd, 1)), res)
    return out


# ---------------------------------------------------------------------------------------------------------------
# norms
# ---------------------------------------------------------------------------------------------------------------
def groupnorm_stats(x, stats, rows_per_sample, nsamples, c, ldx=None, groups=32, pre_zeroed=False):
    assert x.dtype == BF and stats.dtype == torch.float64
    ldx = c if ldx is None else ldx
    v = _strided(x, (nsamples, rows_per_sample, groups, c // groups), (rows_per_sample * ldx, ldx, c // groups, 1))
    v = v.double()
    if not pre_zeroed:
        stats.zero_()
    st = stats.view(nsamples, groups, 2)
    st[..., 0] += v.sum(dim=(1, 3))
    st[..., 1] += (v * v).sum(dim=(1, 3))
    return stats


def groupnorm_workspace(device):
    return torch.zeros(8, dtype=torch.uint8)


def groupnorm(x, y, gamma, beta, rows_per_sample, nsamples, c, eps, silu, workspace, ldx=None, groups=32):
    """single-launch GroupNorm = statistics + apply"""
    st = torch.zeros(nsamples, groups, 2, dtype=torch.float64, device=x.device)
    groupnorm_stats(x, st, rows_per_sample, nsamples, c, ldx=ldx, groups=groups, pre_zeroed=True)
    groupnorm_apply(x, y, st, gamma, beta, rows_per_sample, nsamples, c, eps, silu, ldx=ldx, groups=groups)
    return y


def groupnorm_apply(x, y, stats, gamma, beta, rows_per_sample, nsamples, c, eps, silu, ldx=None, groups=32):
    ldx = c if ldx is None else ldx
    cpg = c // groups
    n = rows_per_sample * cpg                                       # the kernel divides by the LOCAL element count
    st = stats.reshape(-1)[: nsamples * groups * 2].view(nsamples, groups, 2)
    mean = st[..., 0] / n
    rstd = (st[..., 1] / n - mean * mean + eps).rsqrt()
    v = _strided(x, (nsamples, rows_per_sample, groups, cpg), (rows_per_sample * ldx, ldx, cpg, 1)).double()
    v = (v - mean.double()[:, None, :, None]) * rstd.double()[:, None, :, None]
    v = v.reshape(nsamples, rows_per_sample, c) * gamma.double() + beta.double()
    if silu:
        v = F.silu(v)
    _store(_strided(y, (nsamples * rows_per_sample, c), (c, 1)), v.reshape(-1, c))
    return y


def layernorm(x, y, gamma, beta, rows, c, eps=1e-5, add=None, ysum=None, rows_per_frame=1):
    v = _strided(x, (rows, c), (c, 1)).double()
    if add is not None:
        v = v + add.double().reshape(-1, c).repeat_interleave(rows_per_frame, dim=0)[:rows]
        if ysum is not None:
            v = v.to(BF).double()                                   # rounded once: residual stream == LN input
            _store(_strided(ysum, (rows, c), (c, 1)), v)
    _store(_strided(y, (rows, c), (c, 1)), F.layer_norm(v, (c,), gamma.double(), beta.double(), eps))
    return y


def softmax_rows_f32(x, y, rows, n, scale=1.0):
    _store(y.view(rows, n), torch.softmax(x.view(rows, n).double() * scale, dim=-1))
    return y


# ---------------------------------------------------------------------------------------------------------------
# deterministic GroupNorm (v3d_groupnorm_det_blocks, _partials, _fold_apply, _det)
#
# A sample's rows are cut into blocks of min(256, hw) rows that never straddle a frame; a block's (sum, sumsq) per
# group is summed in fp64 and stored as fp32 (the kernel's fp32 tree rounds differently, so the stand-in matches it to
# fp32 rounding, not bit for bit); the per-sample fold adds the pairs in fp64 in the kernel's order (lane l of 32 adds
# blocks l, l + 32, ... in turn, then an xor-shuffle tree).  What the stand-ins share with the kernels is the property
# the host schedules rely on: a block's pair depends on that block's rows only, so a frame-sharded schedule that
# gathers the pairs correctly reproduces the unsharded one BIT FOR BIT.
# ---------------------------------------------------------------------------------------------------------------
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
    pairs = block_pairs(x, rows_per_sample, hw, nsamples, c, ldx=ldx, groups=groups)
    nblk = pairs.shape[1]
    ldp = nblk if ldp is None else ldp
    _strided(partials, (nsamples, nblk, groups, 2), (ldp * groups * 2, groups * 2, 2, 1)).copy_(pairs)
    return partials


def groupnorm_fold_apply(x, y, partials, gamma, beta, rows_per_sample, nsamples, c, eps, silu, nblocks,
                         count_rows=None, ldx=None, groups=32):
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
    """single launch = partials + fold/apply"""
    nblk = groupnorm_det_blocks(rows_per_sample, hw)
    part = torch.empty(nsamples, nblk, groups, 2, dtype=torch.float32, device=x.device)
    groupnorm_partials(x, part, rows_per_sample, hw, nsamples, c, ldx=ldx, groups=groups)
    groupnorm_fold_apply(x, y, part, gamma, beta, rows_per_sample, nsamples, c, eps, silu, nblk, ldx=ldx,
                         groups=groups)
    return y


# ---------------------------------------------------------------------------------------------------------------
# attention (head dim 64)
# ---------------------------------------------------------------------------------------------------------------
def _heads(t, n, tok, nheads):
    return t.double().reshape(n, tok, nheads, 64).transpose(1, 2)


def attention_spatial(qkv, out, nbatch, ntok, nheads, scale):
    c, ld = nheads * 64, qkv.stride(0)
    q, k, v = (_strided(qkv[:, i * c:], (nbatch * ntok, c), (ld, 1)) for i in range(3))
    o = F.scaled_dot_product_attention(_heads(q, nbatch, ntok, nheads), _heads(k, nbatch, ntok, nheads),
                                       _heads(v, nbatch, ntok, nheads), scale=scale)
    _store(_strided(out, (nbatch * ntok, c), (out.stride(0), 1)), o.transpose(1, 2).reshape(nbatch * ntok, c))
    return out


def attention_cross(q, kv, out, nbatch, nq, nk, nheads, scale, kv_bstride=None):
    c = nheads * 64
    bs = nk if kv_bstride is None else kv_bstride
    assert nk >= 1 and bs >= nk
    qm = _strided(q, (nbatch, nq, nheads, 64), (nq * q.stride(0), q.stride(0), 64, 1)).double().transpose(1, 2)
    km, vm = (_strided(kv[:, i * c:] if i else kv, (nbatch, nk, nheads, 64), (bs * kv.stride(0), kv.stride(0), 64, 1))
              .double().transpose(1, 2) for i in range(2))
    o = F.scaled_dot_product_attention(qm, km, vm, scale=scale)                            # [b, h, nq, 64]
    _store(_strided(out, (nbatch * nq, c), (out.stride(0), 1)), o.transpose(1, 2).reshape(nbatch * nq, c))
    return out


def _attend(q, k, v, scale):
    """softmax(q k^T scale) v in fp64, written out: q [..., tq, 64], k / v [..., tk, 64].  The dense and the
    frame-sharded temporal attention share it, so a sharded run equals the unsharded one to the last bit wherever the
    schedule and the row table are right."""
    s = torch.einsum("...qd,...kd->...qk", q, k) * scale
    p = torch.exp(s - s.amax(dim=-1, keepdim=True))
    return torch.einsum("...qk,...kd->...qd", p / p.sum(dim=-1, keepdim=True), v)


def attention_temporal(qkv, out, nb, t, s, nheads, scale):
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


# ---------------------------------------------------------------------------------------------------------------
# data movement / small matrices
# ---------------------------------------------------------------------------------------------------------------
def upsample_nearest2x(x, y, n, h, w, c):
    v = x.view(n, h, w, c)
    _store(y.view(n, 2 * h, 2 * w, c), v.repeat_interleave(2, dim=1).repeat_interleave(2, dim=2))
    return y


def copy_channels(src, ld_src, dst, ld_dst, rows, ncols):
    _strided(dst, (rows, ncols), (ld_dst, 1)).copy_(_strided(src, (rows, ncols), (ld_src, 1)))


def im2col3x3(x, y, n, h, w, c, stride, pad, hout, wout, kpad):
    v = x.view(n, h, w, c).double().permute(0, 3, 1, 2)
    v = F.pad(v, (1, 1, 1, 1)) if pad else F.pad(v, (0, 1, 0, 1))
    cols = F.unfold(v, kernel_size=3, stride=stride)                                       # [n, c*9, L], (c, ky, kx)
    cols = cols.reshape(n, c, 9, hout * wout).permute(0, 3, 2, 1).reshape(n * hout * wout, 9 * c)   # (tap, c)
    full = torch.zeros(n * hout * wout, kpad, dtype=torch.float64, device=x.device)
    full[:, : 9 * c] = cols
    _store(y.view(n * hout * wout, kpad), full)
    return y


def nchw_f32_to_nhwc_bf16(x, y, scale=1.0):
    n, c, h, w = x.shape
    _store(y.view(n, h, w, c), x.double().permute(0, 2, 3, 1) * scale)
    return y


def nhwc_to_nchw_f32(x, y, n, c, hw, ldx, scale=1.0):
    v = _strided(x, (n, hw, c), (hw * ldx, ldx, 1)).double() * scale
    y.view(n, c, hw).copy_(v.transpose(1, 2))
    return y


def _act(v, kind):
    return F.silu(v) if kind == ACT_SILU else v


def small_linear(x, w, bias, y, *, act_in=ACT_NONE, act_out=ACT_NONE, accumulate=False):
    xin = _act(x.double(), act_in)
    if x.shape[1] % 64 == 0 and act_out == ACT_NONE:
        xin = xin.to(BF).double()                                    # tensor-core path: operand converted to bf16
    r = xin @ w.double().t()
    if bias is not None:
        r = r + bias.double()
    r = _act(r, act_out)
    if accumulate:
        y += r
    else:
        y.copy_(r)
    return y


def timestep_embedding(t, out, dim, max_period=10000.0):
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    args = t.float()[:, None] * freqs[None]                         # fp32 like the kernel and the reference
    out.copy_(torch.cat([torch.cos(args), torch.sin(args)], dim=-1))
    return out


def time_mix_conv(x, ldx, w, bias, y, nb, t, hw, c):
    v = _strided(x, (nb, t, hw, c), (t * hw * ldx, hw * ldx, ldx, 1)).double().permute(0, 3, 1, 2)   # [b, c, t, hw]
    o = F.conv3d(v.unsqueeze(-1), w.double().reshape(c, c, 3, 1, 1), bias.double(), padding=(1, 0, 0)).squeeze(-1)
    y.view(nb, t, c, hw).copy_(o.permute(0, 2, 1, 3))
    return y


# ---------------------------------------------------------------------------------------------------------------
# sampler arithmetic (fp32, elementwise; sampler.cu)
# ---------------------------------------------------------------------------------------------------------------
def _per_sample(v, like):
    return v.float().reshape(-1, *([1] * (like.dim() - 1)))


def edm_scale_input(x, sigma, y, c_noise, nsamples, per_sample):
    s = _per_sample(sigma, x)
    y.copy_(x * (1.0 / torch.sqrt(s * s + 1.0)))
    if c_noise is not None:
        c_noise.copy_(0.25 * torch.log(sigma.float()).reshape(c_noise.shape))
    return y


def edm_denoise_combine(net, x, sigma, out, nsamples, per_sample):
    s = _per_sample(sigma, x)
    d = s * s + 1.0
    out.copy_(net * (-s / torch.sqrt(d)) + x * (1.0 / d))
    return out


def cfg_combine(den, scale, out, b, t, per_sample):
    half = b * t
    xu, xc = den[:half], den[half:]
    sc = scale.float().reshape(-1)[:t].repeat(b).reshape(half, *([1] * (den.dim() - 1)))
    out.copy_(xu + sc * (xc - xu))
    return out


def euler_step(x, den, sigma_hat, sigma_next, out, nsamples, per_sample):
    sh, sn = _per_sample(sigma_hat, x), _per_sample(sigma_next, x)
    out.copy_(x + (sn - sh) * ((x - den) / sh))
    return out


def heun_step(x, den, x_euler, den2, sigma_hat, sigma_next, out, nsamples, per_sample):
    sh, sn = _per_sample(sigma_hat, x), _per_sample(sigma_next, x)
    d = (x - den) / sh
    d2 = (x_euler - den2) / sn.clamp_min(1e-30)
    out.copy_(torch.where(sn > 0, x + ((d + d2) / 2.0) * (sn - sh), x_euler))
    return out


# The ancestral / DPM++ / LMS steps: one operation per rounding in the kernel's order, with every scalar held as a 0-dim
# tensor on the data's device (a python scalar would let CUDA torch divide by multiplying with the reciprocal), so
# that tests/test_samplers_gpu.py can hold them against the kernels bit for bit.
def _s(v: float, like: torch.Tensor) -> torch.Tensor:
    return torch.tensor(float(v), dtype=torch.float32, device=like.device)


def _with_noise(r, noise, s_noise, sigma_up, sigma_next):
    return r + (noise * _s(s_noise, r)) * _s(sigma_up, r) if sigma_next > 0 else r


def _euler(x, den, sigma, sigma_down):
    sg = _s(sigma, x)
    return x + (_s(sigma_down, x) - sg) * ((x - den) / sg)


def ancestral_euler_step(x, den, noise, out, sigma, sigma_down, sigma_up, sigma_next, s_noise, nsamples, per_sample):
    out.copy_(_with_noise(_euler(x, den, sigma, sigma_down), noise, s_noise, sigma_up, sigma_next))
    return out


def dpmpp2s_stage(x, den, out, m1, m2, nsamples, per_sample):
    out.copy_(_s(m1, x) * x - _s(m2, x) * den)
    return out


def dpmpp2s_step(x, den, den2, noise, out, sigma, sigma_down, sigma_up, sigma_next, s_noise, m3, m4, nsamples,
                 per_sample):
    r = _s(m3, x) * x - _s(m4, x) * den2 if sigma_down > 0 else _euler(x, den, sigma, sigma_down)
    out.copy_(_with_noise(r, noise, s_noise, sigma_up, sigma_next))
    return out


def dpmpp2m_step(x, den, hist, out, m1, m2, m3, m4, second_order, nsamples, per_sample):
    dd = _s(m3, x) * den - _s(m4, x) * hist if second_order else den
    r = _s(m1, x) * x - _s(m2, x) * dd
    hist.copy_(den)
    out.copy_(r)
    return out


def lms_step(x, den, ring, out, sigma, coeffs, slots, nsamples, per_sample):
    assert 1 <= len(coeffs) <= 8 and len(coeffs) == len(slots) and ring.shape[0] >= len(coeffs)
    ring[slots[0]].copy_((x - den) / _s(sigma, x))
    acc = _s(coeffs[0], x) * ring[slots[0]]
    for c, k in zip(coeffs[1:], slots[1:]):
        acc = acc + _s(c, x) * ring[k]
    out.copy_(x + acc)
    return out


def frames_nchw_to_u8(x, y):
    v = torch.clamp((x.float() + 1.0) / 2.0, 0.0, 1.0) * 255.0
    y.copy_(v.permute(0, 2, 3, 1).to(torch.uint8))                  # truncating cast, like numpy astype
    return y


# ---------------------------------------------------------------------------------------------------------------
# PixelNeRF (fp32, through oracle/ref_pixelnerf.py)
#
# They read and write the same buffers as the kernels: rays [R, 8], limits (set to "no fallback needed": the stand-in
# applies it itself), feat [R, 128], rgb / feats NCHW.  Weights are the packed bf16 images the kernels read, so the
# stand-ins see the kernels' weights.
# ---------------------------------------------------------------------------------------------------------------
def pixelnerf_rays(cams, render_size, rays, limits, box=True, box_half=1.0):
    o, d, ts, te = ref_pixelnerf.rays(cams, render_size, box=box)
    rays.copy_(torch.cat([o.reshape(-1, 3), d.reshape(-1, 3), ts.reshape(-1, 1), te.reshape(-1, 1)], 1))
    limits.fill_(-1)
    return rays


def _mlp(x, mlp, k_in):
    w1, b1, w2, b2, w3, b3 = mlp
    x = torch.relu(x @ w1[:, :k_in].float().T + b1).bfloat16().float()
    x = torch.relu(x @ w2.float().T + b2).bfloat16().float()
    return x @ w3.float().T + b3


def pixelnerf_render(rays, limits, jitter, src, src_w2c, src_k, rays_per_batch, ns, flags, inv_near, inv_far, mlp,
                     d_in, feat):
    n = rays.shape[0]
    o, d, ts, te = rays[None, :, :3], rays[None, :, 3:6], rays[None, :, 6], rays[None, :, 7]
    disp = bool(flags & real_ops.PNERF_DISPARITY)
    pts = ref_pixelnerf.sample_points(o, d, ts, te, jitter, ns, disp, 1.0 / inv_near, 1.0 / inv_far).reshape(ns, n, 3)
    B, S, C, H, W = src.shape
    pts_b = pts.permute(1, 0, 2).reshape(B, -1, 3)  # B (rays ns) 3
    proj = torch.einsum("bsij,bmj->bsmi", src_w2c, torch.cat([pts_b, torch.ones_like(pts_b[..., :1])], -1))
    xy = -proj[..., :2] / proj[..., 2:]
    x = xy[..., 0] * src_k[..., 0, None] + src_k[..., 2, None]
    y = -xy[..., 1] * src_k[..., 1, None] + src_k[..., 3, None]
    grid = (torch.stack([x, y], -1) * 2 - 1).reshape(B * S, -1, 1, 2)
    joint = F.grid_sample(src.flatten(0, 1), grid, mode="nearest" if flags & real_ops.PNERF_NEAREST else "bilinear",
                          padding_mode="zeros" if flags & real_ops.PNERF_ZEROS else "border", align_corners=True)
    joint = joint.reshape(B, S, C, -1).permute(0, 1, 3, 2)  # B S (rays ns) C
    parts = [joint.mean(1)]
    if flags & real_ops.PNERF_STD:
        parts.append(joint.std(1) if S > 1 else torch.zeros_like(parts[0]))
    if flags & real_ops.PNERF_POSENC:
        parts.append(ref_pixelnerf._pos_enc(pts_b))
    red = torch.cat(parts, -1).reshape(n, ns, d_in).bfloat16().float()
    out = _mlp(red, mlp, d_in)
    w = torch.softmax(out[..., 128:129], dim=1)
    feat.copy_((out[..., :128] * w).sum(1))
    return feat


def pixelnerf_decode(feat, hw, mlp, rgb, feats):
    out = _mlp(feat.bfloat16().float(), mlp, 128)
    n = feat.shape[0] // hw
    rgb.copy_(torch.sigmoid(out[:, :3]).reshape(n, hw, 3).permute(0, 2, 1))
    feats.copy_(out[:, 3:131].reshape(n, hw, 128).permute(0, 2, 1))
    return rgb, feats


# ---------------------------------------------------------------------------------------------------------------
# installation
# ---------------------------------------------------------------------------------------------------------------
# every entry point patched() replaces; the host-side helpers among them launch nothing and are neither counted nor
# recorded
ENTRY_POINTS = ["launch_count", "gemm", "groupnorm_stats", "groupnorm_apply", "groupnorm", "groupnorm_workspace",
                "groupnorm_det_blocks", "groupnorm_det_workspace_bytes", "groupnorm_det_workspace",
                "groupnorm_partials", "groupnorm_fold_apply", "groupnorm_det", "layernorm", "softmax_rows_f32", "attention_spatial",
                "attention_cross", "attention_temporal", "attention_temporal_kv", "upsample_nearest2x",
                "copy_channels", "im2col3x3", "nchw_f32_to_nhwc_bf16", "nhwc_to_nchw_f32", "small_linear",
                "timestep_embedding", "time_mix_conv", "edm_scale_input", "edm_denoise_combine", "cfg_combine",
                "euler_step", "heun_step", "ancestral_euler_step", "dpmpp2s_stage", "dpmpp2s_step", "dpmpp2m_step",
                "lms_step", "frames_nchw_to_u8", "pixelnerf_rays", "pixelnerf_render", "pixelnerf_decode",
                "require_current_device"]
HOST_HELPERS = {"launch_count", "groupnorm_workspace", "groupnorm_det_blocks", "groupnorm_det_workspace_bytes",
                "groupnorm_det_workspace", "require_current_device"}


def _describe(v):
    """An argument as the launch record keeps it: tensors by shape, dtype and strides, floats to 9 digits."""
    if isinstance(v, torch.Tensor):
        return ("T", tuple(v.shape), str(v.dtype), tuple(v.stride()))
    if isinstance(v, (list, tuple)):
        return tuple(_describe(e) for e in v)
    if isinstance(v, float):
        return round(v, 9)
    return v


def _launch(name, fn, record):
    def launch(*args, **kw):
        _launches[name] += 1
        if record is not None:
            record.append((name, _describe(args), tuple(sorted((k, _describe(v)) for k, v in kw.items()))))
        return fn(*args, **kw)
    return launch


@contextlib.contextmanager
def patched(record: list | None = None):
    """Install the stand-ins on v3d_b200.ops for the duration of a test (every other op keeps its CUDA-only body).

    Yields the per-entry-point launch Counter (cumulative over the whole session: take differences).  With `record`,
    every launch is also appended to it as (name, described args, sorted described kwargs).  A stand-in that calls
    another one calls the module function, so it counts and records as the one launch it stands for."""
    saved = {n: getattr(real_ops, n) for n in ENTRY_POINTS}
    try:
        for n in ENTRY_POINTS:
            fn = globals()[n]
            setattr(real_ops, n, fn if n in HOST_HELPERS else _launch(n, fn, record))
        yield _launches
    finally:
        for n, f in saved.items():
            setattr(real_ops, n, f)
