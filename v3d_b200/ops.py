"""Thin torch-tensor wrappers over the C ABI (include/v3d_b200.h).

torch is used here only as the owner of device memory and of the current CUDA stream; every function
forwards raw pointers to libv3d_b200.so and raises RuntimeError if the library reports an error.
Activations are bf16 token-major / NHWC ([rows, C]); see DESIGN.md for the layout contract.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from . import _lib
from ._lib import GemmArgs

ACT_NONE, ACT_SILU, ACT_GEGLU = 0, 1, 2


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _ptr(t: Optional[torch.Tensor]) -> Optional[int]:
    return None if t is None else t.data_ptr()


def _need(t: torch.Tensor, dtype, name: str) -> None:
    if not t.is_cuda:
        raise RuntimeError(f"{name}: expected a CUDA tensor (there is no CPU path in v3d_b200)")
    if t.dtype != dtype:
        raise RuntimeError(f"{name}: expected dtype {dtype}, got {t.dtype}")


def require_current_device(t: torch.Tensor, who: str) -> None:
    """The one refusal of the package's entry points: every module forward, sampler call and weight packing calls it
    once.  There is no CPU path, so a tensor that is not on CUDA is refused.  The library launches on the CURRENT
    device's current stream and caches per-device kernel attributes per process (one process per GPU is the deployment
    model): a tensor on another device would be launched on the wrong stream, so it is refused too."""
    if not t.is_cuda:
        raise RuntimeError(f"{who} needs CUDA tensors (got {t.device}); there is no CPU fallback")
    if t.device.index != torch.cuda.current_device():
        raise RuntimeError(f"{who}: tensor on cuda:{t.device.index} but the current device is cuda:"
                           f"{torch.cuda.current_device()}; call torch.cuda.set_device(...) first (one process per GPU)")


def launch_count() -> int:
    return int(_lib.load().v3d_launch_count())


def pick_block_n(n: int, act: int = ACT_NONE) -> int:
    return int(_lib.load().v3d_gemm_pick_block_n(n, act))


def geglu_perm(n_out: int, block_n: int) -> torch.Tensor:
    """Row permutation that packs a GEGLU projection [2*n_out, K] tile-wise (value rows | gate rows)."""
    buf = (C.c_int32 * (2 * n_out))()
    _lib.check(_lib.load().v3d_geglu_pack_rows(n_out, block_n, buf), "v3d_geglu_pack_rows")
    return torch.tensor(list(buf), dtype=torch.long)


def gemm(a: torch.Tensor, w: torch.Tensor, out: torch.Tensor, *, K: int, N: int,
         rows_per_batch: int, batch: int = 1, lda: Optional[int] = None, ldb: Optional[int] = None,
         ldd: Optional[int] = None, a_batch_stride: int = 0, b_batch_stride: int = 0,
         bias: Optional[torch.Tensor] = None, fbias: Optional[torch.Tensor] = None, rows_per_frame: int = 1,
         ldfb: int = 0,
         r1: Optional[torch.Tensor] = None, ldr1: int = 0, r2: Optional[torch.Tensor] = None, ldr2: int = 0,
         s0: float = 1.0, s1: float = 1.0, s2: float = 1.0, act: int = ACT_NONE, ntaps: int = 1,
         tap_shift: int = 0, conv: Optional[tuple] = None, block_n: int = 0, transposed: bool = False,
         valid_cols: int = 0, accumulate: bool = False, a_rows: int = 0, a_row0: int = 0,
         kv: Optional[tuple] = None) -> torch.Tensor:
    """General entry to v3d_gemm_bf16. `conv=(n, h, w)` selects the implicit 3x3 conv gather; `a_rows` / `a_row0`
    describe a halo'd A operand (frame-sharded temporal convs, see include/v3d_b200.h)."""
    _need(a, torch.bfloat16, "gemm A")
    _need(w, torch.bfloat16, "gemm B")
    g = GemmArgs()
    g.A, g.B, g.D = a.data_ptr(), w.data_ptr(), out.data_ptr()
    g.bias, g.fbias = _ptr(bias), _ptr(fbias)
    g.R1, g.R2 = _ptr(r1), _ptr(r2)
    if bias is not None:
        _need(bias, torch.float32, "gemm bias")
    if fbias is not None:
        _need(fbias, torch.float32, "gemm fbias")
    ktot = K * (9 if conv is not None else ntaps)
    g.lda = K if lda is None else lda
    g.ldb = ktot if ldb is None else ldb
    n_out = N // 2 if act == ACT_GEGLU else N
    g.ldd = n_out if ldd is None else ldd
    g.ldr1 = ldr1 or n_out
    g.ldr2 = ldr2 or n_out
    g.a_batch_stride, g.b_batch_stride = a_batch_stride, b_batch_stride
    g.batch, g.rows_per_batch = batch, rows_per_batch
    g.N, g.K = N, K
    g.ntaps, g.tap_shift = ntaps, tap_shift
    g.rows_per_frame = rows_per_frame
    g.ldfb = ldfb
    g.act = act
    g.out_fp32 = 1 if out.dtype == torch.float32 else 0
    if conv is not None:
        g.conv_n, g.conv_h, g.conv_w = conv
    g.block_n = block_n
    g.out_transposed = 1 if transposed else 0
    g.valid_cols = valid_cols
    g.accumulate = 1 if accumulate else 0
    g.s0, g.s1, g.s2 = s0, s1, s2
    g.a_rows, g.a_row0 = a_rows, a_row0
    if kv is not None:
        # fused GEMM -> all-gather: (first scattered column, [destination base addresses], destination row stride)
        col0, dsts, ld = kv
        g.kv_col0, g.kv_n, g.kv_ld = col0, len(dsts), ld
        for i, d in enumerate(dsts):
            g.kv_dst[i] = d
    _lib.check(_lib.load().v3d_gemm_bf16(C.byref(g), _stream()), "v3d_gemm_bf16")
    return out


def groupnorm_stats(x: torch.Tensor, stats: torch.Tensor, rows_per_sample: int, nsamples: int, c: int,
                    ldx: Optional[int] = None, groups: int = 32, pre_zeroed: bool = False) -> torch.Tensor:
    _need(x, torch.bfloat16, "groupnorm x")
    _need(stats, torch.float64, "groupnorm stats")
    _lib.check(_lib.load().v3d_groupnorm_stats(x.data_ptr(), stats.data_ptr(), rows_per_sample, nsamples, c,
                                               c if ldx is None else ldx, groups, 1 if pre_zeroed else 0,
                                               _stream()), "v3d_groupnorm_stats")
    return stats


def groupnorm_apply(x: torch.Tensor, y: torch.Tensor, stats: torch.Tensor, gamma: torch.Tensor,
                    beta: torch.Tensor, rows_per_sample: int, nsamples: int, c: int, eps: float, silu: bool,
                    ldx: Optional[int] = None, groups: int = 32) -> torch.Tensor:
    _need(gamma, torch.float32, "groupnorm gamma")
    _lib.check(_lib.load().v3d_groupnorm_apply(x.data_ptr(), y.data_ptr(), stats.data_ptr(), gamma.data_ptr(),
                                               beta.data_ptr(), rows_per_sample, nsamples, c,
                                               c if ldx is None else ldx, groups, eps, 1 if silu else 0,
                                               _stream()), "v3d_groupnorm_apply")
    return y


def groupnorm_workspace(device) -> torch.Tensor:
    """Zeroed workspace of the single-launch GroupNorm (barrier state + per-CTA partials); one per stream."""
    return torch.zeros(int(_lib.load().v3d_groupnorm_workspace_bytes()), device=device, dtype=torch.uint8)


def groupnorm(x: torch.Tensor, y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, rows_per_sample: int,
              nsamples: int, c: int, eps: float, silu: bool, workspace: torch.Tensor, ldx: Optional[int] = None,
              groups: int = 32) -> torch.Tensor:
    """y = act(GroupNorm(x)) in one launch (statistics, grid barrier, apply); deterministic."""
    _need(x, torch.bfloat16, "groupnorm x")
    _need(gamma, torch.float32, "groupnorm gamma")
    _need(workspace, torch.uint8, "groupnorm workspace")
    _lib.check(_lib.load().v3d_groupnorm(x.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                         rows_per_sample, nsamples, c, c if ldx is None else ldx, groups, eps,
                                         1 if silu else 0, workspace.data_ptr(), workspace.numel(), _stream()),
               "v3d_groupnorm")
    return y


def deterministic() -> bool:
    """Deterministic mode: on under torch.use_deterministic_algorithms(True) or V3D_DETERMINISTIC=1.  The modules then
    take the GroupNorm statistics from the block partials below, which do not depend on the launch grid, nsamples or a
    sharded plan; every other kernel is deterministic in both modes."""
    return torch.are_deterministic_algorithms_enabled() or os.environ.get("V3D_DETERMINISTIC", "0") == "1"


def groupnorm_det_blocks(rows_per_sample: int, hw: int) -> int:
    """Blocks per sample of the deterministic statistics (rows of min(256, hw), never straddling a frame)."""
    n = int(_lib.load().v3d_groupnorm_det_blocks(rows_per_sample, hw))
    if n <= 0:
        raise RuntimeError(f"groupnorm_det_blocks: hw={hw} does not divide rows_per_sample={rows_per_sample}")
    return n


def groupnorm_det_workspace_bytes(rows_per_sample: int, hw: int, nsamples: int, groups: int = 32) -> int:
    return int(_lib.load().v3d_groupnorm_det_workspace_bytes(rows_per_sample, hw, nsamples, groups))


def groupnorm_partials(x: torch.Tensor, partials: torch.Tensor, rows_per_sample: int, hw: int, nsamples: int, c: int,
                       ldx: Optional[int] = None, groups: int = 32, ldp: Optional[int] = None) -> torch.Tensor:
    """partials: fp32 [nsamples, ldp, groups, 2] (a view may start at a block offset of a wider buffer; ldp = its
    blocks per sample, default: this shape's)."""
    _need(x, torch.bfloat16, "groupnorm x")
    _need(partials, torch.float32, "groupnorm partials")
    ldp = groupnorm_det_blocks(rows_per_sample, hw) if ldp is None else ldp
    _lib.check(_lib.load().v3d_groupnorm_partials(x.data_ptr(), partials.data_ptr(), rows_per_sample, hw, nsamples, c,
                                                  c if ldx is None else ldx, groups, ldp, _stream()),
               "v3d_groupnorm_partials")
    return partials


def groupnorm_fold_apply(x: torch.Tensor, y: torch.Tensor, partials: torch.Tensor, gamma: torch.Tensor,
                         beta: torch.Tensor, rows_per_sample: int, nsamples: int, c: int, eps: float, silu: bool,
                         nblocks: int, count_rows: Optional[int] = None, ldx: Optional[int] = None,
                         groups: int = 32) -> torch.Tensor:
    """y = act(GroupNorm(x)) with the statistics folded from `nblocks` block partials per sample; count_rows = the rows
    they cover (default rows_per_sample; the whole video's when x holds one rank's frames)."""
    _need(x, torch.bfloat16, "groupnorm x")
    _need(partials, torch.float32, "groupnorm partials")
    _need(gamma, torch.float32, "groupnorm gamma")
    _lib.check(_lib.load().v3d_groupnorm_fold_apply(x.data_ptr(), y.data_ptr(), partials.data_ptr(), gamma.data_ptr(),
                                                    beta.data_ptr(), rows_per_sample, nsamples, c,
                                                    c if ldx is None else ldx, groups, nblocks,
                                                    rows_per_sample if count_rows is None else count_rows, eps,
                                                    1 if silu else 0, _stream()), "v3d_groupnorm_fold_apply")
    return y


def groupnorm_det_workspace(device, nbytes: int) -> torch.Tensor:
    """Zeroed workspace of the single-launch deterministic GroupNorm (barrier state + block partials)."""
    return torch.zeros(nbytes, device=device, dtype=torch.uint8)


def groupnorm_det(x: torch.Tensor, y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, rows_per_sample: int,
                  hw: int, nsamples: int, c: int, eps: float, silu: bool, workspace: torch.Tensor,
                  ldx: Optional[int] = None, groups: int = 32) -> torch.Tensor:
    """groupnorm_partials + groupnorm_fold_apply in one launch (same bits)."""
    _need(x, torch.bfloat16, "groupnorm x")
    _need(gamma, torch.float32, "groupnorm gamma")
    _need(workspace, torch.uint8, "groupnorm workspace")
    _lib.check(_lib.load().v3d_groupnorm_det(x.data_ptr(), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                             rows_per_sample, hw, nsamples, c, c if ldx is None else ldx, groups, eps,
                                             1 if silu else 0, workspace.data_ptr(), workspace.numel(), _stream()),
               "v3d_groupnorm_det")
    return y


def layernorm(x: torch.Tensor, y: torch.Tensor, gamma: torch.Tensor, beta: torch.Tensor, rows: int, c: int,
              eps: float = 1e-5, add: Optional[torch.Tensor] = None, ysum: Optional[torch.Tensor] = None,
              rows_per_frame: int = 1) -> torch.Tensor:
    _need(x, torch.bfloat16, "layernorm x")
    _need(gamma, torch.float32, "layernorm gamma")
    _lib.check(_lib.load().v3d_layernorm(x.data_ptr(), _ptr(add), _ptr(ysum), y.data_ptr(), gamma.data_ptr(),
                                         beta.data_ptr(), rows, c, rows_per_frame, eps, _stream()),
               "v3d_layernorm")
    return y


def softmax_rows(x: torch.Tensor, rows: int, n: int, scale: float = 1.0) -> torch.Tensor:
    _need(x, torch.bfloat16, "softmax x")
    _lib.check(_lib.load().v3d_softmax_rows(x.data_ptr(), rows, n, scale, _stream()), "v3d_softmax_rows")
    return x


def softmax_rows_f32(x: torch.Tensor, y: torch.Tensor, rows: int, n: int, scale: float = 1.0) -> torch.Tensor:
    _need(x, torch.float32, "softmax x")
    _need(y, torch.bfloat16, "softmax y")
    _lib.check(_lib.load().v3d_softmax_rows_f32(x.data_ptr(), y.data_ptr(), rows, n, scale, _stream()),
               "v3d_softmax_rows_f32")
    return y


def time_mix_conv(x: torch.Tensor, ldx: int, w: torch.Tensor, bias: torch.Tensor, y: torch.Tensor, nb: int, t: int,
                  hw: int, c: int) -> torch.Tensor:
    _need(x, torch.float32, "time_mix_conv x")
    _lib.check(_lib.load().v3d_time_mix_conv(x.data_ptr(), ldx, w.data_ptr(), bias.data_ptr(), y.data_ptr(), nb, t,
                                             hw, c, _stream()), "v3d_time_mix_conv")
    return y


def attention_spatial(qkv: torch.Tensor, out: torch.Tensor, nbatch: int, ntok: int, nheads: int,
                      scale: float) -> torch.Tensor:
    """qkv: [nbatch*ntok, 3*C] packed (q | k | v), out: [nbatch*ntok, C]."""
    _need(qkv, torch.bfloat16, "attention qkv")
    c = nheads * 64
    es = qkv.element_size()
    base = qkv.data_ptr()
    _lib.check(_lib.load().v3d_attention_spatial(base, base + c * es, base + 2 * c * es, out.data_ptr(),
                                                 qkv.shape[-1], out.shape[-1], nbatch, ntok, nheads, scale,
                                                 _stream()), "v3d_attention_spatial")
    return out


def attention_spatial_mma(qkv: torch.Tensor, out: torch.Tensor, nbatch: int, ntok: int, nheads: int,
                          scale: float) -> torch.Tensor:
    """Validation twin of attention_spatial (mma.sync kernel); tests only."""
    _need(qkv, torch.bfloat16, "attention qkv")
    c = nheads * 64
    es = qkv.element_size()
    base = qkv.data_ptr()
    _lib.check(_lib.load().v3d_attention_spatial_mma(base, base + c * es, base + 2 * c * es, out.data_ptr(),
                                                     qkv.shape[-1], out.shape[-1], nbatch, ntok, nheads, scale,
                                                     _stream()), "v3d_attention_spatial_mma")
    return out


MAX_TEMPORAL_FRAMES = 128   # key frames v3d_attention_temporal / _kv take (kMaxTLong, csrc/attention.cu)


def check_temporal_frames(num_frames: int) -> None:
    """Raise before a schedule starts if the video has more view-frames than the temporal attention kernels hold in
    one pass (longer sequences would need an online softmax over key tiles)."""
    if num_frames > MAX_TEMPORAL_FRAMES:
        raise ValueError(f"temporal attention supports at most {MAX_TEMPORAL_FRAMES} frames, got {num_frames}")


def attention_temporal(qkv: torch.Tensor, out: torch.Tensor, nb: int, t: int, s: int, nheads: int,
                       scale: float) -> torch.Tensor:
    _need(qkv, torch.bfloat16, "attention qkv")
    c = nheads * 64
    es = qkv.element_size()
    base = qkv.data_ptr()
    _lib.check(_lib.load().v3d_attention_temporal(base, base + c * es, base + 2 * c * es, out.data_ptr(),
                                                  qkv.shape[-1], out.shape[-1], nb, t, s, nheads, scale,
                                                  _stream()), "v3d_attention_temporal")
    return out


def attention_temporal_kv(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, nb: int, tq: int, s: int, nheads: int,
                          kv_row, kv_bstride, scale: float) -> torch.Tensor:
    """Frame-sharded temporal attention: q = the query columns of the local packed projection ([nb*tq*s, ld_q] view),
    kv = the all-gathered [rows, 2C] K|V buffer, kv_row / kv_bstride = per key frame row offsets (python ints)."""
    _need(q, torch.bfloat16, "attention q")
    _need(kv, torch.bfloat16, "attention kv")
    c = nheads * 64
    tk = len(kv_row)
    rows_t = (C.c_int32 * tk)(*kv_row)
    bstr_t = (C.c_int32 * tk)(*kv_bstride)
    base = kv.data_ptr()
    _lib.check(_lib.load().v3d_attention_temporal_kv(q.data_ptr(), base, base + c * kv.element_size(), out.data_ptr(),
                                                     q.stride(0), kv.stride(0), out.stride(0), nb, tq, tk, s, nheads,
                                                     rows_t, bstr_t, scale, _stream()),
               "v3d_attention_temporal_kv")
    return out


def attention_cross(q: torch.Tensor, kv: torch.Tensor, out: torch.Tensor, nbatch: int, nq: int, nk: int, nheads: int,
                    scale: float, kv_bstride: Optional[int] = None) -> torch.Tensor:
    """Cross-attention over nk context tokens: q = [nbatch*nq, >= C] query rows (a column slice of a wider matrix is
    fine: the row stride is taken from the tensor), kv = K | V in columns [0, C) and [C, 2C) of a row-strided view,
    item b's keys at rows b*kv_bstride + j (default kv_bstride = nk), out = [nbatch*nq, >= C]."""
    _need(q, torch.bfloat16, "attention q")
    _need(kv, torch.bfloat16, "attention kv")
    _need(out, torch.bfloat16, "attention out")
    c = nheads * 64
    base = kv.data_ptr()
    _lib.check(_lib.load().v3d_attention_cross(q.data_ptr(), base, base + c * kv.element_size(), out.data_ptr(),
                                               q.stride(0), kv.stride(0), out.stride(0), nbatch, nq, nk,
                                               nk if kv_bstride is None else kv_bstride, nheads, scale, _stream()),
               "v3d_attention_cross")
    return out


def upsample_nearest2x(x: torch.Tensor, y: torch.Tensor, n: int, h: int, w: int, c: int) -> torch.Tensor:
    _lib.check(_lib.load().v3d_upsample_nearest2x(x.data_ptr(), y.data_ptr(), n, h, w, c, _stream()),
               "v3d_upsample_nearest2x")
    return y


def copy_channels(src: torch.Tensor, ld_src: int, dst: torch.Tensor, ld_dst: int, rows: int, ncols: int) -> None:
    """dst[r, :ncols] = src[r, :ncols] for `rows` rows of two row-strided bf16 buffers (`src` / `dst` may be column
    slices of wider matrices: the views' data pointers carry the column offset, ld_* are the parents' row strides)."""
    _lib.check(_lib.load().v3d_copy_channels(src.data_ptr(), ld_src, dst.data_ptr(), ld_dst, rows, ncols, _stream()),
               "v3d_copy_channels")


def im2col3x3(x: torch.Tensor, y: torch.Tensor, n: int, h: int, w: int, c: int, stride: int, pad: int,
              hout: int, wout: int, kpad: int) -> torch.Tensor:
    _lib.check(_lib.load().v3d_im2col3x3(x.data_ptr(), y.data_ptr(), n, h, w, c, stride, pad, hout, wout, kpad,
                                         _stream()), "v3d_im2col3x3")
    return y


def nchw_f32_to_nhwc_bf16(x: torch.Tensor, y: torch.Tensor, scale: float = 1.0) -> torch.Tensor:
    _need(x, torch.float32, "nchw input")
    n, c, h, w = x.shape
    _lib.check(_lib.load().v3d_nchw_f32_to_nhwc_bf16(x.data_ptr(), y.data_ptr(), n, c, h, w, scale, _stream()),
               "v3d_nchw_f32_to_nhwc_bf16")
    return y


def nhwc_to_nchw_f32(x: torch.Tensor, y: torch.Tensor, n: int, c: int, hw: int, ldx: int,
                     scale: float = 1.0) -> torch.Tensor:
    _lib.check(_lib.load().v3d_nhwc_to_nchw_f32(x.data_ptr(), y.data_ptr(), n, c, hw, ldx,
                                                1 if x.dtype == torch.float32 else 0, scale, _stream()),
               "v3d_nhwc_to_nchw_f32")
    return y


def small_linear(x: torch.Tensor, w: torch.Tensor, bias: Optional[torch.Tensor], y: torch.Tensor, *,
                 act_in: int = ACT_NONE, act_out: int = ACT_NONE, accumulate: bool = False) -> torch.Tensor:
    """y[M,N] fp32 (+)= act_out(act_in(x) @ w.T + bias) for the M<=64-row embedding linears. x and y may be column
    slices of wider row-major buffers (row strides are taken from the tensors).

    K % 64 == 0 and no output activation: tensor-core path — W is the 128-row operand streamed once by TMA,
    act_in(x) is the 64-row operand, results are stored transposed (v3d_gemm_bf16 out_transposed).
    Otherwise: the SIMT kernel v3d_small_linear."""
    _need(x, torch.float32, "small_linear x")
    _need(w, torch.bfloat16, "small_linear w")
    m, k = x.shape
    n = w.shape[0]
    if x.stride(1) != 1 or y.stride(1) != 1 or w.shape[1] != k or not w.is_contiguous():
        raise RuntimeError("small_linear: bad strides/shapes")
    ldx, ldy = x.stride(0), y.stride(0)
    lib = _lib.load()
    if k % 64 == 0 and act_out == ACT_NONE:
        for m0 in range(0, m, 64):
            mm = min(64, m - m0)
            xb = torch.empty(64, k, device=x.device, dtype=torch.bfloat16)
            _lib.check(lib.v3d_prep_small_x(x.data_ptr() + m0 * ldx * 4, ldx, xb.data_ptr(), mm, k, act_in,
                                            _stream()), "v3d_prep_small_x")
            g = GemmArgs()
            g.A, g.B, g.D, g.bias = w.data_ptr(), xb.data_ptr(), y.data_ptr() + m0 * ldy * 4, _ptr(bias)
            g.lda = g.ldb = k
            g.ldd = ldy
            g.batch, g.rows_per_batch, g.N, g.K, g.ntaps, g.rows_per_frame = 1, n, 64, k, 1, 1
            g.out_fp32, g.out_transposed, g.valid_cols, g.accumulate = 1, 1, mm, 1 if accumulate else 0
            g.s0 = g.s1 = g.s2 = 1.0
            _lib.check(lib.v3d_gemm_bf16(C.byref(g), _stream()), "v3d_gemm_bf16(small-M)")
        return y
    for m0 in range(0, m, 64):
        mm = min(64, m - m0)
        _lib.check(lib.v3d_small_linear(x.data_ptr() + m0 * ldx * 4, w.data_ptr(), _ptr(bias),
                                        y.data_ptr() + m0 * ldy * 4, mm, k, n, act_in, act_out,
                                        1 if accumulate else 0, ldx, ldy, _stream()), "v3d_small_linear")
    return y


def timestep_embedding(t: torch.Tensor, out: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    _need(t, torch.float32, "timestep_embedding t")
    _lib.check(_lib.load().v3d_timestep_embedding(t.data_ptr(), out.data_ptr(), t.numel(), dim, max_period,
                                                  _stream()), "v3d_timestep_embedding")
    return out


def edm_scale_input(x, sigma, y, c_noise, nsamples: int, per_sample: int):
    _lib.check(_lib.load().v3d_edm_scale_input(x.data_ptr(), sigma.data_ptr(), y.data_ptr(), _ptr(c_noise),
                                               nsamples, per_sample, _stream()), "v3d_edm_scale_input")
    return y


def edm_denoise_combine(net, x, sigma, out, nsamples: int, per_sample: int):
    _lib.check(_lib.load().v3d_edm_denoise_combine(net.data_ptr(), x.data_ptr(), sigma.data_ptr(),
                                                   out.data_ptr(), nsamples, per_sample, _stream()),
               "v3d_edm_denoise_combine")
    return out


def cfg_combine(den, scale, out, b: int, t: int, per_sample: int):
    _lib.check(_lib.load().v3d_cfg_combine(den.data_ptr(), scale.data_ptr(), out.data_ptr(), b, t, per_sample,
                                           _stream()), "v3d_cfg_combine")
    return out


def euler_step(x, den, sigma_hat, sigma_next, out, nsamples: int, per_sample: int):
    _lib.check(_lib.load().v3d_euler_step(x.data_ptr(), den.data_ptr(), sigma_hat.data_ptr(),
                                          sigma_next.data_ptr(), out.data_ptr(), nsamples, per_sample,
                                          _stream()), "v3d_euler_step")
    return out


def heun_step(x, den, x_euler, den2, sigma_hat, sigma_next, out, nsamples: int, per_sample: int):
    for t, name in ((x, "x"), (den, "den"), (x_euler, "x_euler"), (den2, "den2"), (sigma_hat, "sigma_hat"),
                    (sigma_next, "sigma_next"), (out, "out")):
        _need(t, torch.float32, "heun_step " + name)
    _lib.check(_lib.load().v3d_heun_step(x.data_ptr(), den.data_ptr(), x_euler.data_ptr(), den2.data_ptr(),
                                         sigma_hat.data_ptr(), sigma_next.data_ptr(), out.data_ptr(), nsamples,
                                         per_sample, _stream()), "v3d_heun_step")
    return out


def _need_f32(who: str, **tensors) -> None:
    for name, t in tensors.items():
        _need(t, torch.float32, f"{who} {name}")


def ancestral_euler_step(x, den, noise, out, sigma: float, sigma_down: float, sigma_up: float, sigma_next: float,
                         s_noise: float, nsamples: int, per_sample: int):
    _need_f32("ancestral_euler_step", x=x, den=den, noise=noise, out=out)
    _lib.check(_lib.load().v3d_ancestral_euler_step(x.data_ptr(), den.data_ptr(), noise.data_ptr(), out.data_ptr(),
                                                    sigma, sigma_down, sigma_up, sigma_next, s_noise, nsamples,
                                                    per_sample, _stream()), "v3d_ancestral_euler_step")
    return out


def dpmpp2s_stage(x, den, out, m1: float, m2: float, nsamples: int, per_sample: int):
    _need_f32("dpmpp2s_stage", x=x, den=den, out=out)
    _lib.check(_lib.load().v3d_dpmpp2s_stage(x.data_ptr(), den.data_ptr(), out.data_ptr(), m1, m2, nsamples,
                                             per_sample, _stream()), "v3d_dpmpp2s_stage")
    return out


def dpmpp2s_step(x, den, den2, noise, out, sigma: float, sigma_down: float, sigma_up: float, sigma_next: float,
                 s_noise: float, m3: float, m4: float, nsamples: int, per_sample: int):
    _need_f32("dpmpp2s_step", x=x, den=den, den2=den2, noise=noise, out=out)
    _lib.check(_lib.load().v3d_dpmpp2s_step(x.data_ptr(), den.data_ptr(), den2.data_ptr(), noise.data_ptr(),
                                            out.data_ptr(), sigma, sigma_down, sigma_up, sigma_next, s_noise, m3, m4,
                                            nsamples, per_sample, _stream()), "v3d_dpmpp2s_step")
    return out


def dpmpp2m_step(x, den, hist, out, m1: float, m2: float, m3: float, m4: float, second_order: bool, nsamples: int,
                 per_sample: int):
    _need_f32("dpmpp2m_step", x=x, den=den, hist=hist, out=out)
    _lib.check(_lib.load().v3d_dpmpp2m_step(x.data_ptr(), den.data_ptr(), hist.data_ptr(), out.data_ptr(), m1, m2,
                                            m3, m4, 1 if second_order else 0, nsamples, per_sample, _stream()),
               "v3d_dpmpp2m_step")
    return out


def lms_step(x, den, ring, out, sigma: float, coeffs, slots, nsamples: int, per_sample: int):
    """ring: [ring_slots, *x.shape]; coeffs[j] multiplies the slope stored in ring[slots[j]] (slots[0] receives this
    step's slope)."""
    _need_f32("lms_step", x=x, den=den, ring=ring, out=out)
    order = len(coeffs)
    c_arr = (C.c_float * max(order, 1))(*coeffs)
    s_arr = (C.c_int32 * max(order, 1))(*slots)
    _lib.check(_lib.load().v3d_lms_step(x.data_ptr(), den.data_ptr(), ring.data_ptr(), out.data_ptr(), sigma, c_arr,
                                        s_arr, order, ring.shape[0], nsamples, per_sample, _stream()), "v3d_lms_step")
    return out


def decode_to_u8(x: torch.Tensor, ldx: int, y: torch.Tensor, npix: int):
    _lib.check(_lib.load().v3d_decode_to_u8(x.data_ptr(), ldx, 1 if x.dtype == torch.float32 else 0,
                                            y.data_ptr(), npix, _stream()), "v3d_decode_to_u8")
    return y


def frames_nchw_to_u8(x: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """[T,3,H,W] fp32 in [-1,1] -> [T,H,W,3] uint8 (the wire format of sample_one)."""
    _need(x, torch.float32, "frames")
    t, c, h, w = x.shape
    assert c == 3 and x.is_contiguous() and y.dtype == torch.uint8
    _lib.check(_lib.load().v3d_frames_nchw_to_u8(x.data_ptr(), y.data_ptr(), t, h * w, _stream()),
               "v3d_frames_nchw_to_u8")
    return y


PNERF_STD, PNERF_POSENC, PNERF_NEAREST, PNERF_ZEROS, PNERF_DISPARITY = 1, 2, 4, 8, 16


def _need_contig(name: str, dtype, **ts) -> None:
    for k, t in ts.items():
        _need(t, dtype, f"{name} {k}")
        if not t.is_contiguous():
            raise RuntimeError(f"{name} {k}: expected a contiguous tensor")


def pixelnerf_rays(cams: torch.Tensor, render_size: int, rays: torch.Tensor, limits: torch.Tensor,
                   box: bool = True, box_half: float = 1.0) -> torch.Tensor:
    """cams [ncam, 25] -> rays [ncam * render_size**2, 8] (origin, direction, t_start, t_end); limits: int32 [2]."""
    _need_contig("pixelnerf_rays", torch.float32, cams=cams, rays=rays)
    _need(limits, torch.int32, "pixelnerf_rays limits")
    ncam = cams.numel() // 25
    if cams.numel() != ncam * 25 or ncam == 0 or rays.numel() != ncam * render_size * render_size * 8 \
            or limits.numel() < 2:
        raise RuntimeError(f"pixelnerf_rays: cams {tuple(cams.shape)} / rays {tuple(rays.shape)} / limits "
                           f"{tuple(limits.shape)} do not match [ncam, 25] / [ncam * {render_size}^2, 8] / [2]")
    _lib.check(_lib.load().v3d_pixelnerf_rays(cams.data_ptr(), ncam, render_size, box_half, int(box), rays.data_ptr(),
                                              limits.data_ptr(), _stream()), "v3d_pixelnerf_rays")
    return rays


def _mlp_shapes(name: str, mlp, k1: int) -> None:
    w1, b1, w2, b2, w3, b3 = mlp
    want = ((w1, (128, k1)), (b1, (128,)), (w2, (128, 128)), (b2, (128,)), (w3, (136, 128)), (b3, (136,)))
    for i, (t, shape) in enumerate(want):
        if tuple(t.shape) != shape:
            raise RuntimeError(f"{name}: packed MLP tensor {i} is {tuple(t.shape)}, expected {shape}")


def pixelnerf_render(rays, limits, jitter, src, src_w2c, src_k, rays_per_batch: int, ns: int, flags: int,
                     inv_near: float, inv_far: float, mlp, d_in: int, feat: torch.Tensor) -> torch.Tensor:
    """src [B, S, C, H, W] fp32; src_w2c [B, S, 3, 4]; src_k [B, S, 4]; mlp = (w1, b1, w2, b2, w3, b3) packed as
    include/v3d_b200.h describes; feat out [nrays, 128] fp32.  Every shape relation the kernel relies on is checked
    here: the kernel indexes by them without bounds checks."""
    w1, b1, w2, b2, w3, b3 = mlp
    _need_contig("pixelnerf_render", torch.float32, rays=rays, jitter=jitter, src=src, src_w2c=src_w2c, src_k=src_k,
                 b1=b1, b2=b2, b3=b3, feat=feat)
    _need_contig("pixelnerf_render", torch.bfloat16, w1=w1, w2=w2, w3=w3)
    _need(limits, torch.int32, "pixelnerf_render limits")
    if src.dim() != 5:
        raise RuntimeError(f"pixelnerf_render: src must be [B, S, C, H, W], got {tuple(src.shape)}")
    B, S, Cc, H, W = src.shape
    nrays = rays.shape[0]
    if rays.shape != (nrays, 8) or limits.numel() < 2:
        raise RuntimeError("pixelnerf_render: rays must be [nrays, 8] and limits hold 2 words")
    if rays_per_batch <= 0 or B * rays_per_batch != nrays:
        raise RuntimeError(f"pixelnerf_render: {B} source batches x {rays_per_batch} rays != {nrays} rays "
                           "(the sources' batch must equal the target cameras' batch)")
    if tuple(src_w2c.shape) != (B, S, 3, 4) or tuple(src_k.shape) != (B, S, 4):
        raise RuntimeError(f"pixelnerf_render: src_w2c {tuple(src_w2c.shape)} / src_k {tuple(src_k.shape)} do not "
                           f"match [B={B}, S={S}, 3, 4] / [B, S, 4]")
    want_j = ns if flags & PNERF_DISPARITY else ns * nrays
    if jitter.numel() != want_j:
        raise RuntimeError(f"pixelnerf_render: jitter has {jitter.numel()} values, expected {want_j}")
    _mlp_shapes("pixelnerf_render", mlp, -(-d_in // 64) * 64)
    if tuple(feat.shape) != (nrays, 128):
        raise RuntimeError(f"pixelnerf_render: feat is {tuple(feat.shape)}, expected ({nrays}, 128)")
    _lib.check(_lib.load().v3d_pixelnerf_render(
        rays.data_ptr(), limits.data_ptr(), jitter.data_ptr(), src.data_ptr(), src_w2c.data_ptr(), src_k.data_ptr(),
        nrays, rays_per_batch, S, Cc, H, W, ns, flags, inv_near, inv_far, w1.data_ptr(), d_in, b1.data_ptr(),
        w2.data_ptr(), b2.data_ptr(), w3.data_ptr(), b3.data_ptr(), feat.data_ptr(), _stream()),
        "v3d_pixelnerf_render")
    return feat


def pixelnerf_decode(feat: torch.Tensor, hw: int, mlp, rgb: torch.Tensor, feats: torch.Tensor):
    """feat [nrays, 128] -> rgb [nrays / hw, 3, hw] (sigmoid), feats [nrays / hw, 128, hw]."""
    w1, b1, w2, b2, w3, b3 = mlp
    _need_contig("pixelnerf_decode", torch.float32, feat=feat, b1=b1, b2=b2, b3=b3, rgb=rgb, feats=feats)
    _need_contig("pixelnerf_decode", torch.bfloat16, w1=w1, w2=w2, w3=w3)
    nrays = feat.shape[0]
    if feat.dim() != 2 or feat.shape[1] != 128 or hw <= 0 or nrays % hw != 0:
        raise RuntimeError(f"pixelnerf_decode: feat {tuple(feat.shape)} is not [n * {hw}, 128]")
    n = nrays // hw
    if rgb.numel() != n * 3 * hw or feats.numel() != n * 128 * hw:
        raise RuntimeError(f"pixelnerf_decode: rgb {tuple(rgb.shape)} / feats {tuple(feats.shape)} do not hold "
                           f"[{n}, 3, {hw}] / [{n}, 128, {hw}]")
    _mlp_shapes("pixelnerf_decode", mlp, 128)
    _lib.check(_lib.load().v3d_pixelnerf_decode(feat.data_ptr(), nrays, hw, w1.data_ptr(), b1.data_ptr(),
                                                w2.data_ptr(), b2.data_ptr(), w3.data_ptr(), b3.data_ptr(),
                                                rgb.data_ptr(), feats.data_ptr(), _stream()), "v3d_pixelnerf_decode")
    return rgb, feats
