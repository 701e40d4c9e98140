"""KernelModule: the base of the drop-in kernel modules (VideoUNet, the first-stage VideoDecoder / Encoder, the CLIP
image tower).  Reference-named fp32 parameters, bf16 kernel-side copies packed lazily on first forward, and the launch
helpers the networks' host schedules share: GroupNorm in its 2-D, 3-D and frame-sharded forms, the 3x3 / (3,1,1) convs,
the linears and the time_stack half of a video ResBlock."""
from __future__ import annotations

import contextlib
import math
import os
from typing import Optional, Tuple

import torch
import torch.nn as nn

from . import ops


def _register(root: nn.Module, dotted: str, value: torch.Tensor) -> None:
    parts = dotted.split(".")
    mod = root
    for part in parts[:-1]:
        child = mod._modules.get(part)
        if child is None:
            child = nn.Module()
            mod.add_module(part, child)
        mod = child
    mod.register_parameter(parts[-1], nn.Parameter(value, requires_grad=False))


def conv_tiles_ok(h: int, w: int) -> bool:
    """Mirror of the host-side geometry check of the implicit 3x3 conv (csrc/gemm_tc.cu)."""
    bw = min(w, 128)
    if 128 % bw or w % bw:
        return False
    bh = min(128 // bw, h)
    if h % bh or (128 // bw) % bh:
        return False
    return bw & (bw - 1) == 0 and bh & (bh - 1) == 0


def _invalidate_after_load(module, incompatible_keys) -> None:
    module._invalidate()


class KernelModule(nn.Module):
    """Shared machinery: reference-named fp32 parameters + lazily packed kernel-side weights."""

    def __init__(self):
        super().__init__()
        self._packed: Optional[dict] = None
        self.register_load_state_dict_post_hook(_invalidate_after_load)   # module-level function: picklable

    def _invalidate(self) -> None:
        """Drop the packed bf16 weights and the captured CUDA graphs.  Called automatically by load_state_dict and
        .to() / .cuda(); call it by hand after IN-PLACE edits of parameters (e.g. merging a LoRA with `p.data.add_`)."""
        self._packed = None
        if getattr(self, "_graphs", None):
            self._graphs.clear()  # captured graphs hold pointers into the old packed weights

    def _apply(self, fn, recurse=True):
        self._invalidate()
        return super()._apply(fn, recurse)

    def packed(self) -> dict:
        if self._packed is None:
            p = next(self.parameters())
            ops.require_current_device(p, f"v3d_b200.{type(self).__name__}.packed")
            with torch.no_grad():
                self._packed = self._pack(p.device)
        return self._packed

    def _pack(self, dev: torch.device) -> dict:  # pragma: no cover - abstract
        raise NotImplementedError

    @torch.no_grad()
    def init_random_(self, device, seed: int = 0) -> "KernelModule":
        """Materialise every parameter directly on `device` with non-degenerate random values (conv/linear
        weights N(0, 1/fan_in), biases N(0, 0.05^2), norm scales 1 + N(0, 0.1^2), mix factors N(0, 1)).
        For synthetic-weight benchmarking of a module built under `torch.device("meta")`: no 6 GB host copy."""
        gen = torch.Generator(device=device)
        gen.manual_seed(seed)
        for name, p in list(self.named_parameters()):
            shape = tuple(p.shape)
            if name.endswith("mix_factor"):
                val = torch.randn(shape, device=device, generator=gen)
            elif len(shape) > 1:
                val = torch.randn(shape, device=device, generator=gen) * (1.0 / math.sqrt(math.prod(shape[1:])))
            elif name.endswith(".weight"):
                val = 1.0 + 0.1 * torch.randn(shape, device=device, generator=gen)
            else:
                val = 0.05 * torch.randn(shape, device=device, generator=gen)
            parts = name.split(".")
            mod = self
            for part in parts[:-1]:
                mod = mod._modules[part]
            mod._parameters[parts[-1]] = nn.Parameter(val, requires_grad=False)
        self._invalidate()
        return self

    # ---- packing helpers -------------------------------------------------------------------
    @staticmethod
    def _bf(t: torch.Tensor) -> torch.Tensor:
        return t.detach().to(torch.bfloat16).contiguous()

    @staticmethod
    def _f32(t: torch.Tensor) -> torch.Tensor:
        return t.detach().float().contiguous()

    @classmethod
    def _pack_affine(cls, P: dict, sd: dict, key: str) -> None:
        """A norm's scale and shift, fp32."""
        P[key + ".weight"] = cls._f32(sd[key + ".weight"])
        P[key + ".bias"] = cls._f32(sd[key + ".bias"])

    @classmethod
    def _pack_1x1(cls, P: dict, sd: dict, key: str) -> None:
        """A 1x1 conv [Co, Ci, 1, 1] as the bf16 [Co, Ci] weight of a linear, fp32 bias."""
        w = sd[key + ".weight"]
        P[key + ".weight"] = cls._bf(w.reshape(w.shape[0], w.shape[1]))
        P[key + ".bias"] = cls._f32(sd[key + ".bias"])

    @classmethod
    def _pack_conv3x3(cls, w: torch.Tensor, b: Optional[torch.Tensor], kpad: int = 0):
        """[Co, Ci, 3, 3] -> bf16 [Co16, 9*Ci (padded to kpad)] in (ky, kx, ci) order; Co padded to 16."""
        co, ci = w.shape[:2]
        wp = w.detach().permute(0, 2, 3, 1).reshape(co, 9 * ci)
        k = max(kpad, 9 * ci)
        co16 = (co + 15) // 16 * 16
        out = torch.zeros(co16, k, device=w.device, dtype=torch.float32)
        out[:co, :9 * ci] = wp
        bias = torch.zeros(co16, device=w.device, dtype=torch.float32)
        if b is not None:
            bias[:co] = b.detach()
        return cls._bf(out), bias

    @classmethod
    def _pack_tconv(cls, w: torch.Tensor, b: torch.Tensor):
        """[Co, Ci, 3, 1, 1] -> bf16 [Co16, 3*Ci] in (tap, ci) order."""
        co, ci = w.shape[:2]
        wp = w.detach()[:, :, :, 0, 0].permute(0, 2, 1).reshape(co, 3 * ci)
        co16 = (co + 15) // 16 * 16
        out = torch.zeros(co16, 3 * ci, device=w.device, dtype=torch.float32)
        out[:co] = wp
        bias = torch.zeros(co16, device=w.device, dtype=torch.float32)
        bias[:co] = b.detach()
        return cls._bf(out), bias

    @classmethod
    def _pack_time_stack(cls, P: dict, sd: dict, ts: str) -> None:
        """The time_stack ResBlock `ts` of a video ResBlock: two norms and two (3,1,1) convs."""
        cls._pack_affine(P, sd, ts + ".in_layers.0")
        cls._pack_affine(P, sd, ts + ".out_layers.0")
        for cname in (".in_layers.2", ".out_layers.3"):
            P[ts + cname + ".weight"], P[ts + cname + ".bias"] = cls._pack_tconv(sd[ts + cname + ".weight"],
                                                                               sd[ts + cname + ".bias"])

    # ---- launch helpers ----------------------------------------------------------------------
    @staticmethod
    def _new(rows: int, c: int, dev, dtype=torch.bfloat16) -> torch.Tensor:
        return torch.empty(rows, c, device=dev, dtype=dtype)

    # frame-sharded execution (v3d_b200.viewshard.ViewShard) or None: set by the engine around a sharded call
    view_shard = None

    def _tap(self, name, x, B, c, h, w):
        """With `debug_taps` holding `name`: the block output x (bf16 NHWC) widened to fp32 NCHW, which is exactly
        the next block's input.  Launches nothing when taps are off."""
        if self.debug_taps is not None and name in self.debug_taps:
            tap = torch.empty(B, c, h, w, device=x.device, dtype=torch.float32)
            ops.nhwc_to_nchw_f32(x, tap, B, c, h * w, c)
            self.debug_taps[name] = tap

    @contextlib.contextmanager
    def _stats_pool(self, nsamples: int, dev):
        """Statistics slices for `_take_stats` of up to `nsamples` GroupNorm samples, out of one pool zeroed once per
        forward (one memset instead of one per norm); dropped on exit, also after a failed run (OOM mid-schedule)."""
        object.__setattr__(self, "_gn_pool", [torch.zeros(nsamples * 64, device=dev, dtype=torch.float64), 0])
        try:
            yield
        finally:
            object.__setattr__(self, "_gn_pool", None)

    def _take_stats(self, nsamples: int, dev) -> Tuple[torch.Tensor, bool]:
        pool = getattr(self, "_gn_pool", None)
        need = nsamples * 64
        if pool is not None and pool[1] + need <= pool[0].numel():
            stats = pool[0][pool[1]:pool[1] + need].view(nsamples, 32, 2)
            pool[1] += need
            return stats, True
        return torch.empty(nsamples, 32, 2, device=dev, dtype=torch.float64), False

    def _gn_workspace(self, dev) -> torch.Tensor:
        """Barrier state + partials of the single-launch GroupNorm: one zeroed buffer per module and device (every
        launch of this module is issued on one stream; captured CUDA graphs hold its address)."""
        ws = getattr(self, "_gn_ws", None)
        if ws is None or ws.device != dev:
            ws = ops.groupnorm_workspace(dev)
            object.__setattr__(self, "_gn_ws", ws)
        return ws

    def _gn_det_workspace(self, dev, nbytes: int) -> torch.Tensor:
        """Workspace of the single-launch deterministic GroupNorm, sized by shape: one zeroed buffer per power-of-two
        size class and device.  None is ever freed while the module lives (a captured CUDA graph holds its address)."""
        pool = getattr(self, "_gn_det_ws", None)
        if pool is None:
            pool = {}
            object.__setattr__(self, "_gn_det_ws", pool)
        size = 1 << max(int(nbytes) - 1, 1).bit_length()
        ws = pool.get((dev, size))
        if ws is None:
            ws = pool[(dev, size)] = ops.groupnorm_det_workspace(dev, size)
        return ws

    def _gn(self, P: dict, key: str, x: torch.Tensor, rows_per_sample: int, nsamples: int, c: int, eps: float,
            silu: bool, hw: Optional[int] = None) -> torch.Tensor:
        """act(GroupNorm32(x)) over nsamples x rows_per_sample rows; hw = rows per frame (3-D norms: rows_per_sample =
        T * hw), which defines the blocks of the deterministic statistics."""
        y = torch.empty(x.shape[0], c, device=x.device, dtype=torch.bfloat16)
        # one launch (statistics -> grid barrier -> apply) for the per-frame (2-D) norms: on one H100 it measured faster
        # than the statistics + apply pair at every such UNet shape (tools/microbench.py norm: 0.116 vs 0.139 ms at
        # [36*4096, 320], 0.324 vs 0.325 at 960 channels, 0.063 vs 0.091 at level 1, 0.035 vs 0.042 at level 2) and up to
        # 604 MB tensors (0.641 vs 0.669 ms); the UNet's largest is 283 MB, so the 300 MB bound excludes none of them.
        # At 1.2 GB the two tie.  The 3-D time_stack norms (2 samples) stay on the pair
        fused = 8 <= nsamples <= 256 and x.numel() * 2 <= 300e6
        if ops.deterministic():
            # the same selection between one launch and the pair, on the deterministic kernels (same bits either way)
            hw = rows_per_sample if hw is None else hw
            if fused and os.environ.get("V3D_GN_FUSED", "1") != "0":
                ws = self._gn_det_workspace(x.device, ops.groupnorm_det_workspace_bytes(rows_per_sample, hw, nsamples))
                return ops.groupnorm_det(x, y, P[key + ".weight"], P[key + ".bias"], rows_per_sample, hw, nsamples, c,
                                         eps, silu, ws)
            nblk = ops.groupnorm_det_blocks(rows_per_sample, hw)
            part = torch.empty(nsamples, nblk, 32, 2, device=x.device, dtype=torch.float32)
            ops.groupnorm_partials(x, part, rows_per_sample, hw, nsamples, c)
            return ops.groupnorm_fold_apply(x, y, part, P[key + ".weight"], P[key + ".bias"], rows_per_sample,
                                            nsamples, c, eps, silu, nblk)
        if fused and os.environ.get("V3D_GN_FUSED", "1") != "0":
            return ops.groupnorm(x, y, P[key + ".weight"], P[key + ".bias"], rows_per_sample, nsamples, c, eps, silu,
                                 self._gn_workspace(x.device))
        stats, pre_zeroed = self._take_stats(nsamples, x.device)
        ops.groupnorm_stats(x, stats, rows_per_sample, nsamples, c, pre_zeroed=pre_zeroed)
        ops.groupnorm_apply(x, y, stats, P[key + ".weight"], P[key + ".bias"], rows_per_sample, nsamples, c, eps,
                            silu)
        return y

    def _gn_halo(self, P: dict, key: str, x: torch.Tensor, hw: int, tl: int, nb: int, c: int, eps: float,
                 silu: bool) -> torch.Tensor:
        """3-D GroupNorm (+SiLU) of a frame-sharded video: local (sum, sumsq) -> all-reduce -> apply, written into
        the interior of a [nb, tl + 2, hw, c] buffer whose first / last frame then receive the neighbours' boundary
        frames (zeros at the ends of the video): the operand of the following (3,1,1) convolution."""
        vs = self.view_shard
        if ops.deterministic():
            # block partials of this rank's frames at their global block offset, all-gathered, folded over the whole
            # video in block order on every rank: the unsharded deterministic statistics, bit for bit
            nbf = ops.groupnorm_det_blocks(hw, hw)
            part = vs.gn_partials(nb, vs.num_frames * nbf, x.device)
            ops.groupnorm_partials(x, part[:, vs.t0 * nbf:], tl * hw, hw, nb, c, ldp=vs.num_frames * nbf)
            vs.allgather_partials_(part, nbf)
            pad = vs.new_pad((nb, tl + 2, hw, c), torch.bfloat16, x.device)
            for b in range(nb):
                ops.groupnorm_fold_apply(x[b * tl * hw:(b + 1) * tl * hw], pad[b, 1:tl + 1], part[b:b + 1],
                                         P[key + ".weight"], P[key + ".bias"], tl * hw, 1, c, eps, silu,
                                         vs.num_frames * nbf, count_rows=vs.num_frames * hw)
            vs.exchange_halos(pad)
            return pad
        stats, pre_zeroed = self._take_stats(nb, x.device)
        ops.groupnorm_stats(x, stats, tl * hw, nb, c, pre_zeroed=pre_zeroed)
        vs.allreduce_stats_(stats)
        pad = vs.new_pad((nb, tl + 2, hw, c), torch.bfloat16, x.device)
        for b in range(nb):
            ops.groupnorm_apply(x[b * tl * hw:(b + 1) * tl * hw], pad[b, 1:tl + 1], stats[b:b + 1],
                                P[key + ".weight"], P[key + ".bias"], tl * hw, 1, c, eps, silu)
        vs.exchange_halos(pad)
        return pad

    def _gn3d(self, P: dict, key: str, x: torch.Tensor, hw: int, T: int, nb: int, c: int) -> torch.Tensor:
        """SiLU(GroupNorm32(x)), eps 1e-5, over (C/32, T, H, W) of each of nb videos: the operand of a following
        `_tconv`, dense or (frame-sharded, T = this rank's frames) the halo'd buffer of `_gn_halo`."""
        if self.view_shard is not None:
            return self._gn_halo(P, key, x, hw, T, nb, c, 1e-5, True)
        return self._gn(P, key, x, T * hw, nb, c, 1e-5, True, hw=hw)

    def _tconv(self, P: dict, key: str, a: torch.Tensor, out: torch.Tensor, hw: int, T: int, nb: int, c: int,
               **epi) -> torch.Tensor:
        """Conv3d k=(3,1,1) pad (1,0,0) on the frame-major layout as a 3-tap GEMM.  `a` is either the dense
        [nb*T*hw, c] activation (zero padding at both ends of every video) or, frame-sharded, the halo'd
        [nb, T + 2, hw, c] buffer of `_gn_halo`."""
        halo = a.dim() == 4
        frames = T + 2 if halo else T
        ops.gemm(a.view(-1, c) if halo else a, P[key + ".weight"], out, K=c, N=c, rows_per_batch=T * hw, batch=nb,
                 a_batch_stride=frames * hw * c, bias=P[key + ".bias"], ntaps=3, tap_shift=hw,
                 a_rows=frames * hw if halo else 0, a_row0=hw if halo else 0, **epi)
        return out

    def _time_stack(self, P: dict, ts: str, xs: torch.Tensor, hw: int, T: int, nb: int, c: int, *, s0: float,
                    **first_conv_epilogue) -> torch.Tensor:
        """xs + s0 * time_stack(xs): the time_stack ResBlock of a video ResBlock (3-D GroupNorm + SiLU, (3,1,1) conv,
        3-D GroupNorm + SiLU, (3,1,1) conv) with the AlphaBlender folded into the last conv's epilogue.  Frame-sharded,
        T is this rank's block: the norms all-reduce their statistics and the convs read halos."""
        a = self._gn3d(P, ts + ".in_layers.0", xs, hw, T, nb, c)
        h = torch.empty(xs.shape[0], c, device=xs.device, dtype=torch.bfloat16)
        self._tconv(P, ts + ".in_layers.2", a, h, hw, T, nb, c, **first_conv_epilogue)
        a = self._gn3d(P, ts + ".out_layers.0", h, hw, T, nb, c)
        return self._tconv(P, ts + ".out_layers.3", a, h, hw, T, nb, c, r1=xs, s1=1.0, s0=s0)

    def _conv3x3(self, P: dict, key: str, x: torch.Tensor, n: int, h: int, w: int, cin: int, *, stride: int = 1,
                 out: Optional[torch.Tensor] = None, out_dtype=torch.bfloat16, **epi) -> torch.Tensor:
        """3x3 conv, pad 1. Implicit-GEMM (TMA gather) when Cin % 64 == 0, stride 1 and the image tiles into
        128-pixel boxes; otherwise explicit im2row + the same tensor-core GEMM."""
        wt, bias = P[key + ".weight"], P[key + ".bias"]
        cop = wt.shape[0]
        ho, wo = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
        rows = n * ho * wo
        if out is None:
            out = torch.empty(rows, cop, device=x.device, dtype=out_dtype)
        if stride == 1 and cin % 64 == 0 and conv_tiles_ok(h, w):
            ops.gemm(x, wt, out, K=cin, N=cop, rows_per_batch=rows, bias=bias, conv=(n, h, w), **epi)
        else:
            kpad = wt.shape[1]
            col = torch.empty(rows, kpad, device=x.device, dtype=torch.bfloat16)
            ops.im2col3x3(x, col, n, h, w, cin, stride, 1, ho, wo, kpad)
            ops.gemm(col, wt, out, K=kpad, N=cop, rows_per_batch=rows, bias=bias, **epi)
        return out

    def _linear(self, P: dict, key: str, x: torch.Tensor, rows: int, *, out: Optional[torch.Tensor] = None,
                act: int = ops.ACT_NONE, **epi) -> torch.Tensor:
        wt = P[key + ".weight"]
        n, k = wt.shape
        n_out = n // 2 if act == ops.ACT_GEGLU else n
        if out is None:
            out = torch.empty(rows, n_out, device=x.device, dtype=torch.bfloat16)
        ops.gemm(x, wt, out, K=k, N=n, rows_per_batch=rows, bias=P.get(key + ".bias"), act=act, **epi)
        return out
