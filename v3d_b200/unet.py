"""H100-native drop-in for sgm.modules.diffusionmodules.video_model.VideoUNet (reference
sgm/modules/diffusionmodules/video_model.py:84-493).

Same constructor kwargs, same `state_dict()` keys/shapes (SURVEY.md App. D), same forward signature; the
forward is a host-side schedule of C-ABI kernel launches (v3d_b200.ops) over bf16 NHWC / token-major
activations.  Parameters stay fp32 `nn.Parameter`s under the reference names (so `init_from_ckpt`'s
`load_state_dict(strict=False)`, video_diffusion.py:123-168, works unchanged); kernel-side bf16 copies are
packed lazily on first forward and re-packed after `load_state_dict` / `.to()`.

Layout: the `(b t)` frame-major batch of the reference is kept; every activation is a [B*H*W, C] matrix
with channels contiguous, so a conv output IS the token matrix of the following transformer and the
temporal `(b t) s c <-> (b s) t c` rearranges (video_attention.py:114,137) never materialise.
There is no CPU path: forward on non-CUDA tensors raises.
"""
from __future__ import annotations

import math
import os
from dataclasses import dataclass
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn

from . import ops
from .kernel_module import KernelModule, _register, conv_tiles_ok  # noqa: F401  (conv_tiles_ok: still public here)

_EMB_MULT = 4


@dataclass
class _Step:
    kind: str            # conv_in | res | attn | down | up | save | cat | out
    name: str = ""
    cin: int = 0
    cout: int = 0


class VideoUNet(KernelModule):
    """Drop-in `target:` for `sgm.modules.diffusionmodules.video_model.VideoUNet`."""

    def __init__(
        self,
        in_channels: int,
        model_channels: int,
        out_channels: int,
        num_res_blocks: int,
        attention_resolutions: Sequence[int],
        dropout: float = 0.0,
        channel_mult: Sequence[int] = (1, 2, 4, 8),
        conv_resample: bool = True,
        dims: int = 2,
        num_classes: Optional[Union[int, str]] = None,
        use_checkpoint: bool = False,
        num_heads: int = -1,
        num_head_channels: int = -1,
        num_heads_upsample: int = -1,
        use_scale_shift_norm: bool = False,
        resblock_updown: bool = False,
        transformer_depth: Union[List[int], int] = 1,
        transformer_depth_middle: Optional[int] = None,
        context_dim: Optional[int] = None,
        time_downup: bool = False,
        time_context_dim: Optional[int] = None,
        extra_ff_mix_layer: bool = False,
        use_spatial_context: bool = False,
        merge_strategy: str = "fixed",
        merge_factor: float = 0.5,
        spatial_transformer_attn_type: str = "softmax",
        video_kernel_size: Union[int, List[int]] = 3,
        use_linear_in_transformer: bool = False,
        adm_in_channels: Optional[int] = None,
        disable_temporal_crossattention: bool = False,
        max_ddpm_temb_period: int = 10000,
    ):
        super().__init__()
        assert context_dim is not None
        depth = transformer_depth if isinstance(transformer_depth, int) else None
        if depth is None:
            depth = transformer_depth[0]
            assert all(d == depth for d in transformer_depth), "per-level transformer depth is not supported"
        unsupported = {
            "dims != 2": dims != 2,
            "num_classes != 'sequential'": num_classes != "sequential",
            "num_head_channels != 64": num_head_channels != 64,
            "use_scale_shift_norm": use_scale_shift_norm,
            "resblock_updown": resblock_updown,
            "conv_resample=False": not conv_resample,
            "transformer_depth != 1": depth != 1 or (transformer_depth_middle not in (None, 1)),
            "time_downup": time_downup,
            "extra_ff_mix_layer=False": not extra_ff_mix_layer,
            "use_spatial_context=False": not use_spatial_context,
            "use_linear_in_transformer=False": not use_linear_in_transformer,
            "disable_temporal_crossattention": disable_temporal_crossattention,
            "video_kernel_size != [3,1,1]": list(video_kernel_size) != [3, 1, 1]
            if not isinstance(video_kernel_size, int) else True,
            "dropout != 0": dropout != 0.0,
            "model_channels % 64": model_channels % 64 != 0,
        }
        bad = [k for k, v in unsupported.items() if v]
        if bad:
            raise NotImplementedError(
                "v3d_b200.VideoUNet covers the V3D_512 / SVD configuration family only; unsupported: " + ", ".join(bad))
        assert adm_in_channels is not None and adm_in_channels % 8 == 0
        assert merge_strategy in ("fixed", "learned", "learned_with_images")
        # xformers vs softmax attention modes are numerically the same op (SURVEY.md §0.8); one kernel serves both
        assert spatial_transformer_attn_type in ("softmax", "softmax-xformers")

        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = list(attention_resolutions)
        self.channel_mult = list(channel_mult)
        self.num_classes = num_classes
        self.num_head_channels = num_head_channels
        self.context_dim = context_dim
        self.adm_in_channels = adm_in_channels
        self.merge_strategy = merge_strategy
        self.merge_factor = merge_factor
        self.max_ddpm_temb_period = max_ddpm_temb_period
        self.use_checkpoint = use_checkpoint  # accepted for config compatibility; inference only
        self.time_embed_dim = model_channels * _EMB_MULT

        self.steps = self._plan()
        self._init_parameters()
        self._indicator_seen: Optional[tuple] = None
        self.debug_taps: Optional[dict] = None  # tests: {block name: None} -> filled with NCHW fp32 outputs
        # The forward is a fixed schedule of ~1.1k launches: after one eager call per input shape it is captured
        # into a CUDA graph and replayed (no tracing compiler involved; V3D_CUDA_GRAPH=0 disables).
        self.cuda_graphs: bool = os.environ.get("V3D_CUDA_GRAPH", "1") != "0"
        self._graphs: dict = {}
        self.replayed_launches: int = 0  # kernels executed through graph replays (for launch accounting)

    # ------------------------------------------------------------------------------------------
    # architecture plan (execution order) and parameter table
    # ------------------------------------------------------------------------------------------
    def _plan(self) -> List[_Step]:
        mc = self.model_channels
        steps: List[_Step] = [_Step("conv_in", "input_blocks.0.0", self.in_channels, mc), _Step("save")]
        widths = [mc]
        ch, ds, idx = mc, 1, 1
        last = len(self.channel_mult) - 1
        for level, mult in enumerate(self.channel_mult):
            for _ in range(self.num_res_blocks):
                steps.append(_Step("res", f"input_blocks.{idx}.0", ch, mult * mc))
                ch = mult * mc
                if ds in self.attention_resolutions:
                    steps.append(_Step("attn", f"input_blocks.{idx}.1", ch, ch))
                steps.append(_Step("save"))
                widths.append(ch)
                idx += 1
            if level != last:
                steps += [_Step("down", f"input_blocks.{idx}.0", ch, ch), _Step("save")]
                widths.append(ch)
                ds *= 2
                idx += 1
        steps += [_Step("res", "middle_block.0", ch, ch), _Step("attn", "middle_block.1", ch, ch),
                  _Step("res", "middle_block.2", ch, ch)]
        idx = 0
        for level in range(last, -1, -1):
            mult = self.channel_mult[level]
            for i in range(self.num_res_blocks + 1):
                skip = widths.pop()
                steps.append(_Step("cat", "", ch, ch + skip))
                steps.append(_Step("res", f"output_blocks.{idx}.0", ch + skip, mult * mc))
                ch = mult * mc
                sub = 1
                if ds in self.attention_resolutions:
                    steps.append(_Step("attn", f"output_blocks.{idx}.1", ch, ch))
                    sub = 2
                if level > 0 and i == self.num_res_blocks:
                    steps.append(_Step("up", f"output_blocks.{idx}.{sub}", ch, ch))
                    ds //= 2
                idx += 1
        steps.append(_Step("out", "out", mc, self.out_channels))
        return steps

    def param_shapes(self) -> Dict[str, Tuple[int, ...]]:
        te, ctx = self.time_embed_dim, self.context_dim
        table: Dict[str, Tuple[int, ...]] = {}

        def dense(key, n, k, bias=True):
            table[key + ".weight"] = (n, k)
            if bias:
                table[key + ".bias"] = (n,)

        def conv(key, co, ci, *ks):
            table[key + ".weight"] = (co, ci, *ks)
            table[key + ".bias"] = (co,)

        def affine(key, c):
            table[key + ".weight"] = (c,)
            table[key + ".bias"] = (c,)

        def res_core(key, ci, co, ks):
            affine(key + ".in_layers.0", ci)
            conv(key + ".in_layers.2", co, ci, *ks)
            dense(key + ".emb_layers.1", co, te)
            affine(key + ".out_layers.0", co)
            conv(key + ".out_layers.3", co, co, *ks)
            if ci != co:
                conv(key + ".skip_connection", co, ci, *([1] * len(ks)))

        def attention(key, c, kdim):
            dense(key + ".to_q", c, c, bias=False)
            dense(key + ".to_k", c, kdim, bias=False)
            dense(key + ".to_v", c, kdim, bias=False)
            dense(key + ".to_out.0", c, c)

        def geglu_ff(key, c):
            dense(key + ".net.0.proj", 8 * c, c)
            dense(key + ".net.2", c, 4 * c)

        dense("time_embed.0", te, self.model_channels)
        dense("time_embed.2", te, te)
        dense("label_emb.0.0", te, self.adm_in_channels)
        dense("label_emb.0.2", te, te)
        for st in self.steps:
            if st.kind == "conv_in":
                conv(st.name, st.cout, st.cin, 3, 3)
            elif st.kind == "res":
                res_core(st.name, st.cin, st.cout, (3, 3))
                res_core(st.name + ".time_stack", st.cout, st.cout, (3, 1, 1))
                table[st.name + ".time_mixer.mix_factor"] = (1,)
            elif st.kind == "attn":
                c = st.cin
                affine(st.name + ".norm", c)
                dense(st.name + ".proj_in", c, c)
                for blk, norms in ((".transformer_blocks.0", ("norm1", "norm2", "norm3")),
                                   (".time_stack.0", ("norm_in", "norm1", "norm2", "norm3"))):
                    base = st.name + blk
                    if "time_stack" in blk:
                        geglu_ff(base + ".ff_in", c)
                    attention(base + ".attn1", c, c)
                    attention(base + ".attn2", c, ctx)
                    geglu_ff(base + ".ff", c)
                    for nm in norms:
                        affine(f"{base}.{nm}", c)
                dense(st.name + ".time_pos_embed.0", 4 * c, c)
                dense(st.name + ".time_pos_embed.2", c, 4 * c)
                table[st.name + ".time_mixer.mix_factor"] = (1,)
                dense(st.name + ".proj_out", c, c)
            elif st.kind == "down":
                conv(st.name + ".op", st.cout, st.cin, 3, 3)
            elif st.kind == "up":
                conv(st.name + ".conv", st.cout, st.cin, 3, 3)
            elif st.kind == "out":
                affine("out.0", st.cin)
                conv("out.2", st.cout, st.cin, 3, 3)
        return table

    ZERO_INIT_SUFFIXES = (".out_layers.3.weight", ".out_layers.3.bias", ".proj_out.weight", ".proj_out.bias",
                          "out.2.weight", "out.2.bias")

    def _init_parameters(self) -> None:
        """Reference-like initialisation: uniform(-1/sqrt(fan_in), 1/sqrt(fan_in)) conv/linear weights and biases,
        unit norms, zero-initialised residual outputs (zero_module: openaimodel.py:306-314, attention.py:699-704,
        video_model.py:439) and mix_factor = merge_factor."""
        gen = torch.Generator(device="cpu")
        gen.manual_seed(torch.initial_seed() & 0x7FFFFFFF)
        on_meta = torch.empty(0).device.type == "meta"  # `with torch.device("meta")`: shapes only, no values
        for key, shape in self.param_shapes().items():
            if on_meta:
                val = torch.empty(shape)
            elif key.endswith("mix_factor"):
                val = torch.full(shape, float(self.merge_factor))
            elif key.endswith(self.ZERO_INIT_SUFFIXES):
                val = torch.zeros(shape)
            elif len(shape) == 1 and key.endswith(".weight"):
                val = torch.ones(shape)
            elif len(shape) == 1 and self._is_norm_bias(key):
                val = torch.zeros(shape)
            else:
                fan_in = math.prod(shape[1:]) if len(shape) > 1 else self._bias_fan_in(key)
                bound = 1.0 / math.sqrt(max(fan_in, 1))
                val = (torch.rand(shape, generator=gen) * 2.0 - 1.0) * bound
            _register(self, key, val)

    def _is_norm_bias(self, key: str) -> bool:
        w = key[:-len(".bias")] + ".weight"
        shapes = self._shape_cache()
        return w in shapes and len(shapes[w]) == 1

    def _bias_fan_in(self, key: str) -> int:
        w = self._shape_cache().get(key[:-len(".bias")] + ".weight")
        return math.prod(w[1:]) if w else 1

    def _shape_cache(self):
        if not hasattr(self, "_shapes"):
            object.__setattr__(self, "_shapes", self.param_shapes())
        return self._shapes

    @torch.no_grad()
    def randomize_zero_modules_(self, seed: int = 1) -> "VideoUNet":
        """Give the zero-initialised residual outputs N(0, 1/fan_in) values so a random-weight network is not
        degenerate (SURVEY.md §0.6). Used by bench.py / smoke(); never called on loaded checkpoints."""
        gen = torch.Generator(device="cpu")
        gen.manual_seed(seed)
        for key, p in self.named_parameters():
            if key.endswith(self.ZERO_INIT_SUFFIXES):
                if p.ndim > 1:
                    fan_in = math.prod(p.shape[1:])
                    p.copy_((torch.randn(p.shape, generator=gen) / math.sqrt(fan_in)).to(p.device))
                else:
                    p.copy_((0.05 * torch.randn(p.shape, generator=gen)).to(p.device))
        self._invalidate()
        return self

    # ------------------------------------------------------------------------------------------
    # weight packing
    # ------------------------------------------------------------------------------------------
    def _alpha(self, raw: float) -> float:
        """AlphaBlender.get_alpha with image_only_indicator == 0 (util.py:341-356)."""
        return raw if self.merge_strategy == "fixed" else 1.0 / (1.0 + math.exp(-raw))

    def _pack(self, dev: torch.device) -> dict:
        sd = {k: v.detach() for k, v in self.named_parameters()}
        P: dict = {}

        def dense(key, bias=True):
            P[key + ".weight"] = self._bf(sd[key + ".weight"])
            if bias and key + ".bias" in sd:
                P[key + ".bias"] = self._f32(sd[key + ".bias"])

        def geglu(key):
            w, b = sd[key + ".weight"], sd[key + ".bias"]
            n_out = w.shape[0] // 2
            bn = ops.pick_block_n(w.shape[0], ops.ACT_GEGLU)
            perm = ops.geglu_perm(n_out, bn).to(dev)
            P[key + ".weight"] = self._bf(w[perm])
            P[key + ".bias"] = self._f32(b[perm])

        def attn_self(key):
            P[key + ".qkv.weight"] = self._bf(
                torch.cat([sd[key + ".to_q.weight"], sd[key + ".to_k.weight"], sd[key + ".to_v.weight"]], 0))
            dense(key + ".to_out.0")

        for k in ("time_embed.0", "time_embed.2", "label_emb.0.0", "label_emb.0.2"):
            dense(k)

        mix_keys = [k for k in sd if k.endswith("mix_factor")]
        mix_vals = torch.stack([sd[k].reshape(()) for k in mix_keys]).float().cpu().tolist()
        alpha = {k: self._alpha(v) for k, v in zip(mix_keys, mix_vals)}

        emb_w, emb_b, emb_off = [], [], {}
        cv_w, cv_off, cv_total = [], {}, 0
        off = 0
        for st in self.steps:
            nm = st.name
            if st.kind == "conv_in":
                kpad = (9 * st.cin + 63) // 64 * 64
                P[nm + ".weight"], P[nm + ".bias"] = self._pack_conv3x3(sd[nm + ".weight"], sd[nm + ".bias"], kpad)
            elif st.kind == "res":
                self._pack_affine(P, sd, nm + ".in_layers.0")
                self._pack_affine(P, sd, nm + ".out_layers.0")
                for cname in (".in_layers.2", ".out_layers.3"):
                    P[nm + cname + ".weight"], P[nm + cname + ".bias"] = self._pack_conv3x3(
                        sd[nm + cname + ".weight"], sd[nm + cname + ".bias"])
                self._pack_time_stack(P, sd, nm + ".time_stack")
                for base in (nm, nm + ".time_stack"):
                    emb_w.append(sd[base + ".emb_layers.1.weight"])
                    emb_b.append(sd[base + ".emb_layers.1.bias"])
                    emb_off[base] = (off, st.cout)
                    off += st.cout
                if st.cin != st.cout:
                    self._pack_1x1(P, sd, nm + ".skip_connection")
                P[nm + ".alpha"] = alpha[nm + ".time_mixer.mix_factor"]
            elif st.kind == "attn":
                c = st.cin
                self._pack_affine(P, sd, nm + ".norm")
                dense(nm + ".proj_in")
                dense(nm + ".proj_out")
                dense(nm + ".time_pos_embed.0")
                dense(nm + ".time_pos_embed.2")
                for base, norms in ((nm + ".transformer_blocks.0", ("norm1", "norm3")),
                                    (nm + ".time_stack.0", ("norm_in", "norm1", "norm3"))):
                    attn_self(base + ".attn1")
                    geglu(base + ".ff.net.0.proj")
                    dense(base + ".ff.net.2")
                    for n_ in norms:
                        self._pack_affine(P, sd, f"{base}.{n_}")
                    # single-token cross-attention collapses to to_out(to_v(ctx)) (SURVEY.md §0.4); norm2 / to_q /
                    # to_k of attn2 cannot influence it and are packed only for a multi-token context (_pack_cross)
                    cv_w.append(sd[base + ".attn2.to_v.weight"])
                    cv_off[base] = (cv_total, c)
                    cv_total += c
                    dense(base + ".attn2.to_out.0")
                geglu(nm + ".time_stack.0.ff_in.net.0.proj")
                dense(nm + ".time_stack.0.ff_in.net.2")
                P[nm + ".alpha"] = alpha[nm + ".time_mixer.mix_factor"]
            elif st.kind == "down":
                P[nm + ".op.weight"], P[nm + ".op.bias"] = self._pack_conv3x3(sd[nm + ".op.weight"], sd[nm + ".op.bias"])
            elif st.kind == "up":
                P[nm + ".conv.weight"], P[nm + ".conv.bias"] = self._pack_conv3x3(sd[nm + ".conv.weight"],
                                                                               sd[nm + ".conv.bias"])
            elif st.kind == "out":
                self._pack_affine(P, sd, "out.0")
                P["out.2.weight"], P["out.2.bias"] = self._pack_conv3x3(sd["out.2.weight"], sd["out.2.bias"])
        P["emb_all.weight"] = self._bf(torch.cat(emb_w, 0))
        P["emb_all.bias"] = self._f32(torch.cat(emb_b, 0))
        P["emb_off"], P["emb_total"] = emb_off, off
        P["cv_all.weight"] = self._bf(torch.cat(cv_w, 0))
        P["cv_off"], P["cv_total"] = cv_off, cv_total
        P["pos_cache"] = {}
        return P

    def _pack_cross(self, P: dict) -> None:
        """The attn2 weights only a context of more than one token reads - norm2, to_q, and to_k | to_v of every layer
        stacked into one [sum 2C, context_dim] matrix (layer `base` at rows P["ckv_off"][base][0]: its C K rows, then
        its C V rows) - added to P on the first such forward, so the single-token path never allocates them."""
        if "ckv_all.weight" in P:
            return
        sd = {k: v.detach() for k, v in self.named_parameters()}
        kv_w, kv_off, total = [], {}, 0
        for base, (_, c) in P["cv_off"].items():
            kv_w += [sd[base + ".attn2.to_k.weight"], sd[base + ".attn2.to_v.weight"]]
            kv_off[base] = (total, c)
            total += 2 * c
            P[base + ".attn2.to_q.weight"] = self._bf(sd[base + ".attn2.to_q.weight"])
            P[base + ".norm2.weight"] = self._f32(sd[base + ".norm2.weight"])
            P[base + ".norm2.bias"] = self._f32(sd[base + ".norm2.bias"])
        P["ckv_off"] = kv_off
        P["ckv_all.weight"] = self._bf(torch.cat(kv_w, 0))

    # ------------------------------------------------------------------------------------------
    # forward
    # ------------------------------------------------------------------------------------------
    def _check_indicator(self, ind: Optional[torch.Tensor], b: int, T: int) -> None:
        """merge_strategy 'learned_with_images' needs image_only_indicator (util.py:352-356); the kernels
        implement the all-video case (indicator == 0), which is what every V3D entry point passes
        (scripts/pub/V3D_512.py:273-275).  Checked once per distinct tensor (one host sync), not per step."""
        if self.merge_strategy != "learned_with_images":
            return
        assert ind is not None, "need image_only_indicator ..."
        tag = (ind.data_ptr(), ind._version, tuple(ind.shape))
        if tag == self._indicator_seen:
            return
        assert tuple(ind.shape) == (b, T), f"image_only_indicator must be [{b},{T}], got {tuple(ind.shape)}"
        if bool(ind.bool().any()):
            raise NotImplementedError("image_only_indicator != 0 (image frames mixed into a video batch) is not "
                                      "implemented in the native kernels")
        self._indicator_seen = tag

    def forward(
        self,
        x: torch.Tensor,
        timesteps: torch.Tensor,
        context: Optional[torch.Tensor] = None,
        y: Optional[torch.Tensor] = None,
        time_context: Optional[torch.Tensor] = None,
        num_video_frames: Optional[int] = None,
        image_only_indicator: Optional[torch.Tensor] = None,
    ) -> torch.Tensor:
        ops.require_current_device(x, "v3d_b200.VideoUNet.forward")
        args, dims, graphs = self._prepare(x, timesteps, context, y, time_context, num_video_frames,
                                           image_only_indicator)
        P = self.packed()
        with torch.no_grad():
            if graphs and self.debug_taps is None and not torch.cuda.is_current_stream_capturing():
                return self._run_graphed(P, args, *dims, x.device)
            return self._run(P, *args, *dims, x.device)

    def _prepare(self, x, timesteps, context, y, time_context, num_video_frames, image_only_indicator):
        """Argument checks of VideoUNet.forward (video_model.py:452-461) and assembly of the schedule's inputs:
        -> ((x, timesteps, context rows, y) fp32 contiguous, (B, T, nb, H, W), use CUDA graphs).  The context rows are
        [B (+ nb time-context rows when frame-sharded), M * context_dim]: one row per sample holding its M tokens."""
        assert (y is not None) == (self.num_classes is not None), \
            "must specify y if and only if the model is class-conditional"
        assert y is None or y.shape[0] == x.shape[0]
        assert context is not None and context.ndim == 3, \
            f"n dims of spatial context should be 3 but are {None if context is None else context.ndim}"
        assert num_video_frames, "num_video_frames is required"
        M = context.shape[1]
        assert M >= 1 and context.shape[2] == self.context_dim, \
            f"context must be [B, tokens >= 1, {self.context_dim}], got {tuple(context.shape)}"
        B, cin, H, W = x.shape
        T = int(num_video_frames)
        assert B % T == 0 and cin == self.in_channels
        down = 2 ** (len(self.channel_mult) - 1)
        if H % down or W % down:
            # the reference fails at th.cat([h, hs.pop()]) (video_model.py:483) when a stride-2 level rounds an odd size
            raise RuntimeError(f"latent size {H}x{W} must be divisible by {down}: the skip connections of the "
                               f"{len(self.channel_mult)}-level U-Net would not line up")
        nb = B // T
        vs = self.view_shard
        ops.check_temporal_frames(T if vs is None else vs.num_frames)   # keys = the whole video, also when sharded
        self._check_indicator(image_only_indicator, nb, T)
        dev = x.device
        ctx2d = context.float().reshape(B, -1)
        graphs = self.cuda_graphs and x.is_cuda          # capture needs CUDA inputs (tests run forward on CPU)
        if vs is not None:
            # frame-sharded call: x / context / y hold this rank's T = vs.tl frames of each video; the temporal
            # cross-attention context (frame 0 of each video, video_attention.py:250) may live on another rank and
            # arrives through `time_context` [nb, M, ctx]; its rows are appended to the context matrix
            assert T == vs.tl, f"view-sharded forward expects this rank's {vs.tl} frames, got num_video_frames={T}"
            assert time_context is not None and time_context.ndim == 3 and time_context.shape[:2] == (nb, M), \
                f"view-sharded forward needs time_context = context of frame 0 of each video, [nb, {M}, ctx]"
            ctx2d = torch.cat([ctx2d, time_context.float().reshape(nb, -1).to(dev)], dim=0)
            # the one-sided peer transport is stream-ordered kernels only: always capturable.  torch.distributed
            # collectives inside a captured graph stay opt-in (V3D_VIEWSHARD_GRAPH=1)
            graphs = graphs and (vs.peer is not None or
                                 (os.environ.get("V3D_VIEWSHARD_GRAPH", "0") == "1" and not vs._via_host(x)))
        args = (x.float().contiguous(), timesteps.float().contiguous(), ctx2d.contiguous(), y.float().contiguous())
        return args, (B, T, nb, H, W), graphs

    def _graph_key(self, B, T, H, W, dev, M: int = 1) -> tuple:
        """Cache key of a captured graph: the shape, the context's token count M (a multi-token context runs another
        schedule), the device, the shard and the deterministic mode (the two modes launch different GroupNorm kernels,
        so a graph captured in one is never replayed in the other)."""
        vs = self.view_shard
        key = (B, T, H, W, dev.index) if vs is None else (B, T, H, W, dev.index, vs.num_frames, vs.rank, vs.world)
        return key + (("deterministic",) if ops.deterministic() else ()) + ((("tokens", M),) if M != 1 else ())

    def _run_graphed(self, P, args, B, T, nb, H, W, dev):
        key = self._graph_key(B, T, H, W, dev, args[2].shape[1] // self.context_dim)
        entry = self._graphs.get(key)
        if entry is None:
            # first call with this shape runs eagerly: warms kernel attributes and the positional-embedding cache
            self._graphs[key] = "warm"
            return self._run(P, *args, B, T, nb, H, W, dev)
        if entry == "warm":
            static_in = [a.clone() for a in args]
            graph = torch.cuda.CUDAGraph()
            torch.cuda.synchronize()
            l0 = ops.launch_count()
            with torch.cuda.graph(graph):
                static_out = self._run(P, *static_in, B, T, nb, H, W, dev)
            entry = (graph, static_in, static_out, ops.launch_count() - l0)
            self._graphs[key] = entry
        graph, static_in, static_out, nlaunch = entry
        for dst, src in zip(static_in, args):
            dst.copy_(src)
        graph.replay()
        self.replayed_launches += nlaunch
        return static_out.clone()

    # -- embeddings that depend only on (sigma, y, context, T): computed once per forward ----------------
    def _embeddings(self, P, timesteps, ctx2d, y, B, T, dev):
        te = self.time_embed_dim
        t_emb = torch.empty(B, self.model_channels, device=dev)
        ops.timestep_embedding(timesteps, t_emb, self.model_channels)
        h1 = torch.empty(B, te, device=dev)
        emb = torch.empty(B, te, device=dev)
        # Linear -> SiLU -> Linear: the SiLU is applied on the consumer's input side
        ops.small_linear(t_emb, P["time_embed.0.weight"], P["time_embed.0.bias"], h1)
        ops.small_linear(h1, P["time_embed.2.weight"], P["time_embed.2.bias"], emb, act_in=ops.ACT_SILU)
        ops.small_linear(y, P["label_emb.0.0.weight"], P["label_emb.0.0.bias"], h1)
        ops.small_linear(h1, P["label_emb.0.2.weight"], P["label_emb.0.2.bias"], emb, act_in=ops.ACT_SILU,
                         accumulate=True)
        # every ResBlock's emb_layers (SiLU -> Linear) in one launch: [B, sum(Cout)]
        emb_all = torch.empty(B, P["emb_total"], device=dev)
        ops.small_linear(emb, P["emb_all.weight"], P["emb_all.bias"], emb_all, act_in=ops.ACT_SILU)
        ctx_dim = self.context_dim
        if ctx2d.shape[1] > ctx_dim:
            # multi-token context: K | V of every attn2 layer over all context rows ((B + time-context rows) * M) in
            # one GEMM; the layers' attention reads its column slices in place
            rows = ctx2d.numel() // ctx_dim
            ctx_bf = torch.empty(rows, ctx_dim, device=dev, dtype=torch.bfloat16)
            ops.nchw_f32_to_nhwc_bf16(ctx2d.view(1, 1, rows, ctx_dim), ctx_bf)       # C = 1: a plain bf16 conversion
            return emb_all, self._linear(P, "ckv_all", ctx_bf, rows)
        # single-token cross-attention: v = to_v(ctx) for every layer in one launch, then to_out per layer
        nctx = ctx2d.shape[0]  # B, plus one time-context row per video when frame-sharded
        v_all = torch.empty(nctx, P["cv_total"], device=dev)
        ops.small_linear(ctx2d, P["cv_all.weight"], None, v_all)
        cross = torch.empty(nctx, P["cv_total"], device=dev)
        for base, (o, c) in P["cv_off"].items():
            ops.small_linear(v_all[:, o:o + c], P[base + ".attn2.to_out.0.weight"], P[base + ".attn2.to_out.0.bias"],
                             cross[:, o:o + c])
        return emb_all, cross

    def _pos_emb(self, P, name: str, c: int, B: int, T: int, dev) -> torch.Tensor:
        """time_pos_embed(timestep_embedding(arange(T))) (video_attention.py:266-276): input-independent, cached
        per (layer, B, T) until the weights are re-packed."""
        t0 = self.view_shard.t0 if self.view_shard is not None else 0  # frame ids are global (arange(T_video))
        key = (name, B, T, t0)
        cache = P["pos_cache"]
        if key not in cache:
            frames = torch.arange(t0, t0 + T, device=dev, dtype=torch.float32).repeat(B // T)
            t_emb = torch.empty(B, c, device=dev)
            ops.timestep_embedding(frames, t_emb, c, float(self.max_ddpm_temb_period))
            h = torch.empty(B, 4 * c, device=dev)
            out = torch.empty(B, c, device=dev)
            ops.small_linear(t_emb, P[name + ".time_pos_embed.0.weight"], P[name + ".time_pos_embed.0.bias"], h)
            ops.small_linear(h, P[name + ".time_pos_embed.2.weight"], P[name + ".time_pos_embed.2.bias"], out,
                             act_in=ops.ACT_SILU)
            cache[key] = out
        return cache[key]

    def _res_block(self, P, st: _Step, x, emb_all, B, T, nb, h, w):
        """VideoResBlock.forward (video_model.py:62-81) = ResBlock 2-D (openaimodel.py:338-364) + time_stack
        ResBlock 3-D + AlphaBlender, fused as: x_s + (1-alpha) * conv_t(...)."""
        nm, cin, cout = st.name, st.cin, st.cout
        hw = h * w
        rows = B * hw
        E = emb_all.shape[1]
        o2, _ = P["emb_off"][nm]
        o3, _ = P["emb_off"][nm + ".time_stack"]
        a = self._gn(P, nm + ".in_layers.0", x, hw, B, cin, 1e-5, True)
        h1 = self._conv3x3(P, nm + ".in_layers.2", a, B, h, w, cin, fbias=emb_all[:, o2:], ldfb=E, rows_per_frame=hw)
        a = self._gn(P, nm + ".out_layers.0", h1, hw, B, cout, 1e-5, True)
        skip = x if cin == cout else self._linear(P, nm + ".skip_connection", x, rows)
        xs = self._conv3x3(P, nm + ".out_layers.3", a, B, h, w, cout, r1=skip, s1=1.0, out=h1)
        return self._time_stack(P, nm + ".time_stack", xs, hw, T, nb, cout, s0=1.0 - P[nm + ".alpha"],
                                fbias=emb_all[:, o3:], ldfb=E, rows_per_frame=hw)

    def _attn_block(self, P, st: _Step, x, cross, B, T, nb, h, w, M: int = 1):
        """SpatialVideoTransformer.forward (video_attention.py:230-301) with depth 1.  M = context tokens.  With one
        token, `cross` holds every layer's attn2 output (fp32 rows, folded into attn1.to_out's epilogue as a bias); with
        more, it holds every layer's attn2 K | V rows (bf16, one row per context token) and attn2 runs on its own
        (_cross_attn)."""
        nm, c = st.name, st.cin
        hw = h * w
        rows = B * hw
        heads = c // 64
        scale = 64 ** -0.5
        X = cross.shape[1]
        tb, ts = nm + ".transformer_blocks.0", nm + ".time_stack.0"
        off = P["cv_off"] if M == 1 else P["ckv_off"]
        os_, _ = off[tb]
        ot, _ = off[ts]
        dev = x.device

        def ln(key, src, **kw):
            out = torch.empty(rows, c, device=dev, dtype=torch.bfloat16)
            return ops.layernorm(src, out, P[key + ".weight"], P[key + ".bias"], rows, c, **kw)

        xn = self._gn(P, nm + ".norm", x, hw, B, c, 1e-6, False)
        t = self._linear(P, nm + ".proj_in", xn, rows)
        # --- BasicTransformerBlock (attention.py:556-577)
        a = ln(tb + ".norm1", t)
        qkv = self._linear(P, tb + ".attn1.qkv", a, rows)
        o = torch.empty(rows, c, device=dev, dtype=torch.bfloat16)
        ops.attention_spatial(qkv, o, B, hw, heads, scale)
        if M == 1:
            self._linear(P, tb + ".attn1.to_out.0", o, rows, out=t, r1=t, s1=1.0,
                         fbias=cross[:, os_:], ldfb=X, rows_per_frame=hw)          # + attn2 (single key) folded in
        else:
            self._linear(P, tb + ".attn1.to_out.0", o, rows, out=t, r1=t, s1=1.0)
            # each frame attends to its own M context tokens (attention.py:571-572)
            self._cross_attn(P, tb, t, o, a, cross[:, os_:os_ + 2 * c], B, hw, M, M)
        a = ln(tb + ".norm3", t)
        g = self._linear(P, tb + ".ff.net.0.proj", a, rows, act=ops.ACT_GEGLU)
        self._linear(P, tb + ".ff.net.2", g, rows, out=t, r1=t, s1=1.0)
        # --- VideoTransformerBlock (video_attention.py:109-140) on x + emb
        pos = self._pos_emb(P, nm, c, B, T, dev)
        xm = torch.empty(rows, c, device=dev, dtype=torch.bfloat16)
        a = ln(ts + ".norm_in", t, add=pos, ysum=xm, rows_per_frame=hw)
        g = self._linear(P, ts + ".ff_in.net.0.proj", a, rows, act=ops.ACT_GEGLU)
        self._linear(P, ts + ".ff_in.net.2", g, rows, out=xm, r1=xm, s1=1.0)
        a = ln(ts + ".norm1", xm)
        vs = self.view_shard
        kv_buf = send = kv_dst = None
        if vs is not None:
            kv_buf, send = vs.kv_slots(nb, hw, 2 * c, torch.bfloat16, dev)
            kv_dst = vs.kv_fused(kv_buf)
        # frame-sharded over peer memory: the projection GEMM itself delivers its K|V columns into every rank's gather
        # buffer (fused GEMM -> all-gather: the epilogue's TMA sub-tile stores go out once more per rank over NVLink)
        qkv = self._linear(P, ts + ".attn1.qkv", a, rows, out=qkv,
                           **({"kv": (c, kv_dst, 2 * c)} if kv_dst is not None else {}))
        if vs is None:
            ops.attention_temporal(qkv, o, nb, T, hw, heads, scale)
            # temporal cross-attention context = context[::T] (video_attention.py:250): the rows of frame 0 of each
            # video, row b*T of `cross` (one token) or rows b*T*M .. b*T*M + M - 1 (M tokens)
            tc0, tc_ld = 0, X * T
        else:
            # frame-sharded: all-gather the packed K|V rows of every rank's frames, attend in place through the
            # per-frame row table; the time context (global frame 0 of each CFG half) is rows B.. of `cross`
            # (B*M.. with M tokens)
            if kv_dst is not None:
                gathered = vs.gather_signal(kv_buf)
            else:
                ops.copy_channels(qkv[:, c:], 3 * c, send, 2 * c, rows, 2 * c)
                gathered = vs.gather_rows(send, kv_buf, rows)
            kv_row, kv_bstride = vs.kv_table(nb, hw)
            ops.attention_temporal_kv(qkv, gathered, o, nb, T, hw, heads, kv_row, kv_bstride, scale)
            tc0, tc_ld = B, X
        if M == 1:
            self._linear(P, ts + ".attn1.to_out.0", o, rows, out=xm, r1=xm, s1=1.0,
                         fbias=cross[tc0:, ot:], ldfb=tc_ld, rows_per_frame=T * hw)
        else:
            self._linear(P, ts + ".attn1.to_out.0", o, rows, out=xm, r1=xm, s1=1.0)
            kstride = T * M if vs is None else M
            self._cross_attn(P, ts, xm, o, a, cross[tc0 * M:, ot:ot + 2 * c], nb, T * hw, M, kstride)
        a = ln(ts + ".norm3", xm)
        g = self._linear(P, ts + ".ff.net.0.proj", a, rows, out=g, act=ops.ACT_GEGLU)
        alpha = P[nm + ".alpha"]
        # x = alpha * x_spatial + (1 - alpha) * (ff(.) + x_mix)   (AlphaBlender, util.py:358-369)
        self._linear(P, ts + ".ff.net.2", g, rows, out=t, r1=xm, s1=1.0 - alpha, r2=t, s2=alpha, s0=1.0 - alpha)
        return self._linear(P, nm + ".proj_out", t, rows, out=xn, r1=x, s1=1.0)

    def _cross_attn(self, P, base, x, qbuf, obuf, kv, nbatch, nq, M, kv_bstride):
        """x += attn2(norm2(x), context) over a context of M > 1 tokens (attention.py:286-349): LayerNorm, to_q GEMM,
        attention of item b's nq rows against the K | V rows `kv` [b * kv_bstride, + M), to_out GEMM with the residual
        in its epilogue.  qbuf / obuf: [rows, C] scratch buffers."""
        rows, c = x.shape
        ops.layernorm(x, obuf, P[base + ".norm2.weight"], P[base + ".norm2.bias"], rows, c)
        q = self._linear(P, base + ".attn2.to_q", obuf, rows, out=qbuf)
        ops.attention_cross(q, kv, obuf, nbatch, nq, M, c // 64, 64 ** -0.5, kv_bstride=kv_bstride)
        self._linear(P, base + ".attn2.to_out.0", obuf, rows, out=x, r1=x, s1=1.0)

    def _run(self, P, x, timesteps, ctx2d, y, B, T, nb, H, W, dev):
        if self.view_shard is not None:
            self.view_shard.begin("unet")     # one-sided transport: rewind the exchange sites, bump the epoch
        n_norms = sum({"res": 4, "attn": 1, "out": 1}.get(st.kind, 0) for st in self.steps)
        with self._stats_pool(n_norms * B, dev):
            return self._run_inner(P, x, timesteps, ctx2d, y, B, T, nb, H, W, dev)

    def _run_inner(self, P, x, timesteps, ctx2d, y, B, T, nb, H, W, dev):
        M = ctx2d.shape[1] // self.context_dim
        if M > 1:
            self._pack_cross(P)
        emb_all, cross = self._embeddings(P, timesteps, ctx2d, y, B, T, dev)
        cur = torch.empty(B * H * W, self.in_channels, device=dev, dtype=torch.bfloat16)
        ops.nchw_f32_to_nhwc_bf16(x, cur)
        h, w = H, W
        saved: List[Tuple[torch.Tensor, int]] = []
        ch = self.in_channels
        for st in self.steps:
            if st.kind == "conv_in":
                cur = self._conv3x3(P, st.name, cur, B, h, w, st.cin)
                ch = st.cout
            elif st.kind == "save":
                saved.append((cur, ch))
            elif st.kind == "res":
                cur = self._res_block(P, st, cur, emb_all, B, T, nb, h, w)
                ch = st.cout
            elif st.kind == "attn":
                cur = self._attn_block(P, st, cur, cross, B, T, nb, h, w, M)
            elif st.kind == "down":
                cur = self._conv3x3(P, st.name + ".op", cur, B, h, w, st.cin, stride=2)
                h, w = (h + 2 - 3) // 2 + 1, (w + 2 - 3) // 2 + 1
            elif st.kind == "up":
                up = torch.empty(B * 4 * h * w, ch, device=dev, dtype=torch.bfloat16)
                ops.upsample_nearest2x(cur, up, B, h, w, ch)
                h, w = 2 * h, 2 * w
                cur = self._conv3x3(P, st.name + ".conv", up, B, h, w, ch)
            elif st.kind == "cat":
                skip, sc = saved.pop()
                rows = B * h * w
                cat = torch.empty(rows, ch + sc, device=dev, dtype=torch.bfloat16)
                ops.copy_channels(cur, ch, cat, ch + sc, rows, ch)
                ops.copy_channels(skip, sc, cat[:, ch:], ch + sc, rows, sc)
                cur, ch = cat, ch + sc
            if st.kind in ("conv_in", "res", "attn", "down", "up"):
                self._tap(st.name, cur, B, ch, h, w)
            if st.kind == "out":
                a = self._gn(P, "out.0", cur, h * w, B, st.cin, 1e-5, True)
                o = self._conv3x3(P, "out.2", a, B, h, w, st.cin, out_dtype=torch.float32)
                out = torch.empty(B, self.out_channels, h, w, device=dev, dtype=torch.float32)
                ops.nhwc_to_nchw_f32(o, out, B, self.out_channels, h * w, o.shape[1])
                return out
        raise AssertionError("plan has no output step")
