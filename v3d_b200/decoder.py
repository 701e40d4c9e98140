"""H100-native first-stage decode: drop-ins for `sgm.modules.autoencoding.temporal_ae.VideoDecoder`
(temporal_ae.py:293-349 over diffusionmodules/model.py:604-748) and the decode side of
`sgm.models.autoencoder.AutoencodingEngine` (autoencoder.py:196-212).

Same constructor kwargs and `state_dict()` keys as the reference decoder; forward(z, timesteps=T) takes the
reference's NCHW fp32 latents and returns NCHW fp32 images.  Internally NHWC bf16 with fp32 norms (the
reference decodes in fp32, video_diffusion.py:195; bf16 here is the BASELINE.json configuration and its
tolerance is stated in tests/test_parity_gpu.py).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple, Union

import torch
import torch.nn as nn

from . import ops
from .unet import KernelModule, _register


class VideoDecoder(KernelModule):
    available_time_modes = ["all", "conv-only", "attn-only"]

    def __init__(
        self,
        *,
        ch: int,
        out_ch: int,
        ch_mult: Sequence[int] = (1, 2, 4, 8),
        num_res_blocks: int,
        attn_resolutions: Sequence[int],
        dropout: float = 0.0,
        resamp_with_conv: bool = True,
        in_channels: int,
        resolution: int,
        z_channels: int,
        give_pre_end: bool = False,
        tanh_out: bool = False,
        use_linear_attn: bool = False,
        attn_type: str = "vanilla",
        video_kernel_size: Union[int, list] = 3,
        alpha: float = 0.0,
        merge_strategy: str = "learned",
        time_mode: str = "conv-only",
        **ignorekwargs,
    ):
        super().__init__()
        assert time_mode in self.available_time_modes, f"time_mode parameter has to be in {self.available_time_modes}"
        bad = []
        if time_mode != "conv-only":
            bad.append(f"time_mode={time_mode}")
        if list(attn_resolutions):
            bad.append("attn_resolutions != []")
        if give_pre_end or tanh_out or use_linear_attn or not resamp_with_conv or dropout != 0.0:
            bad.append("give_pre_end/tanh_out/use_linear_attn/resamp_with_conv=False/dropout")
        if attn_type not in ("vanilla", "vanilla-xformers"):
            bad.append(f"attn_type={attn_type}")
        ks = [video_kernel_size] * 3 if isinstance(video_kernel_size, int) else list(video_kernel_size)
        if ks != [3, 1, 1]:
            bad.append(f"video_kernel_size={video_kernel_size}")
        if merge_strategy not in ("learned", "fixed"):
            raise ValueError(f"unknown merge strategy {merge_strategy}")
        if ch % 64 or out_ch > 4:
            bad.append("ch % 64 != 0 or out_ch > 4")
        if bad:
            raise NotImplementedError("v3d_b200.VideoDecoder covers the V3D_512 decoder configuration; unsupported: "
                                      + ", ".join(bad))
        self.ch, self.out_ch, self.ch_mult = ch, out_ch, list(ch_mult)
        self.num_res_blocks = num_res_blocks
        self.z_channels = z_channels
        self.resolution = resolution
        self.alpha0 = alpha
        self.merge_strategy = merge_strategy
        self.time_mode = time_mode
        self.num_resolutions = len(self.ch_mult)
        self.debug_taps: Optional[dict] = None  # tests: {block name: None} -> filled with NCHW fp32 outputs
        for key, shape in self.param_shapes().items():
            _register(self, key, self._init_value(key, shape))

    # --------------------------------------------------------------------------------------------
    def _blocks(self) -> List[Tuple[str, int, int]]:
        """(name, cin, cout) of every VideoResBlock in execution order, with 'attn' / 'up' markers."""
        out: List[Tuple[str, int, int]] = []
        block_in = self.ch * self.ch_mult[-1]
        out.append(("mid.block_1", block_in, block_in))
        out.append(("@attn:mid.attn_1", block_in, block_in))
        out.append(("mid.block_2", block_in, block_in))
        for lvl in range(self.num_resolutions - 1, -1, -1):
            block_out = self.ch * self.ch_mult[lvl]
            for j in range(self.num_res_blocks + 1):
                out.append((f"up.{lvl}.block.{j}", block_in, block_out))
                block_in = block_out
            if lvl != 0:
                out.append((f"@up:up.{lvl}.upsample.conv", block_in, block_in))
        return out

    def param_shapes(self) -> Dict[str, Tuple[int, ...]]:
        table: Dict[str, Tuple[int, ...]] = {}

        def conv(key, co, ci, *ks):
            table[key + ".weight"] = (co, ci, *ks)
            table[key + ".bias"] = (co,)

        def affine(key, c):
            table[key + ".weight"] = (c,)
            table[key + ".bias"] = (c,)

        top = self.ch * self.ch_mult[-1]
        conv("conv_in", top, self.z_channels, 3, 3)
        last = top
        for name, ci, co in self._blocks():
            if name.startswith("@attn:"):
                key = name[6:]
                affine(key + ".norm", ci)
                for n in ("q", "k", "v", "proj_out"):
                    conv(f"{key}.{n}", ci, ci, 1, 1)
            elif name.startswith("@up:"):
                conv(name[4:], co, ci, 3, 3)
            else:
                affine(name + ".norm1", ci)
                conv(name + ".conv1", co, ci, 3, 3)
                affine(name + ".norm2", co)
                conv(name + ".conv2", co, co, 3, 3)
                if ci != co:
                    conv(name + ".nin_shortcut", co, ci, 1, 1)
                ts = name + ".time_stack"
                affine(ts + ".in_layers.0", co)
                conv(ts + ".in_layers.2", co, co, 3, 1, 1)
                affine(ts + ".out_layers.0", co)
                conv(ts + ".out_layers.3", co, co, 3, 1, 1)
                table[name + ".mix_factor"] = (1,)
            last = co
        affine("norm_out", last)
        conv("conv_out", self.out_ch, last, 3, 3)
        conv("conv_out.time_mix_conv", self.out_ch, self.out_ch, 3, 1, 1)
        return table

    def _init_value(self, key: str, shape) -> torch.Tensor:
        if torch.empty(0).device.type == "meta":
            return torch.empty(shape)
        if key.endswith("mix_factor"):
            return torch.full(shape, float(self.alpha0))
        if len(shape) == 1:
            is_norm = "norm" in key.rsplit(".", 2)[-2] or ".in_layers.0." in key or ".out_layers.0." in key
            if is_norm:
                return torch.ones(shape) if key.endswith(".weight") else torch.zeros(shape)
            return torch.zeros(shape)
        if ".time_stack.out_layers.3." in key:
            return torch.zeros(shape)  # zero_module (openaimodel.py:306-314)
        bound = 1.0 / math.sqrt(math.prod(shape[1:]))
        return (torch.rand(shape) * 2.0 - 1.0) * bound

    @torch.no_grad()
    def randomize_zero_modules_(self, seed: int = 1) -> "VideoDecoder":
        gen = torch.Generator(device="cpu").manual_seed(seed)
        for key, p in self.named_parameters():
            if ".time_stack.out_layers.3." in key:
                fan = math.prod(p.shape[1:]) if p.ndim > 1 else 1
                val = torch.randn(p.shape, generator=gen) / math.sqrt(fan) if p.ndim > 1 else 0.05 * torch.randn(
                    p.shape, generator=gen)
                p.copy_(val.to(p.device))
            elif key.endswith("mix_factor"):
                p.copy_(torch.randn(p.shape, generator=gen).to(p.device))
        self._invalidate()
        return self

    # --------------------------------------------------------------------------------------------
    def _pack(self, dev: torch.device) -> dict:
        sd = {k: v.detach() for k, v in self.named_parameters()}
        P: dict = {}

        def affine(key):
            P[key + ".weight"] = self._f32(sd[key + ".weight"])
            P[key + ".bias"] = self._f32(sd[key + ".bias"])

        def conv1x1(key):
            w = sd[key + ".weight"]
            P[key + ".weight"] = self._bf(w.reshape(w.shape[0], w.shape[1]))
            P[key + ".bias"] = self._f32(sd[key + ".bias"])

        kpad = (9 * self.z_channels + 63) // 64 * 64
        P["conv_in.weight"], P["conv_in.bias"] = self._pack_conv3x3(sd["conv_in.weight"], sd["conv_in.bias"], kpad)
        mix_keys = [k for k in sd if k.endswith("mix_factor")]
        mix = torch.stack([sd[k].reshape(()) for k in mix_keys]).float().cpu().tolist()
        for k, v in zip(mix_keys, mix):
            # temporal_ae.VideoResBlock.get_alpha (temporal_ae.py:56-62)
            P[k[:-len(".mix_factor")] + ".alpha"] = v if self.merge_strategy == "fixed" else 1.0 / (1.0 + math.exp(-v))
        for name, ci, co in self._blocks():
            if name.startswith("@attn:"):
                key = name[6:]
                affine(key + ".norm")
                wq, wk = sd[key + ".q.weight"].reshape(ci, ci), sd[key + ".k.weight"].reshape(ci, ci)
                P[key + ".qk.weight"] = self._bf(torch.cat([wq, wk], 0))
                P[key + ".qk.bias"] = self._f32(torch.cat([sd[key + ".q.bias"], sd[key + ".k.bias"]], 0))
                P[key + ".v.weight"] = self._bf(sd[key + ".v.weight"].reshape(ci, ci))
                P[key + ".v.bias"] = self._f32(sd[key + ".v.bias"])
                conv1x1(key + ".proj_out")
            elif name.startswith("@up:"):
                key = name[4:]
                P[key + ".weight"], P[key + ".bias"] = self._pack_conv3x3(sd[key + ".weight"], sd[key + ".bias"])
            else:
                affine(name + ".norm1")
                affine(name + ".norm2")
                for cname in (".conv1", ".conv2"):
                    P[name + cname + ".weight"], P[name + cname + ".bias"] = self._pack_conv3x3(
                        sd[name + cname + ".weight"], sd[name + cname + ".bias"])
                if ci != co:
                    conv1x1(name + ".nin_shortcut")
                ts = name + ".time_stack"
                affine(ts + ".in_layers.0")
                affine(ts + ".out_layers.0")
                for cname in (".in_layers.2", ".out_layers.3"):
                    P[ts + cname + ".weight"], P[ts + cname + ".bias"] = self._pack_tconv(
                        sd[ts + cname + ".weight"], sd[ts + cname + ".bias"])
        affine("norm_out")
        P["conv_out.weight"], P["conv_out.bias"] = self._pack_conv3x3(sd["conv_out.weight"], sd["conv_out.bias"])
        P["time_mix.weight"] = self._f32(sd["conv_out.time_mix_conv.weight"].reshape(self.out_ch, self.out_ch, 3))
        P["time_mix.bias"] = self._f32(sd["conv_out.time_mix_conv.bias"])
        return P

    # --------------------------------------------------------------------------------------------
    def _video_res_block(self, P, name, ci, co, x, B, T, nb, h, w):
        """temporal_ae.VideoResBlock.forward (temporal_ae.py:64-83): ResnetBlock (model.py:131-151), then
        alpha * time_stack(x) + (1 - alpha) * x  ==  x + alpha * conv_t(...)."""
        hw = h * w
        rows = B * hw
        a = self._gn(P, name + ".norm1", x, hw, B, ci, 1e-6, True)
        h1 = self._conv3x3(P, name + ".conv1", a, B, h, w, ci)
        a = self._gn(P, name + ".norm2", h1, hw, B, co, 1e-6, True)
        skip = x if ci == co else self._linear(P, name + ".nin_shortcut", x, rows)
        xs = self._conv3x3(P, name + ".conv2", a, B, h, w, co, r1=skip, s1=1.0, out=h1)
        # (frame-sharded: T is this rank's block; the 3-D norms all-reduce their statistics, the convs read halos)
        ts = name + ".time_stack"
        norm = self._gn_halo if self.view_shard is not None else None
        a = (norm(P, ts + ".in_layers.0", xs, hw, T, nb, co, 1e-5, True) if norm else
             self._gn(P, ts + ".in_layers.0", xs, T * hw, nb, co, 1e-5, True, hw=hw))
        h2 = torch.empty(rows, co, device=x.device, dtype=torch.bfloat16)
        self._tconv(P, ts + ".in_layers.2", a, h2, hw, T, nb, co)
        a = (norm(P, ts + ".out_layers.0", h2, hw, T, nb, co, 1e-5, True) if norm else
             self._gn(P, ts + ".out_layers.0", h2, T * hw, nb, co, 1e-5, True, hw=hw))
        self._tconv(P, ts + ".out_layers.3", a, h2, hw, T, nb, co, r1=xs, s1=1.0, s0=P[name + ".alpha"])
        return h2

    def _attn(self, P, key, c, x, B, h, w):
        """AttnBlock (model.py:161-201): single head, d = C, over h*w tokens per frame.
        S = q k^T (fp32), softmax, O = P v; v's bias is added after P.v (rows of P sum to 1)."""
        hw = h * w
        rows = B * hw
        dev = x.device
        xn = self._gn(P, key + ".norm", x, hw, B, c, 1e-6, False)
        qk = self._linear(P, key + ".qk", xn, rows)                       # [rows, 2C]: q | k
        # V^T for all frames: vt[d, f*hw + j] = sum_k Wv[d,k] xn[f*hw + j, k]
        vt = torch.empty(c, rows, device=dev, dtype=torch.bfloat16)
        ops.gemm(P[key + ".v.weight"], xn, vt, K=c, N=rows, rows_per_batch=c)
        scores = torch.empty(B, hw, hw, device=dev, dtype=torch.float32)
        k_view = qk[:, c:]
        ops.gemm(qk, k_view, scores, K=c, N=hw, rows_per_batch=hw, batch=B, lda=2 * c, ldb=2 * c,
                 a_batch_stride=hw * 2 * c, b_batch_stride=hw * 2 * c)
        probs = torch.empty(B, hw, hw, device=dev, dtype=torch.bfloat16)
        ops.softmax_rows_f32(scores, probs, B * hw, hw, float(c) ** -0.5)
        del scores
        o = torch.empty(rows, c, device=dev, dtype=torch.bfloat16)
        ops.gemm(probs, vt, o, K=hw, N=c, rows_per_batch=hw, batch=B, a_batch_stride=hw * hw, ldb=rows,
                 b_batch_stride=hw, bias=P[key + ".v.bias"])
        return self._linear(P, key + ".proj_out", o, rows, out=xn, r1=x, s1=1.0)

    def _tap(self, name, x, B, c, h, w):
        """With `debug_taps` holding `name`: the block output x (bf16 NHWC) widened to fp32 NCHW, which is exactly
        the next block's input.  Launches nothing when taps are off."""
        if self.debug_taps is not None and name in self.debug_taps:
            tap = torch.empty(B, c, h, w, device=x.device, dtype=torch.float32)
            ops.nhwc_to_nchw_f32(x, tap, B, c, h * w, c)
            self.debug_taps[name] = tap

    def forward(self, z: torch.Tensor, timesteps: Optional[int] = None, skip_video: bool = False, **kwargs):
        if skip_video:
            raise NotImplementedError("skip_video decode is not implemented")
        ops.require_current_device(z, "v3d_b200.VideoDecoder.forward")
        B, zc, H, W = z.shape
        T = int(timesteps) if timesteps else B
        assert B % T == 0 and zc == self.z_channels
        nb = B // T
        vs = self.view_shard
        if vs is not None:
            # frame-sharded decode: z holds this rank's block of ONE video decoded as a whole (the reference with
            # en_and_decode_n_samples_a_time = T, video_diffusion.py:182-210)
            assert nb == 1 and T == vs.tl, f"view-sharded decode expects this rank's {vs.tl} frames, got {B} / T={T}"
        with torch.no_grad():
            return self._run(self.packed(), z, B, T, nb, H, W)

    def _run(self, P: dict, z: torch.Tensor, B: int, T: int, nb: int, H: int, W: int) -> torch.Tensor:
        """The launch schedule of one decode (Decoder.forward, model.py:715-748, through VideoDecoder)."""
        vs = self.view_shard
        if vs is not None:
            if self.debug_taps is not None:
                raise NotImplementedError("debug_taps are not supported by the frame-sharded decode")
            vs.begin("decoder")
        dev, zc = z.device, self.z_channels
        n_norms = 4 * sum(1 for n, _, _ in self._blocks() if not n.startswith("@")) + 2
        object.__setattr__(self, "_gn_pool", [torch.zeros(n_norms * B * 64, device=dev, dtype=torch.float64), 0])
        try:
            cur = torch.empty(B * H * W, zc, device=dev, dtype=torch.bfloat16)
            ops.nchw_f32_to_nhwc_bf16(z.float().contiguous(), cur)
            h, w = H, W
            cur = self._conv3x3(P, "conv_in", cur, B, h, w, zc)
            ch = self.ch * self.ch_mult[-1]
            self._tap("conv_in", cur, B, ch, h, w)
            for name, ci, co in self._blocks():
                if name.startswith("@attn:"):
                    if (h * w) % 64 != 0 or ci % 64 != 0:
                        raise NotImplementedError("decoder AttnBlock needs h*w % 64 == 0")
                    cur = self._attn(P, name[6:], ci, cur, B, h, w)
                elif name.startswith("@up:"):
                    up = torch.empty(B * 4 * h * w, ci, device=dev, dtype=torch.bfloat16)
                    ops.upsample_nearest2x(cur, up, B, h, w, ci)
                    h, w = 2 * h, 2 * w
                    cur = self._conv3x3(P, name[4:], up, B, h, w, ci)
                    del up
                else:
                    cur = self._video_res_block(P, name, ci, co, cur, B, T, nb, h, w)
                    ch = co
                self._tap(name.rsplit(":", 1)[-1], cur, B, ch, h, w)
            a = self._gn(P, "norm_out", cur, h * w, B, ch, 1e-6, True)
            if vs is None:
                o = self._conv3x3(P, "conv_out", a, B, h, w, ch, out_dtype=torch.float32)   # [rows, 16] fp32
                out = torch.empty(B, self.out_ch, h, w, device=dev, dtype=torch.float32)
                ops.time_mix_conv(o, o.shape[1], P["time_mix.weight"], P["time_mix.bias"], out, nb, T, h * w,
                                  self.out_ch)
            else:
                # AE3DConv's time_mix_conv (temporal_ae.py:101-107) is one more (3,1,1) conv: conv_out lands in the
                # interior of a halo'd fp32 buffer, the mix runs over T + 2 frames and the two halo frames are dropped
                cop = P["conv_out.weight"].shape[0]
                pad = vs.new_pad((1, T + 2, h * w, cop), torch.float32, dev)
                self._conv3x3(P, "conv_out", a, B, h, w, ch, out=pad[0, 1:T + 1].view(B * h * w, cop))
                vs.exchange_halos(pad)
                full = torch.empty(T + 2, self.out_ch, h, w, device=dev, dtype=torch.float32)
                ops.time_mix_conv(pad.view(-1, cop), cop, P["time_mix.weight"], P["time_mix.bias"], full, 1, T + 2,
                                  h * w, self.out_ch)
                out = full[1:T + 1].contiguous()
        finally:
            object.__setattr__(self, "_gn_pool", None)   # also after a failed run (OOM mid-schedule)
        return out


class AutoencodingEngine(nn.Module):
    """Drop-in for `sgm.models.autoencoder.AutoencodingEngine` (autoencoder.py:128-212).

    `decoder_config` is always built natively; state_dict keys keep the `decoder.` prefix so
    `first_stage_model.decoder.*` checkpoints load unchanged.  The encode side (SURVEY.md 8(f) rank 1, once per image)
    is built natively only when `encoder_config.target` names this package's Encoder
    (`v3d_b200.sgm.modules.diffusionmodules.model.Encoder`); with the reference's target it stays decode-only, as
    scripts/pub/V3D_512.py:145-162 encodes with a separately loaded `ae_model`.
    """

    def __init__(self, *args, decoder_config: Optional[dict] = None, encoder_config=None, loss_config=None,
                 regularizer_config=None, **kwargs):
        super().__init__()
        assert decoder_config is not None
        params = dict(decoder_config.get("params", dict())) if hasattr(decoder_config, "get") else dict(decoder_config)
        self.decoder = VideoDecoder(**params)
        self.encoder = None
        self.regularization = None
        target = str(encoder_config.get("target", "")) if hasattr(encoder_config, "get") else ""
        if target.startswith("v3d_b200."):
            from .encoder import DiagonalGaussianRegularizer, Encoder

            self.encoder = Encoder(**dict(encoder_config.get("params", dict())))
            rparams = dict(regularizer_config.get("params", dict())) if hasattr(regularizer_config, "get") else {}
            self.regularization = DiagonalGaussianRegularizer(**rparams)

    def encode(self, x: torch.Tensor, return_reg_log: bool = False, unregularized: bool = False):
        """autoencoder.py:196-208: z = encoder(x); (z, log) = regularization(z)."""
        if self.encoder is None:
            raise NotImplementedError("this AutoencodingEngine was built decode-only; point encoder_config.target at "
                                      "v3d_b200.sgm.modules.diffusionmodules.model.Encoder to build the native encoder")
        z = self.encoder(x)
        if unregularized:
            return z, dict()
        z, reg_log = self.regularization(z)
        return (z, reg_log) if return_reg_log else z

    def decode(self, z: torch.Tensor, **kwargs) -> torch.Tensor:
        return self.decoder(z, **kwargs)

    def get_last_layer(self):
        return self.decoder.get_parameter("conv_out.time_mix_conv.weight")
