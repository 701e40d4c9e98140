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
from .first_stage import FirstStage
from .kernel_module import _register


class VideoDecoder(FirstStage):
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
        conv, affine = self._conv_shape, self._affine_shape
        top = self.ch * self.ch_mult[-1]
        conv(table, "conv_in", top, self.z_channels, 3, 3)
        last = top
        for name, ci, co in self._blocks():
            if name.startswith("@attn:"):
                self._attn_block_shapes(table, name[6:], ci)
            elif name.startswith("@up:"):
                conv(table, name[4:], co, ci, 3, 3)
            else:
                self._resnet_block_shapes(table, name, ci, co)
                ts = name + ".time_stack"
                affine(table, ts + ".in_layers.0", co)
                conv(table, ts + ".in_layers.2", co, co, 3, 1, 1)
                affine(table, ts + ".out_layers.0", co)
                conv(table, ts + ".out_layers.3", co, co, 3, 1, 1)
                table[name + ".mix_factor"] = (1,)
            last = co
        affine(table, "norm_out", last)
        conv(table, "conv_out", self.out_ch, last, 3, 3)
        conv(table, "conv_out.time_mix_conv", self.out_ch, self.out_ch, 3, 1, 1)
        return table

    def _init_value(self, key: str, shape) -> torch.Tensor:
        if torch.empty(0).device.type != "meta":
            if key.endswith("mix_factor"):
                return torch.full(shape, float(self.alpha0))
            if ".time_stack.out_layers.3." in key:
                return torch.zeros(shape)  # zero_module (openaimodel.py:306-314)
        return super()._init_value(key, shape)

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
        kpad = (9 * self.z_channels + 63) // 64 * 64
        P["conv_in.weight"], P["conv_in.bias"] = self._pack_conv3x3(sd["conv_in.weight"], sd["conv_in.bias"], kpad)
        mix_keys = [k for k in sd if k.endswith("mix_factor")]
        mix = torch.stack([sd[k].reshape(()) for k in mix_keys]).float().cpu().tolist()
        for k, v in zip(mix_keys, mix):
            # temporal_ae.VideoResBlock.get_alpha (temporal_ae.py:56-62)
            P[k[:-len(".mix_factor")] + ".alpha"] = v if self.merge_strategy == "fixed" else 1.0 / (1.0 + math.exp(-v))
        for name, ci, co in self._blocks():
            if name.startswith("@attn:"):
                self._pack_attn_block(P, sd, name[6:], ci)
            elif name.startswith("@up:"):
                key = name[4:]
                P[key + ".weight"], P[key + ".bias"] = self._pack_conv3x3(sd[key + ".weight"], sd[key + ".bias"])
            else:
                self._pack_resnet_block(P, sd, name, ci, co)
                self._pack_time_stack(P, sd, name + ".time_stack")
        self._pack_affine(P, sd, "norm_out")
        P["conv_out.weight"], P["conv_out.bias"] = self._pack_conv3x3(sd["conv_out.weight"], sd["conv_out.bias"])
        P["time_mix.weight"] = self._f32(sd["conv_out.time_mix_conv.weight"].reshape(self.out_ch, self.out_ch, 3))
        P["time_mix.bias"] = self._f32(sd["conv_out.time_mix_conv.bias"])
        return P

    # --------------------------------------------------------------------------------------------
    def _video_res_block(self, P, name, ci, co, x, B, T, nb, h, w):
        """temporal_ae.VideoResBlock.forward (temporal_ae.py:64-83): ResnetBlock (model.py:131-151), then
        alpha * time_stack(x) + (1 - alpha) * x  ==  x + alpha * conv_t(...)."""
        xs = self._resnet_block(P, name, ci, co, x, B, h, w)
        return self._time_stack(P, name + ".time_stack", xs, h * w, T, nb, co, s0=P[name + ".alpha"])

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
        with self._stats_pool(n_norms * B, dev):
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
