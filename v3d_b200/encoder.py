"""H100-native first-stage ENCODE front-end (SURVEY.md 8(f) rank 1): drop-in for
`sgm.modules.diffusionmodules.model.Encoder` (model.py:463-601, config configs/ae/video.yaml) and the Gaussian
posterior of `DiagonalGaussianRegularizer` (regularizers/__init__.py:13-32, distributions.py:24-41).

It runs once per image (`ae_model.encode(image)`, scripts/pub/V3D_512.py:239; 1.12 TF) on the kernels of the decode
path: implicit-GEMM 3x3 convs, GroupNorm(+SiLU), the single-head mid attention, and an explicit im2row for the
stride-2 convs whose zero padding is bottom/right only (model.py:74-91).  Same constructor kwargs and `state_dict()`
keys as the reference encoder; forward takes NCHW fp32 images in [-1, 1] and returns the NCHW fp32 moments
[B, 2*z, H/8, W/8].

Oracle restatement pinned against the real reference, golden fixtures under tests/golden/encoder_*; the device path is
checked against them in tests/test_parity_gpu.py::test_encoder_matches_reference.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Sequence, Tuple

import torch

from . import ops
from .first_stage import FirstStage
from .kernel_module import _register


class Encoder(FirstStage):
    def __init__(
        self,
        *,
        ch: int,
        out_ch: int = 3,
        ch_mult: Sequence[int] = (1, 2, 4, 8),
        num_res_blocks: int,
        attn_resolutions: Sequence[int],
        dropout: float = 0.0,
        resamp_with_conv: bool = True,
        in_channels: int,
        resolution: int,
        z_channels: int,
        double_z: bool = True,
        use_linear_attn: bool = False,
        attn_type: str = "vanilla",
        **ignore_kwargs,
    ):
        super().__init__()
        bad = []
        if list(attn_resolutions):
            bad.append("attn_resolutions != []")
        if use_linear_attn or not resamp_with_conv or dropout != 0.0:
            bad.append("use_linear_attn / resamp_with_conv=False / dropout")
        if attn_type not in ("vanilla", "vanilla-xformers"):
            bad.append(f"attn_type={attn_type}")
        if ch % 64 or (2 if double_z else 1) * z_channels > 16:
            bad.append("ch % 64 != 0 or more than 16 output channels")
        if bad:
            raise NotImplementedError("v3d_b200.Encoder covers the configs/ae/video.yaml encoder; unsupported: "
                                      + ", ".join(bad))
        self.ch, self.ch_mult, self.num_res_blocks = ch, list(ch_mult), num_res_blocks
        self.in_channels, self.z_channels, self.double_z = in_channels, z_channels, double_z
        self.resolution = resolution
        self.num_resolutions = len(self.ch_mult)
        self.out_channels = (2 if double_z else 1) * z_channels
        self.debug_taps: Optional[dict] = None  # tests: {block name: None} -> filled with NCHW fp32 outputs
        for key, shape in self.param_shapes().items():
            _register(self, key, self._init_value(key, shape))

    # --------------------------------------------------------------------------------------------
    def _blocks(self) -> List[Tuple[str, int, int]]:
        """(name, cin, cout) in execution order; '@down:' = stride-2 conv, '@attn:' = mid attention."""
        out: List[Tuple[str, int, int]] = []
        in_mult = (1,) + tuple(self.ch_mult)
        block_in = self.ch
        for lvl in range(self.num_resolutions):
            block_in = self.ch * in_mult[lvl]
            block_out = self.ch * self.ch_mult[lvl]
            for j in range(self.num_res_blocks):
                out.append((f"down.{lvl}.block.{j}", block_in, block_out))
                block_in = block_out
            if lvl != self.num_resolutions - 1:
                out.append((f"@down:down.{lvl}.downsample.conv", block_in, block_in))
        out.append(("mid.block_1", block_in, block_in))
        out.append(("@attn:mid.attn_1", block_in, block_in))
        out.append(("mid.block_2", block_in, block_in))
        return out

    def param_shapes(self) -> Dict[str, Tuple[int, ...]]:
        table: Dict[str, Tuple[int, ...]] = {}
        conv = self._conv_shape
        conv(table, "conv_in", self.ch, self.in_channels, 3, 3)
        last = self.ch
        for name, ci, co in self._blocks():
            if name.startswith("@attn:"):
                self._attn_block_shapes(table, name[6:], ci)
            elif name.startswith("@down:"):
                conv(table, name[6:], co, ci, 3, 3)
            else:
                self._resnet_block_shapes(table, name, ci, co)
            last = co
        self._affine_shape(table, "norm_out", last)
        conv(table, "conv_out", self.out_channels, last, 3, 3)
        return table

    # --------------------------------------------------------------------------------------------
    def _pack(self, dev: torch.device) -> dict:
        sd = {k: v.detach() for k, v in self.named_parameters()}
        P: dict = {}
        kpad = (9 * self.in_channels + 63) // 64 * 64
        P["conv_in.weight"], P["conv_in.bias"] = self._pack_conv3x3(sd["conv_in.weight"], sd["conv_in.bias"], kpad)
        for name, ci, co in self._blocks():
            if name.startswith("@attn:"):
                self._pack_attn_block(P, sd, name[6:], ci)
            elif name.startswith("@down:"):
                key = name[6:]
                P[key + ".weight"], P[key + ".bias"] = self._pack_conv3x3(sd[key + ".weight"], sd[key + ".bias"])
            else:
                self._pack_resnet_block(P, sd, name, ci, co)
        self._pack_affine(P, sd, "norm_out")
        P["conv_out.weight"], P["conv_out.bias"] = self._pack_conv3x3(sd["conv_out.weight"], sd["conv_out.bias"])
        return P

    # --------------------------------------------------------------------------------------------
    def _downsample(self, P, key, x, B, h, w, c):
        """Downsample (model.py:74-91): F.pad (0,1,0,1) then Conv2d(k=3, stride=2, padding=0): the zero padding is
        bottom/right only, so the im2row runs with pad 0 and output size h/2 x w/2."""
        if h % 2 or w % 2:
            raise NotImplementedError("encoder downsample needs even h, w")
        ho, wo = h // 2, w // 2
        wt, bias = P[key + ".weight"], P[key + ".bias"]
        kpad = wt.shape[1]
        col = torch.empty(B * ho * wo, kpad, device=x.device, dtype=torch.bfloat16)
        ops.im2col3x3(x, col, B, h, w, c, 2, 0, ho, wo, kpad)
        out = torch.empty(B * ho * wo, wt.shape[0], device=x.device, dtype=torch.bfloat16)
        ops.gemm(col, wt, out, K=kpad, N=wt.shape[0], rows_per_batch=B * ho * wo, bias=bias)
        return out, ho, wo

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        ops.require_current_device(x, "v3d_b200.Encoder.forward")
        assert x.shape[1] == self.in_channels
        with torch.no_grad():
            return self._run(self.packed(), x)

    def _run(self, P: dict, x: torch.Tensor) -> torch.Tensor:
        """The launch schedule of one encode (Encoder.forward, model.py:576-601)."""
        B, cin, H, W = x.shape
        dev = x.device
        n_norms = 2 * sum(1 for n, _, _ in self._blocks() if not n.startswith("@")) + 2
        with self._stats_pool(n_norms * B, dev):
            cur = torch.empty(B * H * W, cin, device=dev, dtype=torch.bfloat16)
            ops.nchw_f32_to_nhwc_bf16(x.float().contiguous(), cur)
            h, w = H, W
            cur = self._conv3x3(P, "conv_in", cur, B, h, w, cin)
            ch = self.ch
            self._tap("conv_in", cur, B, ch, h, w)
            for name, ci, co in self._blocks():
                if name.startswith("@attn:"):
                    if (h * w) % 64 != 0 or ci % 64 != 0:
                        raise NotImplementedError("encoder AttnBlock needs h*w % 64 == 0")
                    cur = self._attn(P, name[6:], ci, cur, B, h, w)
                elif name.startswith("@down:"):
                    cur, h, w = self._downsample(P, name[6:], cur, B, h, w, ci)
                else:
                    cur = self._resnet_block(P, name, ci, co, cur, B, h, w)
                    ch = co
                self._tap(name.rsplit(":", 1)[-1], cur, B, ch, h, w)
            a = self._gn(P, "norm_out", cur, h * w, B, ch, 1e-6, True)
            o = self._conv3x3(P, "conv_out", a, B, h, w, ch, out_dtype=torch.float32)   # [rows, 16] fp32
            out = torch.empty(B, self.out_channels, h, w, device=dev, dtype=torch.float32)
            ops.nhwc_to_nchw_f32(o, out, B, self.out_channels, h * w, ldx=o.shape[1])
        return out


class DiagonalGaussianRegularizer(torch.nn.Module):
    """`DiagonalGaussianDistribution(moments).sample()` / `.mode()` (regularizers/__init__.py:13-32,
    distributions.py:24-41).  The normal draw is made with torch.randn on the CPU generator and moved to the device,
    exactly as the reference does (so a seeded run reproduces its latents); a caller-supplied `noise` overrides it."""

    def __init__(self, sample: bool = True):
        super().__init__()
        self.sample = sample

    def forward(self, z: torch.Tensor, noise: Optional[torch.Tensor] = None):
        mean, logvar = torch.chunk(z, 2, dim=1)
        logvar = torch.clamp(logvar, -30.0, 20.0)
        if not self.sample:
            return mean, {}
        if noise is None:
            noise = torch.randn(mean.shape).to(device=z.device)
        return mean + torch.exp(0.5 * logvar) * noise.to(z.device), {}
