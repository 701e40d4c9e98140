"""fp32 CPU restatement of the first-stage decode used by V3D_512 (TEST INFRASTRUCTURE).

DiffusionEngine.decode_first_stage (sgm/models/video_diffusion.py:182-210) -> AutoencodingEngine.decode
(sgm/models/autoencoder.py:210-212) -> temporal_ae.VideoDecoder (= model.py Decoder.forward with
VideoResBlock / AE3DConv plugged in, time_mode "conv-only").
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Sequence, Tuple

import torch
import torch.nn.functional as F

from .ref_unet import res_block

SD = Dict[str, torch.Tensor]


@dataclass
class DecoderSpec:
    """decoder_config of scripts/pub/configs/V3D_512.yaml:111-132."""
    ch: int = 128
    out_ch: int = 3
    ch_mult: Sequence[int] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4


def _norm(x, sd: SD, p: str):
    """Normalize(): GroupNorm(32, C, eps=1e-6) (model.py:52-55)."""
    return F.group_norm(x, 32, sd[p + ".weight"], sd[p + ".bias"], 1e-6)


def _swish(x):
    return x * torch.sigmoid(x)  # nonlinearity(), model.py:47-49


def resnet_block(sd: SD, p: str, x):
    """ResnetBlock.forward with temb=None (model.py:131-151)."""
    h = F.conv2d(_swish(_norm(x, sd, p + ".norm1")), sd[p + ".conv1.weight"], sd[p + ".conv1.bias"], padding=1)
    h = F.conv2d(_swish(_norm(h, sd, p + ".norm2")), sd[p + ".conv2.weight"], sd[p + ".conv2.bias"], padding=1)
    if p + ".nin_shortcut.weight" in sd:
        x = F.conv2d(x, sd[p + ".nin_shortcut.weight"], sd[p + ".nin_shortcut.bias"])
    return x + h


def video_res_block(sd: SD, p: str, x, T: int):
    """temporal_ae.VideoResBlock.forward (temporal_ae.py:64-83): ResnetBlock, then time_stack (3-D ResBlock,
    skip_t_emb) and alpha = sigmoid(mix_factor) weighting the TEMPORAL branch (opposite of the UNet)."""
    x = resnet_block(sd, p, x)
    bt, c, h, w = x.shape
    x5 = x.reshape(bt // T, T, c, h, w).permute(0, 2, 1, 3, 4)
    xt = res_block(sd, p + ".time_stack", x5, None, dims=3, exchange_temb=False)
    alpha = torch.sigmoid(sd[p + ".mix_factor"])
    out = alpha * xt + (1.0 - alpha) * x5
    return out.permute(0, 2, 1, 3, 4).reshape(bt, c, h, w)


def attn_block(sd: SD, p: str, x):
    """AttnBlock (model.py:161-201): GN, 1x1 q/k/v, single-head SDPA over h*w with d = C, 1x1 proj, residual."""
    h_ = _norm(x, sd, p + ".norm")
    q = F.conv2d(h_, sd[p + ".q.weight"], sd[p + ".q.bias"])
    k = F.conv2d(h_, sd[p + ".k.weight"], sd[p + ".k.bias"])
    v = F.conv2d(h_, sd[p + ".v.weight"], sd[p + ".v.bias"])
    b, c, h, w = q.shape

    def flat(t):
        return t.reshape(b, c, h * w).permute(0, 2, 1)[:, None]  # "b c h w -> b 1 (h w) c"

    o = F.scaled_dot_product_attention(flat(q), flat(k), flat(v))
    o = o[:, 0].permute(0, 2, 1).reshape(b, c, h, w)
    return x + F.conv2d(o, sd[p + ".proj_out.weight"], sd[p + ".proj_out.bias"])


def upsample(sd: SD, p: str, x):
    """Upsample (model.py:60-71): nearest 2x, then the 3x3 conv `p`."""
    return F.conv2d(F.interpolate(x, scale_factor=2.0, mode="nearest"), sd[p + ".weight"], sd[p + ".bias"], padding=1)


def decoder_tail(sd: SD, h, T: int):
    """norm_out -> swish -> conv_out, then AE3DConv's time_mix_conv (temporal_ae.py:101-107): a (3, 1, 1) conv over
    each clip of T frames, zero-padded at the clip's two ends."""
    h = _swish(_norm(h, sd, "norm_out"))
    h = F.conv2d(h, sd["conv_out.weight"], sd["conv_out.bias"], padding=1)
    bt, c, hh, ww = h.shape
    h5 = h.reshape(bt // T, T, c, hh, ww).permute(0, 2, 1, 3, 4)
    h5 = F.conv3d(h5, sd["conv_out.time_mix_conv.weight"], sd["conv_out.time_mix_conv.bias"], padding=(1, 0, 0))
    return h5.permute(0, 2, 1, 3, 4).reshape(bt, c, hh, ww)


def decoder_forward(sd: SD, spec: DecoderSpec, z, T: int, taps=None):
    """Decoder.forward (model.py:715-748) with AE3DConv.forward at the end (temporal_ae.py:101-107)."""
    nres = len(spec.ch_mult)
    h = F.conv2d(z, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    h = video_res_block(sd, "mid.block_1", h, T)
    h = attn_block(sd, "mid.attn_1", h)
    h = video_res_block(sd, "mid.block_2", h, T)
    if taps is not None:
        taps["mid"] = h
    for lvl in reversed(range(nres)):
        for j in range(spec.num_res_blocks + 1):
            h = video_res_block(sd, f"up.{lvl}.block.{j}", h, T)
        if lvl != 0:
            h = upsample(sd, f"up.{lvl}.upsample.conv", h)
        if taps is not None:
            taps[f"up.{lvl}"] = h
    return decoder_tail(sd, h, T)


def decode_first_stage(sd: SD, spec: DecoderSpec, z, n_samples_a_time: int, scale_factor: float = 0.18215):
    """DiffusionEngine.decode_first_stage (video_diffusion.py:182-210): z/scale, chunks of n frames, each
    chunk decoded with timesteps=len(chunk) (temporal convs zero-pad at chunk edges)."""
    z = 1.0 / scale_factor * z
    outs = []
    for n in range(math.ceil(z.shape[0] / n_samples_a_time)):
        chunk = z[n * n_samples_a_time:(n + 1) * n_samples_a_time]
        outs.append(decoder_forward(sd, spec, chunk, T=len(chunk)))
    return torch.cat(outs, dim=0)


def decoder_param_shapes(spec: DecoderSpec) -> Dict[str, Tuple[int, ...]]:
    sh: Dict[str, Tuple[int, ...]] = {}

    def wb(p, w):
        sh[p + ".weight"] = tuple(w)
        sh[p + ".bias"] = (w[0],)

    def norm(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)

    def vres(p, cin, cout):
        norm(p + ".norm1", cin); wb(p + ".conv1", (cout, cin, 3, 3))
        norm(p + ".norm2", cout); wb(p + ".conv2", (cout, cout, 3, 3))
        if cin != cout:
            wb(p + ".nin_shortcut", (cout, cin, 1, 1))
        ts = p + ".time_stack"
        norm(ts + ".in_layers.0", cout); wb(ts + ".in_layers.2", (cout, cout, 3, 1, 1))
        norm(ts + ".out_layers.0", cout); wb(ts + ".out_layers.3", (cout, cout, 3, 1, 1))
        sh[p + ".mix_factor"] = (1,)

    nres = len(spec.ch_mult)
    block_in = spec.ch * spec.ch_mult[-1]
    wb("conv_in", (block_in, spec.z_channels, 3, 3))
    vres("mid.block_1", block_in, block_in)
    norm("mid.attn_1.norm", block_in)
    for n in ("q", "k", "v", "proj_out"):
        wb(f"mid.attn_1.{n}", (block_in, block_in, 1, 1))
    vres("mid.block_2", block_in, block_in)
    for lvl in reversed(range(nres)):
        block_out = spec.ch * spec.ch_mult[lvl]
        for j in range(spec.num_res_blocks + 1):
            vres(f"up.{lvl}.block.{j}", block_in, block_out)
            block_in = block_out
        if lvl != 0:
            wb(f"up.{lvl}.upsample.conv", (block_in, block_in, 3, 3))
    norm("norm_out", block_in)
    wb("conv_out", (spec.out_ch, block_in, 3, 3))
    wb("conv_out.time_mix_conv", (spec.out_ch, spec.out_ch, 3, 1, 1))
    return sh
