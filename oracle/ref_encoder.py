"""fp32 CPU restatement of the first-stage ENCODE front-end of V3D_512 (TEST INFRASTRUCTURE; SURVEY 8(f)-1).

scripts/pub/V3D_512.py:239 `ae_model.encode(image)` -> AutoencodingEngine.encode (sgm/models/autoencoder.py:196-208)
-> Encoder.forward (sgm/modules/diffusionmodules/model.py:576-601, config configs/ae/video.yaml) ->
DiagonalGaussianRegularizer / DiagonalGaussianDistribution.sample (regularizers/__init__.py:13-32,
distributions/distributions.py:24-41).  The Gaussian noise is an explicit argument here (the reference draws it with
torch.randn on the CPU generator).
"""
from __future__ import annotations

from dataclasses import dataclass
from typing import Dict, Sequence, Tuple

import torch
import torch.nn.functional as F

from .ref_decoder import _norm, _swish, attn_block, resnet_block

SD = Dict[str, torch.Tensor]


@dataclass
class EncoderSpec:
    """encoder_config of configs/ae/video.yaml:7-19 (attn_resolutions = [], so only mid.attn_1 attends)."""
    ch: int = 128
    in_channels: int = 3
    ch_mult: Sequence[int] = (1, 2, 4, 4)
    num_res_blocks: int = 2
    z_channels: int = 4
    double_z: bool = True


def downsample(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """Downsample (model.py:74-91): zero padding on the bottom / right only, then the stride-2 3x3 conv `p`."""
    return F.conv2d(F.pad(x, (0, 1, 0, 1), mode="constant", value=0), sd[p + ".weight"], sd[p + ".bias"], stride=2)


def encoder_tail(sd: SD, h: torch.Tensor) -> torch.Tensor:
    """norm_out -> swish -> conv_out: the moments [B, 2z, H/8, W/8]"""
    return F.conv2d(_swish(_norm(h, sd, "norm_out")), sd["conv_out.weight"], sd["conv_out.bias"], padding=1)


def encoder_forward(sd: SD, spec: EncoderSpec, x: torch.Tensor) -> torch.Tensor:
    """Encoder.forward with temb = None: conv_in, per level num_res_blocks ResnetBlocks (+ asymmetric-pad stride-2
    conv between levels, model.py:74-91), mid block/attn/block, GroupNorm + swish + conv_out -> [B, 2z, H/8, W/8]."""
    nres = len(spec.ch_mult)
    h = F.conv2d(x, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    for lvl in range(nres):
        for blk in range(spec.num_res_blocks):
            h = resnet_block(sd, f"down.{lvl}.block.{blk}", h)
        if lvl != nres - 1:
            h = downsample(sd, f"down.{lvl}.downsample.conv", h)
    h = resnet_block(sd, "mid.block_1", h)
    h = attn_block(sd, "mid.attn_1", h)
    h = resnet_block(sd, "mid.block_2", h)
    return encoder_tail(sd, h)


def gaussian_sample(moments: torch.Tensor, noise: torch.Tensor) -> torch.Tensor:
    """DiagonalGaussianDistribution(moments).sample() with the normal draw passed in (distributions.py:24-41)."""
    mean, logvar = torch.chunk(moments, 2, dim=1)
    logvar = torch.clamp(logvar, -30.0, 20.0)
    return mean + torch.exp(0.5 * logvar) * noise


def gaussian_mode(moments: torch.Tensor) -> torch.Tensor:
    return torch.chunk(moments, 2, dim=1)[0]


def encoder_param_shapes(spec: EncoderSpec) -> Dict[str, Tuple[int, ...]]:
    sh: Dict[str, Tuple[int, ...]] = {}

    def conv(p, co, ci, k):
        sh[p + ".weight"] = (co, ci, k, k)
        sh[p + ".bias"] = (co,)

    def norm(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)

    def resnet(p, ci, co):
        norm(p + ".norm1", ci)
        conv(p + ".conv1", co, ci, 3)
        norm(p + ".norm2", co)
        conv(p + ".conv2", co, co, 3)
        if ci != co:
            conv(p + ".nin_shortcut", co, ci, 1)

    conv("conv_in", spec.ch, spec.in_channels, 3)
    in_mult = (1,) + tuple(spec.ch_mult)
    nres = len(spec.ch_mult)
    block_in = spec.ch
    for lvl in range(nres):
        block_in = spec.ch * in_mult[lvl]
        block_out = spec.ch * spec.ch_mult[lvl]
        for blk in range(spec.num_res_blocks):
            resnet(f"down.{lvl}.block.{blk}", block_in, block_out)
            block_in = block_out
        if lvl != nres - 1:
            conv(f"down.{lvl}.downsample.conv", block_in, block_in, 3)
    resnet("mid.block_1", block_in, block_in)
    norm("mid.attn_1.norm", block_in)
    for n in ("q", "k", "v", "proj_out"):
        conv(f"mid.attn_1.{n}", block_in, block_in, 1)
    resnet("mid.block_2", block_in, block_in)
    norm("norm_out", block_in)
    conv("conv_out", (2 if spec.double_z else 1) * spec.z_channels, block_in, 3)
    return sh
