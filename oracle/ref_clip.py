"""fp32 CPU restatement of the CLIP ViT-H/14 IMAGE TOWER the conditioner runs once per image (TEST INFRASTRUCTURE;
SURVEY 8(f)-4).

Call site: scripts/pub/V3D_512.py:146-153,238 `clip_model(image)` -> FrozenOpenCLIPImagePredictionEmbedder.forward
(sgm/modules/encoders/modules.py:1054-1072) -> FrozenOpenCLIPImageEmbedder.forward / encode_with_vision_transformer
(:594-752): preprocess (:645-657: kornia bicubic antialiased resize to 224 x 224, (x + 1) / 2, CLIP mean / std) ->
`self.model.visual(img)` -> [B, 1024] -> "(b t) d -> b t d".

The tower itself lives in a THIRD-PARTY dependency that is absent here: open_clip (`open_clip.create_model_and_transforms
("ViT-H-14", pretrained="laion2b_s32b_b79k")`, requirements pin open_clip_torch 2.x) and the resize in kornia
(`kornia.geometry.resize`).  Their published algorithms are restated below:
  * open_clip.transformer.VisionTransformer.forward: conv1 (14 x 14 patches, no bias) -> [class_embedding; patches] +
    positional_embedding -> ln_pre -> 32 pre-LN ResidualAttentionBlocks (nn.MultiheadAttention with a packed in_proj,
    16 heads of width 80; MLP 1280 -> 5120 -> 1280 with exact-erf GELU) -> ln_post on the class token -> @ proj;
  * kornia.geometry.transform.resize(antialias=True): Gaussian blur with sigma = (factor - 1) / 2 per axis, kernel size
    max(int(4 sigma), 3) made odd, reflect border, then F.interpolate(bicubic, align_corners=True).
PARITY PIN: open_clip / kornia cannot be imported offline, so this file is pinned against an INDEPENDENT implementation of
the same architecture that is present - Hugging Face transformers' CLIPVisionModelWithProjection with the state dict
mapped name by name (tests/test_oracle_cpu.py::test_clip_tower_oracle_matches_hf_transformers, error ~1e-6) - and the
preprocess against its closed-form pieces; parity on the real laion2b checkpoint is unpinned (weights unavailable).
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Dict, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)   # encoders/modules.py:634-639
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


@dataclass
class ClipSpec:
    """open_clip model config "ViT-H-14" (vision_cfg: image_size 224, layers 32, width 1280, head_width 80, patch 14;
    embed_dim 1024, mlp_ratio 4)."""
    image_size: int = 224
    patch: int = 14
    width: int = 1280
    layers: int = 32
    heads: int = 16
    mlp: int = 5120
    embed_dim: int = 1024


def clip_visual_param_shapes(spec: ClipSpec) -> Dict[str, Tuple[int, ...]]:
    """state_dict of open_clip's VisionTransformer (keys below `model.visual.` in the reference checkpoint)"""
    w, n = spec.width, (spec.image_size // spec.patch) ** 2 + 1
    out = {"class_embedding": (w,), "positional_embedding": (n, w), "proj": (w, spec.embed_dim),
           "conv1.weight": (w, 3, spec.patch, spec.patch), "ln_pre.weight": (w,), "ln_pre.bias": (w,),
           "ln_post.weight": (w,), "ln_post.bias": (w,)}
    for i in range(spec.layers):
        p = f"transformer.resblocks.{i}."
        out.update({p + "ln_1.weight": (w,), p + "ln_1.bias": (w,), p + "attn.in_proj_weight": (3 * w, w),
                    p + "attn.in_proj_bias": (3 * w,), p + "attn.out_proj.weight": (w, w),
                    p + "attn.out_proj.bias": (w,), p + "ln_2.weight": (w,), p + "ln_2.bias": (w,),
                    p + "mlp.c_fc.weight": (spec.mlp, w), p + "mlp.c_fc.bias": (spec.mlp,),
                    p + "mlp.c_proj.weight": (w, spec.mlp), p + "mlp.c_proj.bias": (w,)})
    return out


def gaussian_kernel1d(ks: int, sigma: float) -> torch.Tensor:
    x = torch.arange(ks, dtype=torch.float32) - ks // 2
    if ks % 2 == 0:
        x = x + 0.5
    g = torch.exp(-x.pow(2.0) / (2 * sigma ** 2))
    return g / g.sum()


def resize_antialias_bicubic(x: torch.Tensor, size: Tuple[int, int]) -> torch.Tensor:
    """kornia.geometry.transform.resize(x, size, interpolation="bicubic", align_corners=True, antialias=True)"""
    h, w = x.shape[-2:]
    fy, fx = h / size[0], w / size[1]
    if max(fy, fx) > 1.0:
        sig = (max((fy - 1.0) / 2.0, 0.001), max((fx - 1.0) / 2.0, 0.001))
        ks = [int(max(2.0 * 2 * s, 3)) for s in sig]
        ks = [k + 1 if k % 2 == 0 else k for k in ks]
        ky, kx = gaussian_kernel1d(ks[0], sig[0]).to(x), gaussian_kernel1d(ks[1], sig[1]).to(x)
        c = x.shape[1]
        xp = F.pad(x, (ks[1] // 2, ks[1] // 2, ks[0] // 2, ks[0] // 2), mode="reflect")
        xp = F.conv2d(xp, kx.view(1, 1, 1, -1).repeat(c, 1, 1, 1), groups=c)
        x = F.conv2d(xp, ky.view(1, 1, -1, 1).repeat(c, 1, 1, 1), groups=c)
    return F.interpolate(x, size=size, mode="bicubic", align_corners=True)


def preprocess(x: torch.Tensor, size: int = 224) -> torch.Tensor:
    """FrozenOpenCLIPImageEmbedder.preprocess (encoders/modules.py:645-657): x in [-1, 1]"""
    x = resize_antialias_bicubic(x, (size, size))
    x = (x + 1.0) / 2.0
    mean = torch.tensor(CLIP_MEAN).to(x).view(1, 3, 1, 1)
    std = torch.tensor(CLIP_STD).to(x).view(1, 3, 1, 1)
    return (x - mean) / std


def clip_embed(sd: SD, spec: ClipSpec, img: torch.Tensor) -> torch.Tensor:
    """conv1 patches, [class_embedding; patches] + positional_embedding, ln_pre -> residual stream [B, n, width]"""
    B, w = img.shape[0], spec.width
    x = F.conv2d(img, sd["conv1.weight"], None, stride=spec.patch)            # [B, w, g, g]
    x = x.reshape(B, w, -1).permute(0, 2, 1)                                  # [B, g*g, w]
    x = torch.cat([sd["class_embedding"].to(x).expand(B, 1, w), x], dim=1) + sd["positional_embedding"]
    return F.layer_norm(x, (w,), sd["ln_pre.weight"], sd["ln_pre.bias"], 1e-5)


def clip_attn_half(sd: SD, spec: ClipSpec, i: int, x: torch.Tensor) -> torch.Tensor:
    """x + out_proj(MHA(ln_1(x))) of residual block i (16 heads of width 80 at ViT-H/14)"""
    B, n, w = x.shape
    hd = w // spec.heads
    p = f"transformer.resblocks.{i}."
    h = F.layer_norm(x, (w,), sd[p + "ln_1.weight"], sd[p + "ln_1.bias"], 1e-5)
    qkv = F.linear(h, sd[p + "attn.in_proj_weight"], sd[p + "attn.in_proj_bias"])
    q, k, v = [t.reshape(B, n, spec.heads, hd).permute(0, 2, 1, 3) for t in qkv.chunk(3, dim=-1)]
    att = torch.softmax(q @ k.transpose(-1, -2) / math.sqrt(hd), dim=-1) @ v
    att = att.permute(0, 2, 1, 3).reshape(B, n, w)
    return x + F.linear(att, sd[p + "attn.out_proj.weight"], sd[p + "attn.out_proj.bias"])


def clip_mlp_half(sd: SD, spec: ClipSpec, i: int, x: torch.Tensor) -> torch.Tensor:
    """x + c_proj(gelu_erf(c_fc(ln_2(x)))) of residual block i"""
    p = f"transformer.resblocks.{i}."
    h = F.layer_norm(x, (spec.width,), sd[p + "ln_2.weight"], sd[p + "ln_2.bias"], 1e-5)
    h = F.gelu(F.linear(h, sd[p + "mlp.c_fc.weight"], sd[p + "mlp.c_fc.bias"]))
    return x + F.linear(h, sd[p + "mlp.c_proj.weight"], sd[p + "mlp.c_proj.bias"])


def clip_head(sd: SD, spec: ClipSpec, x: torch.Tensor) -> torch.Tensor:
    """ln_post on the class token, @ proj -> pooled embedding [B, embed_dim]"""
    pooled = F.layer_norm(x[:, 0], (spec.width,), sd["ln_post.weight"], sd["ln_post.bias"], 1e-5)
    return pooled @ sd["proj"]


def clip_visual_forward(sd: SD, spec: ClipSpec, img: torch.Tensor) -> torch.Tensor:
    """open_clip VisionTransformer.forward on preprocessed images [B, 3, 224, 224] -> pooled embedding [B, embed_dim]"""
    x = clip_embed(sd, spec, img)
    for i in range(spec.layers):
        x = clip_mlp_half(sd, spec, i, clip_attn_half(sd, spec, i, x))
    return clip_head(sd, spec, x)


def image_embedder_forward(sd: SD, spec: ClipSpec, image: torch.Tensor, n_cond_frames: int = 1,
                           n_copies: int = 1) -> torch.Tensor:
    """FrozenOpenCLIPImagePredictionEmbedder.forward (encoders/modules.py:1066-1072) around the embedder's forward with
    ucg_rate = 0, unsqueeze_dim / repeat_to_max_len / output_tokens off (configs/embedder/clip_image.yaml):
    image [B*t, 3, H, W] in [-1, 1] -> [(B*copies), t, embed_dim]."""
    z = clip_visual_forward(sd, spec, preprocess(image, spec.image_size))
    z = z.reshape(-1, n_cond_frames, z.shape[-1])
    return z.repeat_interleave(n_copies, dim=0)


def to_hf_state_dict(sd: SD, spec: ClipSpec) -> SD:
    """the same weights under Hugging Face transformers' CLIPVisionModelWithProjection names (pinning only)"""
    w = spec.width
    out = {"vision_model.embeddings.class_embedding": sd["class_embedding"],
           "vision_model.embeddings.patch_embedding.weight": sd["conv1.weight"],
           "vision_model.embeddings.position_embedding.weight": sd["positional_embedding"],
           "vision_model.pre_layrnorm.weight": sd["ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["ln_pre.bias"],
           "vision_model.post_layernorm.weight": sd["ln_post.weight"],
           "vision_model.post_layernorm.bias": sd["ln_post.bias"],
           "visual_projection.weight": sd["proj"].t().contiguous()}
    for i in range(spec.layers):
        p, h = f"transformer.resblocks.{i}.", f"vision_model.encoder.layers.{i}."
        wq, wk, wv = sd[p + "attn.in_proj_weight"].chunk(3, dim=0)
        bq, bk, bv = sd[p + "attn.in_proj_bias"].chunk(3, dim=0)
        out.update({h + "self_attn.q_proj.weight": wq, h + "self_attn.k_proj.weight": wk, h + "self_attn.v_proj.weight": wv,
                    h + "self_attn.q_proj.bias": bq, h + "self_attn.k_proj.bias": bk, h + "self_attn.v_proj.bias": bv,
                    h + "self_attn.out_proj.weight": sd[p + "attn.out_proj.weight"],
                    h + "self_attn.out_proj.bias": sd[p + "attn.out_proj.bias"],
                    h + "layer_norm1.weight": sd[p + "ln_1.weight"], h + "layer_norm1.bias": sd[p + "ln_1.bias"],
                    h + "layer_norm2.weight": sd[p + "ln_2.weight"], h + "layer_norm2.bias": sd[p + "ln_2.bias"],
                    h + "mlp.fc1.weight": sd[p + "mlp.c_fc.weight"], h + "mlp.fc1.bias": sd[p + "mlp.c_fc.bias"],
                    h + "mlp.fc2.weight": sd[p + "mlp.c_proj.weight"], h + "mlp.fc2.bias": sd[p + "mlp.c_proj.bias"]})
    return out
