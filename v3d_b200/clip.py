"""CLIP ViT-H/14 image tower of the conditioner on the path's own kernels (SURVEY.md 8(f)-4).

Drop-ins for `sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder` (encoders/modules.py:594-752) and
`FrozenOpenCLIPImagePredictionEmbedder` (:1054-1072), the `clip_model` of scripts/pub/V3D_512.py:146-153,238 that turns
the conditioning image into the single cross-attention token of the denoiser.  The reference builds the tower with
open_clip (`create_model_and_transforms("ViT-H-14")`, deletes the text transformer, keeps the text-side embedding
tensors); the state_dict here has the same keys - `model.visual.*` (the ViT) and the leftover text-side tensors
`model.{positional_embedding, text_projection, logit_scale, token_embedding.weight, ln_final.*}`, which are loaded and
never used - so `clip_model.load_state_dict(clip_sd)` of V3D_512.py:148-152 works unchanged.

Runs once per image, so the schedule favours reuse over speed: every contraction is the wgmma GEMM of the denoiser
(`v3d_gemm_bf16`), LayerNorm and softmax are the path's kernels, and torch is used for layout glue only (patch
unfolding, the class token / positional add, head-major repacking, the bicubic resize of the preprocessing):
  * conv1 (14 x 14 stride-14 patches, no bias) = unfold + GEMM with K = 588 zero-padded to 640;
  * attention with head width 80: per (image, head) S = Q K^T as ONE batched GEMM with the contraction zero-padded to
    128 and the keys to 320 (pad columns forced to -inf before the softmax), fp32 scores -> v3d_softmax_rows_f32 ->
    P V as a second batched GEMM against V^T - the decoder AttnBlock's recipe;
  * the MLP's exact-erf GELU rides on the GEGLU epilogue: the "value" half of the packed projection has zero weights
    and bias 1, so the epilogue computes 1 * gelu(c_fc(x)).
bf16 operands, fp32 accumulation / statistics; against the fp32 oracle (oracle/ref_clip.py, pinned to Hugging Face
transformers' CLIP): rel-L2 <= 3e-2 of the pooled embedding (tests/test_parity_gpu.py::test_clip_tower_matches_oracle).
No CPU fallback: forward() raises on non-CUDA tensors.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .sampling import instantiate_from_config
from .kernel_module import KernelModule

CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
CLIP_STD = (0.26862954, 0.26130258, 0.27577711)


class _VisualTower(nn.Module):
    """Parameters of open_clip's VisionTransformer under its names; the compute lives in the embedder's schedule."""

    def __init__(self, image_size=224, patch=14, width=1280, layers=32, heads=16, mlp=5120, embed_dim=1024):
        super().__init__()
        self.image_size, self.patch, self.width, self.layers, self.heads, self.mlp, self.embed_dim = \
            image_size, patch, width, layers, heads, mlp, embed_dim
        n = (image_size // patch) ** 2 + 1
        P = lambda *s: nn.Parameter(torch.zeros(*s), requires_grad=False)  # noqa: E731
        self.class_embedding = P(width)
        self.positional_embedding = P(n, width)
        self.proj = P(width, embed_dim)
        self.conv1 = nn.Conv2d(3, width, patch, patch, bias=False)
        self.ln_pre, self.ln_post = nn.LayerNorm(width), nn.LayerNorm(width)
        self.transformer = nn.Module()
        self.transformer.resblocks = nn.ModuleList()
        for _ in range(layers):
            blk = nn.Module()
            blk.ln_1, blk.ln_2 = nn.LayerNorm(width), nn.LayerNorm(width)
            blk.attn = nn.Module()
            blk.attn.in_proj_weight, blk.attn.in_proj_bias = P(3 * width, width), P(3 * width)
            blk.attn.out_proj = nn.Linear(width, width)
            blk.mlp = nn.Module()
            blk.mlp.c_fc, blk.mlp.c_proj = nn.Linear(width, mlp), nn.Linear(mlp, width)
            self.transformer.resblocks.append(blk)
        for p in self.parameters():
            p.requires_grad_(False)


class _OpenClipShell(nn.Module):
    """What is left of open_clip's CLIP model after `del model.transformer` (encoders/modules.py:620): the visual tower
    plus the text-side embedding tensors, kept so that the reference checkpoint loads with strict=True."""

    def __init__(self, text_width=1024, vocab=49408, context=77, **vision):
        super().__init__()
        self.visual = _VisualTower(**vision)
        self.positional_embedding = nn.Parameter(torch.zeros(context, text_width), requires_grad=False)
        self.text_projection = nn.Parameter(torch.zeros(text_width, vision.get("embed_dim", 1024)), requires_grad=False)
        self.logit_scale = nn.Parameter(torch.zeros(()), requires_grad=False)
        self.token_embedding = nn.Embedding(vocab, text_width)
        self.ln_final = nn.LayerNorm(text_width)
        for p in self.parameters():
            p.requires_grad_(False)


class FrozenOpenCLIPImageEmbedder(KernelModule):
    """encoders/modules.py:594-752 for the configuration V3D uses (configs/embedder/clip_image.yaml: freeze, every
    other option at its default).  Options that change the output structure raise at construction."""

    def __init__(self, arch="ViT-H-14", version="laion2b_s32b_b79k", device="cuda", max_length=77, freeze=True,
                 antialias=True, ucg_rate=0.0, unsqueeze_dim=False, repeat_to_max_len=False, num_image_crops=0,
                 output_tokens=False, init_device=None, vision_cfg: Optional[Dict] = None):
        super().__init__()
        if arch != "ViT-H-14" and vision_cfg is None:
            raise NotImplementedError(f"only the ViT-H-14 image tower is built natively (got {arch!r})")
        if num_image_crops or output_tokens or repeat_to_max_len:
            raise NotImplementedError("num_image_crops / output_tokens / repeat_to_max_len are not used by V3D")
        self.model = _OpenClipShell(**(vision_cfg or {}))
        self.antialias, self.ucg_rate, self.unsqueeze_dim, self.max_length = antialias, ucg_rate, unsqueeze_dim, max_length
        self.register_buffer("mean", torch.tensor(CLIP_MEAN), persistent=False)
        self.register_buffer("std", torch.tensor(CLIP_STD), persistent=False)
        # tests: {name: None} -> filled with the fp32 residual stream [B, n, width] after ln_pre ("pre") and after the
        # attention / MLP half of layer i ("L{i}.attn", "L{i}.mlp")
        self.debug_taps: Optional[dict] = None

    def freeze(self):
        self.eval()
        return self

    # ---- preprocessing (encoders/modules.py:645-657; kornia.geometry.resize restated, see oracle/ref_clip.py) -------
    def preprocess(self, x: torch.Tensor) -> torch.Tensor:
        size = self.model.visual.image_size
        x = x.float()
        h, w = x.shape[-2:]
        fy, fx = h / size, w / size
        if self.antialias and max(fy, fx) > 1.0:
            c = x.shape[1]
            for dim, f in ((2, fy), (3, fx)):
                sig = max((f - 1.0) / 2.0, 0.001)
                ks = int(max(4.0 * sig, 3))
                ks += 1 - ks % 2
                g = torch.arange(ks, device=x.device, dtype=torch.float32) - ks // 2
                g = torch.exp(-g.pow(2.0) / (2 * sig * sig))
                g = (g / g.sum()).view(1, 1, -1, 1) if dim == 2 else (g / g.sum()).view(1, 1, 1, -1)
                pad = (0, 0, ks // 2, ks // 2) if dim == 2 else (ks // 2, ks // 2, 0, 0)
                x = F.conv2d(F.pad(x, pad, mode="reflect"), g.repeat(c, 1, 1, 1), groups=c)
        x = F.interpolate(x, size=(size, size), mode="bicubic", align_corners=True)
        x = (x + 1.0) / 2.0
        return (x - self.mean.view(1, 3, 1, 1)) / self.std.view(1, 3, 1, 1)

    # ---- weights: bf16 operands packed once (KernelModule.packed) -------------------------------------------------
    def _pack(self, dev: torch.device) -> dict:
        v, bf, f32 = self.model.visual, self._bf, self._f32
        kp = v.patch * v.patch * 3
        kpad = (kp + 63) // 64 * 64
        w1 = torch.zeros(v.width, kpad, device=dev)
        w1[:, :kp] = v.conv1.weight.detach().reshape(v.width, kp)       # (c, ky, kx) order = F.unfold's
        P = {"conv1": bf(w1), "kpad": kpad, "kp": kp, "cls": f32(v.class_embedding), "pos": f32(v.positional_embedding),
             "ln_pre": (f32(v.ln_pre.weight), f32(v.ln_pre.bias)), "ln_post": (f32(v.ln_post.weight), f32(v.ln_post.bias)),
             "proj_t": bf(v.proj.detach().t()), "blocks": []}
        bn = ops.pick_block_n(2 * v.mlp, ops.ACT_GEGLU)
        perm = ops.geglu_perm(v.mlp, bn).to(dev)
        for blk in v.transformer.resblocks:
            fc_w = torch.cat([torch.zeros_like(blk.mlp.c_fc.weight), blk.mlp.c_fc.weight.detach()], 0)[perm]
            fc_b = torch.cat([torch.ones_like(blk.mlp.c_fc.bias), blk.mlp.c_fc.bias.detach()], 0)[perm]
            P["blocks"].append({
                "ln1": (f32(blk.ln_1.weight), f32(blk.ln_1.bias)), "ln2": (f32(blk.ln_2.weight), f32(blk.ln_2.bias)),
                "qkv_w": bf(blk.attn.in_proj_weight), "qkv_b": f32(blk.attn.in_proj_bias),
                "out_w": bf(blk.attn.out_proj.weight), "out_b": f32(blk.attn.out_proj.bias),
                "fc_w": bf(fc_w), "fc_b": f32(fc_b),
                "proj_w": bf(blk.mlp.c_proj.weight), "proj_b": f32(blk.mlp.c_proj.bias)})
        return P

    # ---- the tower ---------------------------------------------------------------------------------------------------
    def _tap(self, name: str, x: torch.Tensor, B: int, n: int) -> None:
        if self.debug_taps is not None and name in self.debug_taps:
            self.debug_taps[name] = x.view(B, n, -1).float()     # exactly what the next half reads

    @torch.no_grad()
    def encode_with_vision_transformer(self, img: torch.Tensor) -> torch.Tensor:
        ops.require_current_device(img, "v3d_b200.FrozenOpenCLIPImageEmbedder")
        v, P = self.model.visual, self.packed()
        dev = img.device
        x = self.preprocess(img)
        B = x.shape[0]
        w, heads, hd = v.width, v.heads, v.width // v.heads
        g = v.image_size // v.patch
        n = g * g + 1
        rows = B * n
        bf16 = torch.bfloat16
        # conv1 as unfold + GEMM
        cols = F.unfold(x, v.patch, stride=v.patch).transpose(1, 2).reshape(B * g * g, P["kp"])
        a = torch.zeros(B * g * g, P["kpad"], device=dev, dtype=bf16)
        a[:, :P["kp"]] = cols
        pt = torch.empty(B * g * g, w, device=dev, dtype=bf16)
        ops.gemm(a, P["conv1"], pt, K=P["kpad"], N=w, rows_per_batch=B * g * g)
        tok = torch.cat([P["cls"].expand(B, 1, w), pt.float().view(B, g * g, w)], 1) + P["pos"]
        xa = tok.reshape(rows, w).to(bf16).contiguous()
        xb = torch.empty_like(xa)
        ops.layernorm(xa, xb, *P["ln_pre"], rows, w)
        x_res = xb                                                           # residual stream, bf16 [rows, w]
        self._tap("pre", x_res, B, n)
        hp = (hd + 63) // 64 * 64                                            # head width padded for the contraction
        nk = (n + 63) // 64 * 64                                             # keys padded for the P V contraction
        h_ln = torch.empty_like(x_res)
        qkv = torch.empty(rows, 3 * w, device=dev, dtype=bf16)
        for i, blk in enumerate(P["blocks"]):
            ops.layernorm(x_res, h_ln, *blk["ln1"], rows, w)
            ops.gemm(h_ln, blk["qkv_w"], qkv, K=w, N=3 * w, rows_per_batch=rows, bias=blk["qkv_b"])
            q, k, val = [t.reshape(B, n, heads, hd).permute(0, 2, 1, 3) for t in qkv.view(B, n, 3 * w).split(w, dim=-1)]
            qp = torch.zeros(B * heads, n, hp, device=dev, dtype=bf16)
            kpd = torch.zeros(B * heads, nk, hp, device=dev, dtype=bf16)
            vt = torch.zeros(B * heads, hd, nk, device=dev, dtype=bf16)
            qp[:, :, :hd] = q.reshape(B * heads, n, hd)
            kpd[:, :n, :hd] = k.reshape(B * heads, n, hd)
            vt[:, :, :n] = val.reshape(B * heads, n, hd).transpose(1, 2)
            s = torch.empty(B * heads, n, nk, device=dev, dtype=torch.float32)
            ops.gemm(qp, kpd, s, K=hp, N=nk, rows_per_batch=n, batch=B * heads, a_batch_stride=n * hp,
                     b_batch_stride=nk * hp, s0=1.0 / math.sqrt(hd))
            s[:, :, n:] = -1e30                                              # padded keys never attend
            p = torch.empty(B * heads * n, nk, device=dev, dtype=bf16)
            ops.softmax_rows_f32(s.view(-1, nk), p, B * heads * n, nk)
            o = torch.empty(B * heads, n, hd, device=dev, dtype=bf16)
            ops.gemm(p, vt, o, K=nk, N=hd, rows_per_batch=n, batch=B * heads, a_batch_stride=n * nk,
                     b_batch_stride=hd * nk)
            att = o.view(B, heads, n, hd).permute(0, 2, 1, 3).reshape(rows, w).contiguous()
            x_new = torch.empty_like(x_res)
            ops.gemm(att, blk["out_w"], x_new, K=w, N=w, rows_per_batch=rows, bias=blk["out_b"], r1=x_res, s1=1.0)
            self._tap(f"L{i}.attn", x_new, B, n)
            ops.layernorm(x_new, h_ln, *blk["ln2"], rows, w)
            m = torch.empty(rows, v.mlp, device=dev, dtype=bf16)
            ops.gemm(h_ln, blk["fc_w"], m, K=w, N=2 * v.mlp, rows_per_batch=rows, bias=blk["fc_b"], act=ops.ACT_GEGLU)
            x_res = torch.empty_like(x_new)
            ops.gemm(m, blk["proj_w"], x_res, K=v.mlp, N=w, rows_per_batch=rows, bias=blk["proj_b"], r1=x_new, s1=1.0)
            self._tap(f"L{i}.mlp", x_res, B, n)
        cls = x_res.view(B, n, w)[:, 0].contiguous()
        pooled = torch.empty_like(cls)
        ops.layernorm(cls, pooled, *P["ln_post"], B, w)
        z = torch.empty(B, v.embed_dim, device=dev, dtype=torch.float32)
        ops.small_linear(pooled.float(), P["proj_t"], None, z)
        return z

    def forward(self, image: torch.Tensor, no_dropout: bool = False) -> torch.Tensor:
        z = self.encode_with_vision_transformer(image).to(image.dtype)
        if self.ucg_rate > 0.0 and not no_dropout:
            z = torch.bernoulli((1.0 - self.ucg_rate) * torch.ones(z.shape[0], device=z.device))[:, None] * z
        return z[:, None, :] if self.unsqueeze_dim else z

    def encode(self, image):
        return self(image)


class FrozenOpenCLIPImagePredictionEmbedder(nn.Module):
    """encoders/modules.py:1054-1072: "(b t) d -> b t d" of the embedder's output, repeated n_copies times."""

    def __init__(self, open_clip_embedding_config: Dict, n_cond_frames: int, n_copies: int):
        super().__init__()
        self.n_cond_frames, self.n_copies = n_cond_frames, n_copies
        self.open_clip = instantiate_from_config(open_clip_embedding_config)

    def forward(self, vid: torch.Tensor) -> torch.Tensor:
        z = self.open_clip(vid)
        z = z.reshape(-1, self.n_cond_frames, z.shape[-1])
        return z.repeat_interleave(self.n_copies, dim=0)
