"""The steps of `sample_one` either side of the hot path (scripts/pub/V3D_512.py:235-306; SURVEY.md 8(f)-1/-2), composed
from the drop-in pieces: first-stage encode of the conditioning image, conditioning-augmentation noise, conditioner +
per-frame repeat, latent noise, sampler loop + decode, uint8 wire format.  The CLIP image embedding is an INPUT of these
functions ([1, k, 1024]: one token per image, or k with n_cond_frames = k); the native ViT-H/14 image tower that
produces it is v3d_b200.clip.

Random draws happen in the reference's order and on the reference's generators, so that with the same
`torch.manual_seed(seed)` (V3D_512.py:177) a run reproduces the reference's noise: posterior sample of the encoder on
the CPU generator (distributions.py:37-41), then `randn_like(latent)` and `randn(shape)` on the device generator
(V3D_512.py:239-242,269).
"""
from __future__ import annotations

from typing import Dict, Optional, Tuple

import torch

from .conditioning import assemble_v3d_conditioning


@torch.no_grad()
def condition_on_image(engine, image: torch.Tensor, clip_emb: torch.Tensor, num_frames: int, fps_id: float = 1,
                       motion_bucket_id: float = 300, cond_aug: float = 0.02) -> Tuple[Dict, Dict]:
    """image [1,3,H,W] in [-1,1] -> (c, uc) as the sampler receives them.  `ae_model.encode(image)` of the reference is
    the UNSCALED first-stage latent (V3D_512.py:239: no scale_factor), noised by cond_aug * randn_like."""
    latent = engine.first_stage_model.encode(image)
    latent = latent + cond_aug * torch.randn_like(latent)
    return assemble_v3d_conditioning(engine.conditioner, clip_emb.to(image.device), latent, fps_id, motion_bucket_id,
                                     cond_aug, num_frames)


@torch.no_grad()
def views_from_image(engine, image: torch.Tensor, clip_emb: torch.Tensor, num_frames: int = 18, fps_id: float = 1,
                     motion_bucket_id: float = 300, cond_aug: float = 0.02, noise: Optional[torch.Tensor] = None,
                     decoding_t: Optional[int] = None, shard=None) -> torch.Tensor:
    """One conditioning image -> the T generated views [T,3,H,W] fp32 in [-1,1] (this rank's frames when `shard` is a
    ShardPlan).  `v3d_b200.wire.frames_to_u8` / `write_video` / `orbit_poses` take it from there."""
    _, _, H, W = image.shape
    assert image.shape[:2] == (1, 3) and H % 64 == 0 and W % 64 == 0, "one RGB image, sides divisible by 64"
    c, uc = condition_on_image(engine, image, clip_emb, num_frames, fps_id, motion_bucket_id, cond_aug)
    randn = torch.randn((num_frames, 4, H // 8, W // 8), device=image.device) if noise is None else noise.to(image.device)
    return engine.sample_views(randn, c, uc, num_frames, decoding_t=decoding_t or num_frames, shard=shard)
