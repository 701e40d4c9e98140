"""Torch stand-ins (CPU, fp32) for the three PixelNeRF entry points of v3d_b200.ops, so the host logic of PixelNeRF /
PixelNeRFEmbedder / ExtraConditioner runs without a GPU.  They read and write the same buffers as the kernels:
rays [R, 8], limits (set to "no fallback needed": the stand-in applies it itself), feat [R, 128], rgb / feats NCHW.
Weights are the packed bf16 images the kernels read, so the stand-ins see the kernels' weights.
`patched()` installs them and counts the calls."""
from __future__ import annotations

import contextlib
from collections import Counter

import torch
import torch.nn.functional as F

from oracle import ref_pixelnerf as R

CALLS: Counter = Counter()


def _rays(cams, render_size, rays, limits, box=True, box_half=1.0):
    CALLS["pixelnerf_rays"] += 1
    o, d, ts, te = R.rays(cams, render_size, box=box)
    rays.copy_(torch.cat([o.reshape(-1, 3), d.reshape(-1, 3), ts.reshape(-1, 1), te.reshape(-1, 1)], 1))
    limits.fill_(-1)
    return rays


def _mlp(x, mlp, k_in):
    w1, b1, w2, b2, w3, b3 = mlp
    x = torch.relu(x @ w1[:, :k_in].float().T + b1).bfloat16().float()
    x = torch.relu(x @ w2.float().T + b2).bfloat16().float()
    return x @ w3.float().T + b3


def _render(rays, limits, jitter, src, src_w2c, src_k, rays_per_batch, ns, flags, inv_near, inv_far, mlp, d_in,
            feat):
    from v3d_b200 import ops

    CALLS["pixelnerf_render"] += 1
    n = rays.shape[0]
    o, d, ts, te = rays[None, :, :3], rays[None, :, 3:6], rays[None, :, 6], rays[None, :, 7]
    disp = bool(flags & ops.PNERF_DISPARITY)
    pts = R.sample_points(o, d, ts, te, jitter, ns, disp, 1.0 / inv_near, 1.0 / inv_far).reshape(ns, n, 3)
    B, S, C, H, W = src.shape
    pts_b = pts.permute(1, 0, 2).reshape(B, -1, 3)  # B (rays ns) 3
    proj = torch.einsum("bsij,bmj->bsmi", src_w2c, torch.cat([pts_b, torch.ones_like(pts_b[..., :1])], -1))
    xy = -proj[..., :2] / proj[..., 2:]
    x = xy[..., 0] * src_k[..., 0, None] + src_k[..., 2, None]
    y = -xy[..., 1] * src_k[..., 1, None] + src_k[..., 3, None]
    grid = (torch.stack([x, y], -1) * 2 - 1).reshape(B * S, -1, 1, 2)
    joint = F.grid_sample(src.flatten(0, 1), grid, mode="nearest" if flags & ops.PNERF_NEAREST else "bilinear",
                          padding_mode="zeros" if flags & ops.PNERF_ZEROS else "border", align_corners=True)
    joint = joint.reshape(B, S, C, -1).permute(0, 1, 3, 2)  # B S (rays ns) C
    parts = [joint.mean(1)]
    if flags & ops.PNERF_STD:
        parts.append(joint.std(1) if S > 1 else torch.zeros_like(parts[0]))
    if flags & ops.PNERF_POSENC:
        parts.append(R._pos_enc(pts_b))
    red = torch.cat(parts, -1).reshape(n, ns, d_in).bfloat16().float()
    out = _mlp(red, mlp, d_in)
    w = torch.softmax(out[..., 128:129], dim=1)
    feat.copy_((out[..., :128] * w).sum(1))
    return feat


def _decode(feat, hw, mlp, rgb, feats):
    CALLS["pixelnerf_decode"] += 1
    out = _mlp(feat.bfloat16().float(), mlp, 128)
    n = feat.shape[0] // hw
    rgb.copy_(torch.sigmoid(out[:, :3]).reshape(n, hw, 3).permute(0, 2, 1))
    feats.copy_(out[:, 3:131].reshape(n, hw, 128).permute(0, 2, 1))
    return rgb, feats


@contextlib.contextmanager
def patched():
    from v3d_b200 import ops

    saved = (ops.pixelnerf_rays, ops.pixelnerf_render, ops.pixelnerf_decode)
    ops.pixelnerf_rays, ops.pixelnerf_render, ops.pixelnerf_decode = _rays, _render, _decode
    CALLS.clear()
    try:
        yield CALLS
    finally:
        ops.pixelnerf_rays, ops.pixelnerf_render, ops.pixelnerf_decode = saved
