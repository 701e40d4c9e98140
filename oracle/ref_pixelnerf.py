"""Oracle for PixelNeRF scene conditioning: a functional restatement of sgm/modules/encoders/pixelnerf.py (RayGenerator
77-158, RaySampler 161-201, PixelNeRF.project / forward 237-313), math_utils.get_ray_limits_box / linspace and
PixelNeRFEmbedder.forward (encoders/modules.py:1075-1131), over a reference-keyed state_dict.

`precision="fp32"` is the reference's arithmetic (pinned against the real PixelNeRF by oracle/make_golden_scene.py).
`precision="kernel"` is the fp64 restatement of the fused kernel: rays, depths and sample points in fp32 (the
kernel's own order), everything after in fp64, rounded to bf16 exactly where the kernel rounds -- the MLP weights,
the MLP input row (mean | std | positional encoding), both hidden activations of each MLP and the per-ray feature
before the decoder.  `precision="kernel32"` rounds at the same points with fp32 arithmetic in between: its distance
from "kernel" is the floor any correct fp32 evaluation of the kernel's rounding schedule sits at.
"""
from __future__ import annotations

import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F


def rays(cams: torch.Tensor, rs: int, box: bool = True):
    """cams [N, 25] -> origins, directions [N, rs*rs, 3], t_start, t_end [N, rs*rs] (fp32; miss fallback applied)."""
    cams = cams.float()
    N = cams.shape[0]
    c2w = cams[:, :16].reshape(N, 4, 4)
    K = cams[:, 16:].reshape(N, 3, 3)
    fx, fy, cx, cy, sk = (K[:, 0, 0, None], K[:, 1, 1, None], K[:, 0, 2, None], K[:, 1, 2, None], K[:, 0, 1, None])
    dev = cams.device
    ar = torch.arange(rs, dtype=torch.float32, device=dev)
    uv = torch.stack(torch.meshgrid(ar, ar, indexing="ij")).flip(0).reshape(2, -1).transpose(1, 0)
    x_cam = uv[None, :, 0] * (1.0 / rs) + (0.5 / rs)
    y_cam = uv[None, :, 1] * (1.0 / rs) + (0.5 / rs)
    x_lift = (x_cam - cx + cy * sk / fy - sk * y_cam / fy) / fx
    y_lift = (y_cam - cy) / fy
    flip = torch.diag(torch.tensor([1.0, -1.0, -1.0, 1.0], device=dev))
    m = c2w @ flip
    pts = torch.stack([x_lift, y_lift, torch.ones_like(x_lift), torch.ones_like(x_lift)], -1)  # [N, M, 4]
    world = torch.einsum("nij,nmj->nmi", m, pts)[..., :3]
    o = c2w[:, None, :3, 3].expand_as(world)
    d = F.normalize(world - o, dim=2)
    if box:
        ts, te = _box_limits(o.reshape(-1, 3), d.reshape(-1, 3), 1.0)
        ts, te = ts.reshape(N, -1), te.reshape(N, -1)
        valid = te > ts
        if bool(valid.any()):
            lo, hi = ts[valid].min(), ts[valid].max()
            ts = torch.where(valid, ts, lo)
            te = torch.where(valid, te, hi)
    else:
        ts = te = torch.zeros(N, rs * rs, device=dev)
    return o.contiguous(), d.contiguous(), ts, te


def _box_limits(o, d, half):
    inv = 1 / d
    neg = inv < 0
    bmin = torch.where(neg, half, -half)
    bmax = torch.where(neg, -half, half)
    lo = (bmin - o) * inv
    hi = (bmax - o) * inv
    valid = ~((lo[:, 0] > hi[:, 1]) | (lo[:, 1] > hi[:, 0]))
    tmin, tmax = torch.maximum(lo[:, 0], lo[:, 1]), torch.minimum(hi[:, 0], hi[:, 1])
    valid &= ~((tmin > hi[:, 2]) | (lo[:, 2] > tmax))
    tmin, tmax = torch.maximum(tmin, lo[:, 2]), torch.minimum(tmax, hi[:, 2])
    return torch.where(valid, tmin, -1.0), torch.where(valid, tmax, -2.0)


def sample_points(o, d, ts, te, jitter, ns: int, disparity=False, near=0.5, far=10000.0):
    """[ns, N, M, 3] fp32.  jitter: [ns, N*M] uniforms, or z[ns] (linspace + jitter) with `disparity`."""
    if not disparity:
        steps = (torch.arange(ns, dtype=torch.float32, device=o.device) / (ns - 1))[:, None, None]
        diff = (te - ts)[None]
        depth = ts[None] + steps * diff
        depth = depth + jitter.reshape(ns, *ts.shape) * diff / (ns - 1)
    else:
        depth = (1 / (1 / near * (1 - jitter) + 1 / far * jitter))[:, None, None]
    return o[None] + d[None] * depth[..., None]


def _pos_enc(x):
    freqs = math.pi * 2.0 ** torch.arange(0, 6)  # fp32, as PositionalEncoding builds them
    f = torch.repeat_interleave(freqs, 2).to(x.device, x.dtype)
    ph = torch.zeros(12)
    ph[1::2] = math.pi * 0.5
    ph = ph.to(x.device, x.dtype)
    emb = torch.sin(ph[:, None] + x[..., None, :] * f[:, None])  # [..., 12, 3]
    return torch.cat([x, emb.flatten(-2)], dim=-1)


def _mlp(x, sd, prefix, q):
    for i in (0, 2, 4):
        w = q(sd[f"{prefix}.{i}.weight"].to(x.device, x.dtype))
        x = x @ w.T + sd[f"{prefix}.{i}.bias"].to(x.device, x.dtype)
        if i != 4:
            x = q(torch.relu(x))
    return x


def pixelnerf(sd: Dict[str, torch.Tensor], image_feats, source_c2ws, source_intrinsics, cams, rs: int, jitter,
              ns: int, *, use_std=False, use_pe=False, interp="bilinear", padding="border", disparity=False,
              near=0.5, far=10000.0, precision="fp32"):
    """Runs on the inputs' device.  image_feats [B, S, C, H, W]; source_c2ws [B, S, 4, 4]; source_intrinsics
    [B, S, 3, 3]; cams [B, T, 25].  Returns rgb [B, T, 3, rs, rs], feats [B, T, 128, rs, rs] and the per-ray feature [B*T*rs*rs, 128]."""
    kern = precision in ("kernel", "kernel32")
    dt = torch.float64 if precision == "kernel" else torch.float32
    q = (lambda t: t.to(torch.bfloat16).to(dt)) if kern else (lambda t: t)
    B, T = cams.shape[:2]
    S = source_c2ws.shape[1]
    o, d, ts, te = rays(cams.reshape(B * T, 25), rs, box=not disparity)
    pts = sample_points(o, d, ts, te, jitter.to(cams.device).float(), ns, disparity, near, far)  # [ns, BT, M, 3] fp32
    M = rs * rs
    pts = pts.reshape(ns, B, T, M, 3).permute(1, 2, 3, 0, 4).to(dt)  # B T M ns 3
    w2c = torch.inverse(source_c2ws.float()).to(dt)
    Kk = source_intrinsics.to(dt)
    homo = torch.cat([pts, torch.ones_like(pts[..., :1])], -1)
    proj = torch.einsum("bsij,btmnj->bstmni", w2c, homo)[..., :3]
    xy = -proj[..., :2] / proj[..., 2:]
    x = xy[..., 0] * Kk[:, :, 0, 0, None, None, None] + Kk[:, :, 0, 2, None, None, None]
    y = -xy[..., 1] * Kk[:, :, 1, 1, None, None, None] + Kk[:, :, 1, 2, None, None, None]
    grid = torch.stack([x, y], -1).reshape(B * S, T * M * ns, 1, 2) * 2.0 - 1.0
    feats_src = image_feats.to(dt).flatten(0, 1)
    joint = F.grid_sample(feats_src, grid, mode=interp, padding_mode=padding, align_corners=True)
    C = feats_src.shape[1]
    joint = joint.reshape(B, S, C, T, M, ns).permute(0, 1, 3, 4, 5, 2)  # B S T M ns C
    parts = [joint.mean(dim=1)]
    if use_std:
        parts.append(joint.std(dim=1) if S > 1 else torch.zeros_like(parts[0]))
    if use_pe:
        parts.append(_pos_enc(pts))
    red = q(torch.cat(parts, -1))
    out = _mlp(red, sd, "feature_aggregator", q)
    f, w = out[..., :128], out[..., 128:]
    w = torch.softmax(w, dim=-2)
    ray_feat = (f * w).sum(-2)  # B T M 128
    dec = _mlp(q(ray_feat), sd, "decoder", q)
    rgb = torch.sigmoid(dec[..., :3]).permute(0, 1, 3, 2).reshape(B, T, 3, rs, rs)
    fe = dec[..., 3:].permute(0, 1, 3, 2).reshape(B, T, 128, rs, rs)
    return rgb, fe, ray_feat.reshape(-1, 128)


def embedder_inputs(pixelnerf_input: Dict):
    """PixelNeRFEmbedder.forward's slicing (modules.py:1094-1121) with the identity image encoder:
    (image_feats, source_c2ws, source_intrinsics, target camera rows)."""
    if "source_index" not in pixelnerf_input:
        feats = pixelnerf_input["frames"][:, 0][:, None]
        src = pixelnerf_input["cameras"][:, :1]
    else:
        feats = pixelnerf_input["source_images"]
        src = pixelnerf_input["source_cameras"]
    cams = pixelnerf_input["cameras"]
    return (feats, src[..., :16].reshape(*src.shape[:-1], 4, 4), src[..., 16:].reshape(*src.shape[:-1], 3, 3), cams)


def embedder(sd, pixelnerf_input: Dict, rs: int, jitter, ns: int, precision: str = "fp32", **kw):
    """PixelNeRFEmbedder.forward: rgb [(b t), 3, rs, rs], feats [(b t), 128, rs, rs]."""
    feats, sc2w, sk, cams = embedder_inputs(pixelnerf_input)
    rgb, fe, _ = pixelnerf(sd, feats, sc2w, sk, cams, rs, jitter, ns, precision=precision, **kw)
    return rgb.flatten(0, 1), fe.flatten(0, 1)


def state_dict(d_in: int, seed: int, scale: Optional[float] = None) -> Dict[str, torch.Tensor]:
    """Seeded weights in the reference layout (nn.Linear's default init, optionally scaled)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}
    freqs = math.pi * 2.0 ** torch.arange(0, 6)
    sd["positional_encoder._freqs"] = torch.repeat_interleave(freqs, 2).view(1, -1, 1)
    ph = torch.zeros(12)
    ph[1::2] = math.pi * 0.5
    sd["positional_encoder._phases"] = ph.view(1, -1, 1)
    for prefix, dims in (("feature_aggregator", (d_in, 128, 128, 129)), ("decoder", (128, 128, 128, 131))):
        for i, (a, b) in enumerate(zip(dims[:-1], dims[1:])):
            bound = (scale or 1.0) / math.sqrt(a)
            sd[f"{prefix}.{2 * i}.weight"] = (torch.rand(b, a, generator=g) * 2 - 1) * bound
            sd[f"{prefix}.{2 * i}.bias"] = (torch.rand(b, generator=g) * 2 - 1) * bound
    return sd


FIXTURE_REL_L2 = 3e-2  # the project's output bound, applied to the whole output and to its pixel-varying part


def fixture_errors(out: torch.Tensor, ref: torch.Tensor):
    """(rel-L2 of the whole output, rel-L2 of its pixel-varying part) against a reference [..., C, H, W].  The
    pixel-varying part (each image channel minus its mean over pixels) is what the source images and cameras decide;
    the per-channel mean is mostly the MLP biases, so the whole-output error alone cannot tell a render that ignores
    the sources from a correct one."""
    out, ref = out.double().cpu(), ref.double().cpu()

    def cen(t):
        return t - t.mean(dim=(-2, -1), keepdim=True)
    return float((out - ref).norm() / ref.norm()), float((cen(out) - cen(ref)).norm() / cen(ref).norm())


def altered_sources(pixelnerf_input: Dict):
    """Two wrong inputs a correct embedder must tell apart from the right one: the sources zeroed, and the sources
    swapped (the last frame instead of the first; source order reversed and batch items exchanged)."""
    zero, swap = dict(pixelnerf_input), dict(pixelnerf_input)
    key = "source_images" if "source_index" in pixelnerf_input else "frames"
    zero[key] = torch.zeros_like(pixelnerf_input[key])
    swap[key] = pixelnerf_input[key].flip(1) if key == "frames" else pixelnerf_input[key].flip(1).flip(0)
    return {"zeroed": zero, "swapped": swap}
