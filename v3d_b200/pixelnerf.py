"""Sparse-view scene conditioning of V3D: drop-ins for `sgm.modules.encoders.pixelnerf.{PixelNeRF, ImageEncoder}`
(sgm/modules/encoders/pixelnerf.py), `sgm.modules.encoders.modules.PixelNeRFEmbedder` (modules.py:1075-1131) and
`ExtraConditioner` (modules.py:1134-1187).

The whole per-sample computation (jittered depths, projection into every source, grid_sample, mean / std /
positional encoding, the feature MLP and the softmax over the samples of each ray) is one fused kernel
(csrc/pixelnerf.cu); the reference materialises every per-sample tensor.  torch only owns the buffers, draws the
jitter and does the per-source 4x4 inverse.  Weights keep the reference's state_dict layout; their bf16 / padded
kernel image is packed on first use and re-packed whenever a parameter changes.
"""
from __future__ import annotations

from typing import Callable, Dict, List, Optional

import numpy as np
import torch
import torch.nn as nn

from . import ops
from .conditioning import AbstractEmbModel, GeneralConditioner
from .sampling import instantiate_from_config

MAX_D_IN = 192  # three 64-column panels of the fused kernel's A tile


class ImageEncoder(nn.Module):
    """pixelnerf.py:13-19: the identity (the only image encoder the native path runs)."""

    def __init__(self, output_dim: int = 64) -> None:
        super().__init__()
        self.output_dim = output_dim

    def forward(self, image):
        return image


class PositionalEncoding(nn.Module):
    """pixelnerf.py:22-61, default arguments only (what PixelNeRF builds): holds the persistent `_freqs` / `_phases`
    buffers of the reference's state_dict.  The kernel evaluates sin(x * f + phase) with these same fp32 values."""

    def __init__(self, num_freqs: int = 6, d_in: int = 3, freq_factor: float = np.pi, include_input: bool = True):
        super().__init__()
        if (num_freqs, d_in, freq_factor, include_input) != (6, 3, np.pi, True):
            raise NotImplementedError("the native positional encoding is PixelNeRF's default (6 frequencies of xyz)")
        self.num_freqs, self.d_in, self.include_input = num_freqs, d_in, include_input
        self.freqs = freq_factor * 2.0 ** torch.arange(0, num_freqs)
        self.d_out = num_freqs * 2 * d_in + d_in
        self.register_buffer("_freqs", torch.repeat_interleave(self.freqs, 2).view(1, -1, 1))
        phases = torch.zeros(2 * num_freqs)
        phases[1::2] = np.pi * 0.5
        self.register_buffer("_phases", phases.view(1, -1, 1))


def _default_jitter(shape, device) -> torch.Tensor:
    return torch.rand(shape, dtype=torch.float32, device=device)


class PixelNeRF(nn.Module):
    """pixelnerf.py:192-313 on three launches: rays, the fused render, the per-ray decoder.

    `jitter_sampler(shape, device)` returns the uniforms the reference draws with `torch.rand_like` (shape
    [Ns, B*T, H*W, 1], or [Ns] with `disparity`); the default draws them with torch.rand, in the reference's order."""

    def __init__(self, num_samples_per_ray: int = 128, feature_dim: int = 64, interp: str = "bilinear",
                 padding: str = "border", disparity: bool = False, near: float = 0.5, far: float = 10000.0,
                 use_feats_std: bool = False, use_pos_emb: bool = False,
                 jitter_sampler: Optional[Callable] = None) -> None:
        super().__init__()
        if interp not in ("bilinear", "nearest"):
            raise NotImplementedError(f"grid_sample mode {interp!r}: the native render has bilinear and nearest")
        if padding not in ("border", "zeros"):
            raise NotImplementedError(f"grid_sample padding {padding!r}: the native render has border and zeros")
        if num_samples_per_ray < 2:
            raise NotImplementedError("num_samples_per_ray < 2 (the reference's linspace divides by Ns - 1)")
        self.num_samples_per_ray = num_samples_per_ray
        self.interp, self.padding = interp, padding
        self.disparity, self.near, self.far = disparity, near, far
        self.use_feats_std, self.use_pos_emb = use_feats_std, use_pos_emb
        self.jitter_sampler = jitter_sampler or _default_jitter
        self.positional_encoder = PositionalEncoding()
        d_in = feature_dim * (2 if use_feats_std else 1) + (self.positional_encoder.d_out if use_pos_emb else 0)
        if d_in > MAX_D_IN:
            raise NotImplementedError(f"feature MLP input width {d_in} > {MAX_D_IN}")
        self.d_in = d_in
        self.feature_aggregator = nn.Sequential(nn.Linear(d_in, 128), nn.ReLU(), nn.Linear(128, 128), nn.ReLU(),
                                                nn.Linear(128, 129))
        self.decoder = nn.Sequential(nn.Linear(128, 128), nn.ReLU(), nn.Linear(128, 128), nn.ReLU(),
                                     nn.Linear(128, 131))
        self._packed = None
        self._packed_key = None

    @property
    def flags(self) -> int:
        return ((ops.PNERF_STD if self.use_feats_std else 0) | (ops.PNERF_POSENC if self.use_pos_emb else 0)
                | (ops.PNERF_NEAREST if self.interp == "nearest" else 0)
                | (ops.PNERF_ZEROS if self.padding == "zeros" else 0)
                | (ops.PNERF_DISPARITY if self.disparity else 0))

    @staticmethod
    def _pack_mlp(seq: nn.Sequential, device) -> tuple:
        def w(lin, rows, cols):
            out = torch.zeros(rows, cols, dtype=torch.bfloat16, device=device)
            out[:lin.weight.shape[0], :lin.weight.shape[1]] = lin.weight.detach().to(device, torch.bfloat16)
            return out

        def b(lin, n):
            out = torch.zeros(n, dtype=torch.float32, device=device)
            out[:lin.bias.shape[0]] = lin.bias.detach().to(device, torch.float32)
            return out

        l1, l2, l3 = seq[0], seq[2], seq[4]
        k1 = -(-l1.weight.shape[1] // 64) * 64
        return (w(l1, 128, k1), b(l1, 128), w(l2, 128, 128), b(l2, 128), w(l3, 136, 128), b(l3, 136))

    def packed(self, device):
        key = (str(device),) + tuple((p.data_ptr(), p._version) for p in self.parameters())
        if self._packed_key != key:
            self._packed = (self._pack_mlp(self.feature_aggregator, device), self._pack_mlp(self.decoder, device))
            self._packed_key = key
        return self._packed

    def draw_jitter(self, BT: int, HW: int, device) -> torch.Tensor:
        """The reference's uniforms (RaySampler.forward, pixelnerf.py:189-201), in the form the kernel reads."""
        ns = self.num_samples_per_ray
        if not self.disparity:
            return self.jitter_sampler((ns, BT, HW, 1), device).float().reshape(ns, BT * HW).contiguous()
        step = 1.0 / ns
        z = torch.linspace(0, 1 - step, ns, device=device)
        z += self.jitter_sampler((ns,), device).float().reshape(ns) * step
        return z.contiguous()

    def ray_features(self, image_feats, source_c2ws, source_intrinsics, c2ws, intrinsics, render_size: int,
                     feat: Optional[torch.Tensor] = None) -> torch.Tensor:
        """The per-ray softmax-weighted feature [B*T*render_size**2, 128] fp32 (pixelnerf.py:263-303), written into
        `feat` when given."""
        B, T = c2ws.shape[:2]
        if image_feats.shape[0] != B or source_c2ws.shape[:2] != image_feats.shape[:2] \
                or source_intrinsics.shape[:2] != image_feats.shape[:2]:
            raise ValueError(f"PixelNeRF: sources {tuple(image_feats.shape)} / {tuple(source_c2ws.shape)} / "
                             f"{tuple(source_intrinsics.shape)} do not match the {B} target camera batches")
        dev = c2ws.device
        # PixelNeRF takes the device check only: a CPU tensor is refused by its first launch (ops._need), so the
        # conditioner keeps running on CPU under the launch stand-ins alone, as its existing tests do
        if c2ws.is_cuda:
            ops.require_current_device(c2ws, "PixelNeRF")
        hw = render_size * render_size
        nrays = B * T * hw
        cams = torch.cat([c2ws.reshape(B * T, 16), intrinsics.reshape(B * T, 9)], dim=1).float().contiguous()
        rays = torch.empty(nrays, 8, device=dev, dtype=torch.float32)
        limits = torch.empty(2, device=dev, dtype=torch.int32)
        ops.pixelnerf_rays(cams, render_size, rays, limits, box=not self.disparity)
        jitter = self.draw_jitter(B * T, hw, dev)
        src = image_feats.float().contiguous()
        w2c = torch.inverse(source_c2ws.float())[..., :3, :].contiguous()
        k = source_intrinsics.float()
        src_k = torch.stack([k[..., 0, 0], k[..., 1, 1], k[..., 0, 2], k[..., 1, 2]], dim=-1).contiguous()
        agg, _ = self.packed(dev)
        if feat is None:
            feat = torch.empty(nrays, 128, device=dev, dtype=torch.float32)
        ops.pixelnerf_render(rays, limits, jitter, src, w2c, src_k, T * hw, self.num_samples_per_ray, self.flags,
                             float(1.0 / self.near), float(1.0 / self.far), agg, self.d_in, feat)
        return feat

    def forward(self, image_feats, source_c2ws, source_intrinsics, c2ws, intrinsics, render_size: int):
        B, T = c2ws.shape[:2]
        hw = render_size * render_size
        feat = self.ray_features(image_feats, source_c2ws, source_intrinsics, c2ws, intrinsics, render_size)
        _, dec = self.packed(c2ws.device)
        rgb = torch.empty(B * T, 3, hw, device=c2ws.device, dtype=torch.float32)
        feats = torch.empty(B * T, 128, hw, device=c2ws.device, dtype=torch.float32)
        ops.pixelnerf_decode(feat, hw, dec, rgb, feats)
        return (rgb.reshape(B, T, 3, render_size, render_size),
                feats.reshape(B, T, 128, render_size, render_size))


class PixelNeRFEmbedder(AbstractEmbModel):
    """modules.py:1075-1131: both input forms (the first frame as the one source, or source_images / source_cameras).
    Camera rows are 25 floats: c2w (4x4, row-major), then the normalised intrinsics (3x3)."""

    def __init__(self, image_encoder_config: dict, pixelnerf_encoder_config: dict, render_size: int,
                 num_video_frames: int):
        super().__init__()
        self.render_size = render_size
        self.num_video_frames = num_video_frames
        self.image_encoder = instantiate_from_config(image_encoder_config)
        if type(self.image_encoder) is not ImageEncoder:
            raise NotImplementedError("only the identity ImageEncoder runs natively (learned encoders are not ported)")
        self.pixelnerf_encoder = instantiate_from_config(pixelnerf_encoder_config)
        if not isinstance(self.pixelnerf_encoder, PixelNeRF):
            raise NotImplementedError("pixelnerf_encoder_config must build v3d_b200's PixelNeRF")

    def forward(self, pixelnerf_input: Dict):
        if "source_index" not in pixelnerf_input:
            image_feats = self.image_encoder(pixelnerf_input["frames"][:, 0])[:, None]
            source_cameras = pixelnerf_input["cameras"][:, :1]
        else:
            source_images = pixelnerf_input["source_images"]
            b, n = source_images.shape[:2]
            image_feats = self.image_encoder(source_images.reshape(b * n, *source_images.shape[2:]))
            image_feats = image_feats.reshape(b, n, *image_feats.shape[1:])
            source_cameras = pixelnerf_input["source_cameras"]
        cameras = pixelnerf_input["cameras"]
        rgb, feats = self.pixelnerf_encoder(
            image_feats,
            source_cameras[..., :16].reshape(*source_cameras.shape[:-1], 4, 4),
            source_cameras[..., 16:].reshape(*source_cameras.shape[:-1], 3, 3),
            cameras[..., :16].reshape(*cameras.shape[:-1], 4, 4),
            cameras[..., 16:].reshape(*cameras.shape[:-1], 3, 3),
            self.render_size,
        )
        return rgb.flatten(0, 1), feats.flatten(0, 1)


class ExtraConditioner(GeneralConditioner):
    """modules.py:1134-1187: GeneralConditioner with the PixelNeRF `rgb` output key, `bs = batch["frames"].shape[0]`,
    and crossattn / concat repeated "b ... -> (b t) ..." (t = batch["num_video_frames"]) whenever their batch size is
    not bs -- checked after every concatenation, as the reference does."""

    def forward(self, batch: Dict, force_zero_embeddings: Optional[List[str]] = None) -> Dict:
        bs = batch["frames"].shape[0]
        num_frames = batch["num_video_frames"]
        out: Dict[str, torch.Tensor] = {}
        force_zero_embeddings = force_zero_embeddings or []
        for e in self.embedders:
            with torch.no_grad():
                if getattr(e, "input_key", None) is not None:
                    emb_out = e(batch[e.input_key])
                else:
                    emb_out = e(*[batch[k] for k in e.input_keys])
            if not isinstance(emb_out, (list, tuple)):
                emb_out = [emb_out]
            if isinstance(e, PixelNeRFEmbedder):
                out["rgb"] = emb_out[0]
                emb_out = emb_out[1:]
            for emb in emb_out:
                key = self.OUTPUT_DIM2KEYS[emb.dim()]
                if e.ucg_rate > 0.0:
                    keep = torch.bernoulli((1.0 - e.ucg_rate) * torch.ones(emb.shape[0], device=emb.device))
                    emb = keep.reshape(-1, *([1] * (emb.dim() - 1))) * emb
                if getattr(e, "input_key", None) in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                out[key] = torch.cat((out[key], emb), self.KEY2CATDIM[key]) if key in out else emb
                if key in ("crossattn", "concat") and out[key].shape[0] != bs:
                    t = out[key]
                    out[key] = t.unsqueeze(1).expand(t.shape[0], num_frames, *t.shape[1:]).reshape(
                        -1, *t.shape[1:])
        return out
