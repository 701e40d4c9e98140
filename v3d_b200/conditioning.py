"""Conditioning assembly of V3D_512 on the device (SURVEY.md 8(f) rank 1): drop-ins for
`sgm.modules.encoders.modules.{GeneralConditioner, ConcatTimestepEmbedderND, IdentityEncoder}`
(encoders/modules.py:85-206, 937-953) and the `get_batch` / per-frame repeat steps of scripts/pub/V3D_512.py:31-69,
247-262.  Runs once per image; the only arithmetic is the sinusoidal embedding (`v3d_timestep_embedding`).

Oracle pinned bit-exactly against the real GeneralConditioner (tests/golden/conditioning.pt); host logic tested on CPU,
the device path in tests/test_kernels_gpu.py::test_concat_timestep_embedder_device.
"""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple

import torch
import torch.nn as nn

from . import ops
from .sampling import instantiate_from_config


class AbstractEmbModel(nn.Module):
    """encoders/modules.py:43-82: carries is_trainable / ucg_rate / input_key set by the conditioner."""

    def __init__(self):
        super().__init__()
        self.is_trainable = False
        self.ucg_rate = 0.0
        self.input_key: Optional[str] = None
        self.legacy_ucg_val = None


class IdentityEncoder(AbstractEmbModel):
    def encode(self, x):
        return x

    def forward(self, x):
        return x


class ConcatTimestepEmbedderND(AbstractEmbModel):
    """Every scalar of x embedded on its own with timestep_embedding(., outdim), concatenated per row."""

    def __init__(self, outdim: int):
        super().__init__()
        self.outdim = outdim

    def forward(self, x: torch.Tensor) -> torch.Tensor:
        if x.ndim == 1:
            x = x[:, None]
        assert x.ndim == 2
        b, dims = x.shape
        flat = x.reshape(-1).float().contiguous()
        emb = torch.empty(flat.numel(), self.outdim, device=x.device, dtype=torch.float32)
        ops.timestep_embedding(flat, emb, self.outdim)   # raises on CPU tensors: no CPU fallback
        return emb.reshape(b, dims * self.outdim)


class GeneralConditioner(nn.Module):
    OUTPUT_DIM2KEYS = {2: "vector", 3: "crossattn", 4: "concat", 5: "concat"}
    KEY2CATDIM = {"vector": 1, "crossattn": 2, "concat": 1}

    def __init__(self, emb_models: List[dict]):
        super().__init__()
        embedders = []
        for cfg in emb_models:
            e = instantiate_from_config(cfg)
            e.is_trainable = cfg.get("is_trainable", False)
            e.ucg_rate = cfg.get("ucg_rate", 0.0)
            if "input_key" in cfg:
                e.input_key = cfg["input_key"]
            elif "input_keys" in cfg:
                e.input_keys = cfg["input_keys"]
            else:
                raise KeyError(f"need either 'input_key' or 'input_keys' for embedder {type(e).__name__}")
            if cfg.get("legacy_ucg_value", None) is not None:
                raise NotImplementedError("legacy_ucg_value is a training-time option")
            embedders.append(e.eval())
        self.embedders = nn.ModuleList(embedders)

    def forward(self, batch: Dict, force_zero_embeddings: Optional[List[str]] = None) -> Dict:
        out: Dict[str, torch.Tensor] = {}
        force_zero_embeddings = force_zero_embeddings or []
        for e in self.embedders:
            with torch.no_grad():
                if getattr(e, "input_key", None) is not None:
                    emb_out = e(batch[e.input_key])
                else:
                    emb_out = e(*[batch[k] for k in e.input_keys])
            for emb in (emb_out if isinstance(emb_out, (list, tuple)) else [emb_out]):
                key = self.OUTPUT_DIM2KEYS[emb.dim()]
                if e.ucg_rate > 0.0:
                    keep = torch.bernoulli((1.0 - e.ucg_rate) * torch.ones(emb.shape[0], device=emb.device))
                    emb = keep.reshape(-1, *([1] * (emb.dim() - 1))) * emb
                if getattr(e, "input_key", None) in force_zero_embeddings:
                    emb = torch.zeros_like(emb)
                out[key] = torch.cat((out[key], emb), self.KEY2CATDIM[key]) if key in out else emb
        return out

    def get_unconditional_conditioning(self, batch_c: Dict, batch_uc: Optional[Dict] = None,
                                       force_uc_zero_embeddings: Optional[List[str]] = None,
                                       force_cond_zero_embeddings: Optional[List[str]] = None):
        rates = [e.ucg_rate for e in self.embedders]
        for e in self.embedders:
            e.ucg_rate = 0.0
        try:
            c = self(batch_c, force_cond_zero_embeddings)
            uc = self(batch_c if batch_uc is None else batch_uc, force_uc_zero_embeddings or [])
        finally:
            for e, r in zip(self.embedders, rates):
                e.ucg_rate = r
        return c, uc


V3D_512_EMB_MODELS = [  # scripts/pub/configs/V3D_512.yaml:59-86, native targets
    {"input_key": "cond_frames_without_noise", "is_trainable": False, "ucg_rate": 0.2,
     "target": "v3d_b200.conditioning.IdentityEncoder"},
    {"input_key": "fps_id", "is_trainable": True, "target": "v3d_b200.conditioning.ConcatTimestepEmbedderND",
     "params": {"outdim": 256}},
    {"input_key": "motion_bucket_id", "is_trainable": True,
     "target": "v3d_b200.conditioning.ConcatTimestepEmbedderND", "params": {"outdim": 256}},
    {"input_key": "cond_frames", "is_trainable": False, "ucg_rate": 0.2,
     "target": "v3d_b200.conditioning.IdentityEncoder"},
    {"input_key": "cond_aug", "is_trainable": True, "target": "v3d_b200.conditioning.ConcatTimestepEmbedderND",
     "params": {"outdim": 256}},
]


def get_batch(keys, value_dict: Dict, N: List[int], T: Optional[int], device) -> Tuple[Dict, Dict]:
    """scripts/pub/V3D_512.py:31-69: scalars repeated prod(N) times, the two frame tensors repeated N[0] times."""
    n = 1
    for v in N:
        n *= int(v)
    batch: Dict = {}
    for key in keys:
        if key in ("fps_id", "motion_bucket_id", "cond_aug"):
            batch[key] = torch.tensor([value_dict[key]]).to(device).repeat(n)
        elif key in ("cond_frames", "cond_frames_without_noise"):
            v = value_dict[key]
            batch[key] = v[:1].expand(N[0], *v.shape[1:]).clone()
        else:
            batch[key] = value_dict[key]
    if T is not None:
        batch["num_video_frames"] = T
    batch_uc = {k: v.clone() for k, v in batch.items() if isinstance(v, torch.Tensor)}
    return batch, batch_uc


def assemble_v3d_conditioning(conditioner: GeneralConditioner, clip_emb: torch.Tensor, cond_latent: torch.Tensor,
                              fps_id: float, motion_bucket_id: float, cond_aug: float, T: int):
    """(c, uc) as `sample_one` hands them to the sampler (V3D_512.py:247-262): conditioner on the [1, T] batch with the
    two frame embedders zeroed in uc, then crossattn / concat repeated "b ... -> (b t) ...".  `cond_latent` is the
    already noised first-stage latent (`ae.encode(image) + cond_aug * randn`, V3D_512.py:239-242)."""
    keys = [e.input_key for e in conditioner.embedders]
    value = {"fps_id": fps_id, "motion_bucket_id": motion_bucket_id, "cond_aug": cond_aug,
             "cond_frames": cond_latent, "cond_frames_without_noise": clip_emb}
    batch, batch_uc = get_batch(keys, value, [1, T], T, clip_emb.device)
    c, uc = conditioner.get_unconditional_conditioning(
        batch, batch_uc=batch_uc, force_uc_zero_embeddings=["cond_frames", "cond_frames_without_noise"])
    for d in (c, uc):
        for k in ("crossattn", "concat"):
            t = d[k]
            d[k] = t.unsqueeze(1).expand(t.shape[0], T, *t.shape[1:]).reshape(-1, *t.shape[1:]).contiguous()
    return c, uc
