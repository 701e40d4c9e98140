"""Engine / plugin hub: drop-in for the inference side of `sgm.models.video_diffusion.DiffusionEngine`
(sgm/models/video_diffusion.py:34-210): owns `.model` (OpenAIWrapper around the UNet), `.denoiser`,
`.sampler`, `.first_stage_model`, `.conditioner`; `decode_first_stage(z)` keeps the reference's chunking
semantics (`en_and_decode_n_samples_a_time`, video_diffusion.py:182-210).  Training hooks (Lightning steps,
EMA, losses, loggers) are out of scope (SURVEY.md §2 rows 14, 19).
"""
from __future__ import annotations

import contextlib
import copy
import math
import os
from typing import Dict, Optional

import torch
import torch.nn as nn

from .sampling import instantiate_from_config

OPENAIUNETWRAPPER = "v3d_b200.sampling.OpenAIWrapper"


def v3d_512_config(num_frames: int = 18, num_steps: int = 25, min_cfg: float = 3.5, max_cfg: float = 3.5,
                   sigma_max: float = 700.0) -> Dict:
    """scripts/pub/configs/V3D_512.yaml with `target:`s pointing at this package and the run-time pokes of
    load_model (scripts/pub/V3D_512.py:72-112) already applied. Conditioner omitted (out of scope)."""
    return {
        "scale_factor": 0.18215,
        "disable_first_stage_autocast": True,
        "denoiser_config": {
            "target": "v3d_b200.sampling.Denoiser",
            "params": {"scaling_config": {"target": "v3d_b200.sampling.VScalingWithEDMcNoise"}},
        },
        "network_config": {
            "target": "v3d_b200.unet.VideoUNet",
            "params": dict(
                adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
                model_channels=320, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
                num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
                spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
                merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1]),
        },
        "first_stage_config": {
            "target": "v3d_b200.decoder.AutoencodingEngine",
            "params": {
                "decoder_config": {
                    "target": "v3d_b200.decoder.VideoDecoder",
                    "params": dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256, in_channels=3,
                                   out_ch=3, ch=128, ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[],
                                   dropout=0.0, video_kernel_size=[3, 1, 1]),
                },
            },
        },
        "sampler_config": {
            "target": "v3d_b200.sampling.EulerEDMSampler",
            "params": {
                "num_steps": num_steps,
                "discretization_config": {"target": "v3d_b200.sampling.EDMDiscretization",
                                          "params": {"sigma_max": sigma_max}},
                "guider_config": {"target": "v3d_b200.sampling.LinearPredictionGuider",
                                  "params": {"max_scale": max_cfg, "min_scale": min_cfg, "num_frames": num_frames}},
            },
        },
    }


class DiffusionEngine(nn.Module):
    def __init__(self, network_config, denoiser_config, first_stage_config, conditioner_config=None,
                 sampler_config=None, optimizer_config=None, scheduler_config=None, loss_fn_config=None,
                 network_wrapper: Optional[str] = None, ckpt_path: Optional[str] = None, use_ema: bool = False,
                 ema_decay_rate: float = 0.9999, scale_factor: float = 1.0, disable_first_stage_autocast=False,
                 input_key: str = "jpg", log_keys=None, no_cond_log: bool = False, compile_model: bool = False,
                 en_and_decode_n_samples_a_time: Optional[int] = None, **ignored):
        super().__init__()
        self.input_key = input_key
        network = instantiate_from_config(network_config)
        wrapper = {"target": network_wrapper or OPENAIUNETWRAPPER}
        from .sampling import get_obj_from_str

        self.model = get_obj_from_str(wrapper["target"])(network, compile_model=compile_model)
        self.denoiser = instantiate_from_config(denoiser_config)
        self.sampler = instantiate_from_config(sampler_config) if sampler_config is not None else None
        self.conditioner = instantiate_from_config(conditioner_config) if conditioner_config is not None else None
        self.first_stage_model = instantiate_from_config(first_stage_config).eval()
        for p in self.first_stage_model.parameters():
            p.requires_grad = False
        self.scale_factor = scale_factor
        self.disable_first_stage_autocast = disable_first_stage_autocast
        self.en_and_decode_n_samples_a_time = en_and_decode_n_samples_a_time
        if ckpt_path is not None:
            self.init_from_ckpt(ckpt_path)

    def init_from_ckpt(self, path: str) -> None:
        """Same filtering as video_diffusion.py:123-168: drop shape-mismatched keys, load non-strictly."""
        if path.endswith("ckpt"):
            sd = torch.load(path, map_location="cpu")["state_dict"]
        elif path.endswith("safetensors"):
            from safetensors.torch import load_file

            sd = load_file(path)
        else:
            raise NotImplementedError
        own = self.state_dict()
        sd = {k: v for k, v in sd.items() if k not in own or tuple(own[k].shape) == tuple(v.shape)}
        missing, unexpected = self.load_state_dict(sd, strict=False)
        print(f"Restored from {path} with {len(missing)} missing and {len(unexpected)} unexpected keys")

    @contextlib.contextmanager
    def ema_scope(self, context=None):
        """`with model.ema_scope():` of the reference's callers (sgm/inference/helpers.py:123, video_diffusion.py:324-338
        swaps in the EMA weights when `use_ema`); this engine is inference-only and holds one set of weights, so the
        scope is a no-op - it exists so that `do_sample` runs against the drop-in engine unchanged."""
        yield None

    @torch.no_grad()
    def decode_first_stage(self, z: torch.Tensor) -> torch.Tensor:
        z = 1.0 / self.scale_factor * z
        is_video_input = z.dim() == 5
        bs = z.shape[0]
        if is_video_input:
            z = z.reshape(-1, *z.shape[2:])
        n_samples = self.en_and_decode_n_samples_a_time or z.shape[0]
        outs = []
        for n in range(math.ceil(z.shape[0] / n_samples)):
            chunk = z[n * n_samples:(n + 1) * n_samples]
            outs.append(self.first_stage_model.decode(chunk, timesteps=len(chunk)))
        out = torch.cat(outs, dim=0) if len(outs) > 1 else outs[0]
        if is_video_input:
            out = out.reshape(bs, -1, *out.shape[1:])
        return out

    @torch.no_grad()
    def encode_first_stage(self, x: torch.Tensor) -> torch.Tensor:
        """video_diffusion.py:212-237: images (or a [b,t,c,h,w] video, flattened and NOT folded back, as in the
        reference) -> scale_factor * first_stage_model.encode(.), in chunks of `en_and_decode_n_samples_a_time`.
        Needs the native encoder (AutoencodingEngine built with `encoder_config.target` = this package's Encoder)."""
        if self.input_key == "latents":
            return x * self.scale_factor
        if x.dim() == 5:
            x = x.reshape(-1, *x.shape[2:])
        n_samples = self.en_and_decode_n_samples_a_time or x.shape[0]
        outs = [self.first_stage_model.encode(x[n * n_samples:(n + 1) * n_samples])
                for n in range(math.ceil(x.shape[0] / n_samples))]
        z = torch.cat(outs, dim=0) if len(outs) > 1 else outs[0]
        return self.scale_factor * z

    @torch.no_grad()
    def sample_views(self, randn: torch.Tensor, c: Dict, uc: Dict, num_frames: int,
                     decoding_t: Optional[int] = None, view_shard=None, shard=None) -> torch.Tensor:
        """The hot path of sample_one (scripts/pub/V3D_512.py:269-285): sampler loop + first-stage decode.
        randn [T,4,h,w] fp32 (scaled in place, as in the reference); returns [T,3,8h,8w] fp32.

        ONE image over several ranks: `shard` = a v3d_b200.viewshard.ShardPlan (frame blocks, CFG-pair split, or both;
        `view_shard=ViewShard` is shorthand for the frame-block plan).  Every rank passes the SAME full-video randn / c /
        uc and gets back the decoded frames of its own block [t_local,3,8h,8w]; `gather_frames` of the plan (or of the
        ViewShard) assembles the video.  The video is decoded as one chunk (decoding_t = T).

        Samplers that inject noise every step (those with a `noise_sampler`: EulerAncestralSampler,
        DPMPP2SAncestralSampler) draw it, on every rank, for the WHOLE video - `noise_sampler` is called on a [T, ...]
        tensor - and keep this rank's frames of the draw.  So all ranks must start from the same generator state (seed
        them identically, as they already pass the identical `randn`); they then inject exactly the noise of the
        unsharded call."""
        if view_shard is not None and shard is None:
            from .viewshard import ShardPlan

            shard = ShardPlan("views", num_frames, view_shard, None, view_shard)
        if shard is not None:
            return self._sample_views_sharded(randn, c, uc, num_frames, shard)
        extra = {"image_only_indicator": torch.zeros(2, num_frames, device=randn.device),
                 "num_video_frames": num_frames}

        def denoiser(inp, sigma, cond):
            return self.denoiser(self.model, inp, sigma, cond, **extra)

        samples_z = self.sampler(denoiser, randn, cond=c, uc=uc)
        self.en_and_decode_n_samples_a_time = decoding_t or min(24, num_frames)
        return self.decode_first_stage(samples_z)

    @torch.no_grad()
    def _sample_views_sharded(self, randn: torch.Tensor, c: Dict, uc: Dict, num_frames: int, plan) -> torch.Tensor:
        """One image spread over ranks (SURVEY.md 8(e)).  Frame blocks: the sampler state, the CFG pair and the Euler
        update of a frame stay on its rank, the UNet exchanges K|V, conv halos and 3-D GroupNorm statistics.  CFG split:
        each rank of a pair runs the network on one half of [uc; c] and the halves are all-gathered before the
        guidance.  The decode always runs on frame blocks (`plan.decode`)."""
        from .viewshard import CfgSplitGuider

        vs, cs, dvs = plan.sample, plan.cfg, plan.decode
        assert plan.num_frames == num_frames and randn.shape[0] == num_frames
        unet = self.model.diffusion_model
        decoder = self.first_stage_model.decoder
        frames = vs.frames if vs is not None else slice(0, num_frames)
        tl = vs.tl if vs is not None else num_frames
        x = randn[frames].clone()
        c_l, uc_l = (vs.shard_cond(c), vs.shard_cond(uc)) if vs is not None else (c, uc)
        nb = 1 if cs is not None else 2
        extra = {"image_only_indicator": torch.zeros(nb, tl, device=randn.device), "num_video_frames": tl}
        if vs is not None:
            tc = vs.time_context(c, uc)                       # [2, M, ctx] in [uc; c] order
            extra["time_context"] = tc[cs.rank:cs.rank + 1] if cs is not None else tc

        def denoiser(inp, sigma, cond):
            return self.denoiser(self.model, inp, sigma, cond, **extra)

        sampler = copy.copy(self.sampler)
        guider = vs.shard_guider(self.sampler.guider) if vs is not None else self.sampler.guider
        sampler.guider = CfgSplitGuider(guider, cs) if cs is not None else guider
        if getattr(sampler, "noise_sampler", None) is not None:
            draw_full = sampler.noise_sampler

            def noise_sampler(x_local):
                # the unsharded draw, restricted to this rank's frames (see sample_views)
                return draw_full(x_local.new_empty((num_frames,) + tuple(x_local.shape[1:])))[frames]

            sampler.noise_sampler = noise_sampler
        try:
            unet.view_shard = vs
            z = sampler(denoiser, x, cond=c_l, uc=uc_l)       # this rank's sampling frames, identical across a CFG pair
            # decode blocks are the sampling blocks or nested inside them
            off = dvs.t0 - (vs.t0 if vs is not None else 0)
            assert 0 <= off and off + dvs.tl <= z.shape[0], "decode blocks must lie inside the sampling blocks"
            decoder.view_shard = dvs
            out = self.first_stage_model.decode(1.0 / self.scale_factor * z[off:off + dvs.tl].contiguous(),
                                                timesteps=dvs.tl)
            if os.environ.get("V3D_PEER_CHECK", "1") != "0":
                plan.check_status()      # a one-sided exchange that timed out invalidates the image: fail loudly
            return out
        finally:
            unet.view_shard = decoder.view_shard = None
