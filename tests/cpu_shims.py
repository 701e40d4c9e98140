"""TEST INFRASTRUCTURE: subclasses that run the drop-in modules' host schedules on CPU tensors.

The product classes refuse non-CUDA tensors in `forward` / `__call__` (there is no CPU path).  These subclasses skip
exactly that check and call the same `_prepare` / `_run` / `_loop` the product path calls next, so that - with
tests/emu_ops.py patched over `v3d_b200.ops` - a whole `DiffusionEngine.sample_views` executes on a box without a GPU.
"""
import torch

from v3d_b200.decoder import VideoDecoder
from v3d_b200.encoder import Encoder
from v3d_b200.sampling import (DPMPP2MSampler, DPMPP2SAncestralSampler, EulerAncestralSampler, EulerEDMSampler,
                               HeunEDMSampler, LinearMultistepSampler)
from v3d_b200.unet import VideoUNet

CPU = torch.device("cpu")


class CpuUNet(VideoUNet):
    def forward(self, x, timesteps, context=None, y=None, time_context=None, num_video_frames=None,
                image_only_indicator=None):
        args, dims, _ = self._prepare(x, timesteps, context, y, time_context, num_video_frames, image_only_indicator)
        if self._packed is None:
            self._packed = self._pack(CPU)
        with torch.no_grad():
            return self._run(self._packed, *args, *dims, CPU)


class CpuDecoder(VideoDecoder):
    def forward(self, z, timesteps=None, **kwargs):
        B, _, H, W = z.shape
        T = int(timesteps) if timesteps else B
        if self._packed is None:
            self._packed = self._pack(CPU)
        with torch.no_grad():
            return self._run(self._packed, z, B, T, B // T, H, W)


class CpuEncoder(Encoder):
    def forward(self, x):
        if self._packed is None:
            self._packed = self._pack(CPU)
        with torch.no_grad():
            return self._run(self._packed, x)


class CpuEuler(EulerEDMSampler):
    __call__ = EulerEDMSampler._loop


class CpuHeun(HeunEDMSampler):
    __call__ = HeunEDMSampler._loop


class CpuEulerAncestral(EulerAncestralSampler):
    __call__ = EulerAncestralSampler._loop


class CpuDPMPP2SAncestral(DPMPP2SAncestralSampler):
    __call__ = DPMPP2SAncestralSampler._loop


class CpuDPMPP2M(DPMPP2MSampler):
    __call__ = DPMPP2MSampler._loop


class CpuLMS(LinearMultistepSampler):
    __call__ = LinearMultistepSampler._loop


CPU_SHIMS = {"EulerEDMSampler": CpuEuler, "HeunEDMSampler": CpuHeun, "EulerAncestralSampler": CpuEulerAncestral,
             "DPMPP2SAncestralSampler": CpuDPMPP2SAncestral, "DPMPP2MSampler": CpuDPMPP2M,
             "LinearMultistepSampler": CpuLMS}


def cpu_engine(num_frames: int, num_steps: int, min_cfg: float = 1.5, max_cfg: float = 3.5, width: int = 64,
               sampler: str = "EulerEDMSampler"):
    """The smoke-sized V3D_512 engine (model_channels / decoder ch = `width`) with seeded weights, on CPU shims; its
    sampler is the CPU shim of `sampler` with V3D_512's schedule and guider."""
    from oracle import synth
    from v3d_b200 import engine

    cfg = engine.v3d_512_config(num_frames=num_frames, num_steps=num_steps, min_cfg=min_cfg, max_cfg=max_cfg)
    cfg["network_config"]["params"]["model_channels"] = width
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = width
    eng = engine.DiffusionEngine(**cfg).eval()
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    sd_u = synth.synth_state_dict(unet.param_shapes(), seed=11)
    sd_d = synth.synth_state_dict(dec.param_shapes(), seed=12)
    unet.load_state_dict(sd_u, strict=True)
    dec.load_state_dict(sd_d, strict=True)
    unet.__class__, dec.__class__ = CpuUNet, CpuDecoder
    eng.sampler = CPU_SHIMS[sampler](**cfg["sampler_config"]["params"])
    return eng, sd_u, sd_d
