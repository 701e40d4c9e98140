"""TEST INFRASTRUCTURE: the smoke-sized engine the CPU suite runs through tests/emu_ops.py's stand-ins.

The product classes run unchanged: under `emu_ops.patched()` their one CUDA gate (`ops.require_current_device`) lets
CPU tensors through, so a whole `DiffusionEngine.sample_views` executes on a box without a GPU.
"""


def cpu_engine(num_frames: int, num_steps: int, min_cfg: float = 1.5, max_cfg: float = 3.5, width: int = 64,
               sampler: str = "EulerEDMSampler"):
    """The smoke-sized V3D_512 engine (model_channels / decoder ch = `width`) with seeded weights; its sampler is
    `v3d_b200.sampling.<sampler>` with V3D_512's schedule and guider."""
    from oracle import synth
    from v3d_b200 import engine, sampling

    cfg = engine.v3d_512_config(num_frames=num_frames, num_steps=num_steps, min_cfg=min_cfg, max_cfg=max_cfg)
    cfg["network_config"]["params"]["model_channels"] = width
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = width
    eng = engine.DiffusionEngine(**cfg).eval()
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    sd_u = synth.synth_state_dict(unet.param_shapes(), seed=11)
    sd_d = synth.synth_state_dict(dec.param_shapes(), seed=12)
    unet.load_state_dict(sd_u, strict=True)
    dec.load_state_dict(sd_d, strict=True)
    eng.sampler = getattr(sampling, sampler)(**cfg["sampler_config"]["params"])
    return eng, sd_u, sd_d
