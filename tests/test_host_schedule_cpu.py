"""The HOST SCHEDULES of the drop-in VideoUNet / VideoDecoder, executed on CPU with tests/emu_ops.py standing in for
the C-ABI kernels (each stand-in restates one entry point's documented contract in torch).

  * schedule vs oracle: every buffer, stride, fused-epilogue operand, packing permutation and layout decision of
    `_run` must reproduce the reference arithmetic (oracle/ref_unet.py, oracle/ref_decoder.py) within the bf16
    tolerance of SURVEY.md App. C (rel-L2 <= 3e-2, cosine >= 0.999);
  * frame-sharded vs unsharded (2 ranks over gloo, uneven 3/2 split of T=5): the view-sharded schedule - halo'd
    GroupNorm buffers, K|V gather + row table, time-context rows, frame-offset positional embedding, the decoder's
    halo'd time_mix_conv - must agree with the unsharded schedule BIT FOR BIT (the stand-ins compute in fp64, so a
    result does not depend on the shape a BLAS call happens to see; the only arithmetic difference left is the
    summation order of the fp64 GroupNorm statistics, far below one bf16 ulp): rel-L2 <= 1e-6.
The CUDA kernels themselves are checked on the GPU (tests/test_kernels_gpu.py, test_parity_gpu.py,
test_viewshard_gpu.py); nothing here touches a device.
"""
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = str(Path(__file__).resolve().parent.parent)
sys.path.insert(0, str(Path(__file__).resolve().parent))

from framewise import assert_per_sample, per_sample  # noqa: E402

UNET_KW = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
               model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
               num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
               spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
               merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])
DEC_KW = dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=64,
              ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0, video_kernel_size=[3, 1, 1])

# (ops calls, sha256 of the call sequence: entry point, tensor shapes / dtypes / strides, scalar arguments) of the
# schedules below, recorded when the CPU suite still reached them through test-only subclasses and private `_run`
# calls: reached through forward() / sample_views they must launch exactly the same kernels with the same arguments.
# The frame-sharded UNet ranks and the deterministic-mode schedules were recorded before the time_stack, ResnetBlock
# and AttnBlock launches moved into shared helpers of KernelModule / FirstStage
LAUNCHES = {
    "decoder_t3": (191, "fe7e4dfc0dc41f632bc332fbde1e75648f008d1065bf40de9b4eccfd837c2500"),
    "decoder_t5_rank0_of_2": (191, "b94005a5eda61ebe3d9eb9821a5050dbeaa51585ca109cbfc03002d119c06daf"),
    "decoder_t5_rank1_of_2": (191, "362197510c94f182a28cc70c75f786bb7031eef8b2e514aba5910207a48a2988"),
    "encoder_64": (83, "53e76c186384f95d11aa98266b7ee34267fdf66d34dc8d76fd58391277a8703b"),
    "sample_views": (1639, "a705de874c93f680b818978057b2369e95b6a8faf19e3f13591e145a948a8300"),
    "unet_t5_rank0_of_2": (804, "534ce2260dbd140f9aa649c3f690d34b220f07eddf2bb8bb912b922bd73ce97b"),
    "unet_t5_rank1_of_2": (804, "ac58c24c2b31b690605c6f24babb1a1662f342e905c58ccac7e063d32aea7697"),
    "unet_t3_deterministic": (744, "63934c3e40e2a3a6eac4f8c5063471a720495992fe302626fca083a5c4023284"),
    "decoder_t3_deterministic": (191, "6c5145ab17ad9dd9a2155d483e1436f0b0bfe8b6e3509f0c54e4083ad8e8e1a6"),
}


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _cos(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-12)).item()


def _build_unet():
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**UNET_KW)
    sd = synth.synth_state_dict(net.param_shapes(), seed=11)
    net.load_state_dict(sd, strict=True)
    return net.eval(), sd


def _build_decoder():
    from oracle import synth
    from v3d_b200.decoder import VideoDecoder

    dec = VideoDecoder(**DEC_KW)
    sd = synth.synth_state_dict(dec.param_shapes(), seed=12)
    dec.load_state_dict(sd, strict=True)
    return dec.eval(), sd


def _unet_inputs(T, hw):
    from oracle import synth

    x, c, uc = synth.synth_inputs(T, hw)
    # make the frames' contexts differ so that "frame 0 of each video" matters for the temporal cross-attention
    g = torch.Generator().manual_seed(5)
    c = dict(c, crossattn=c["crossattn"] + 0.5 * torch.randn(T, 1, 1024, generator=g))
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    ts = torch.linspace(-0.5, 1.2, 2 * T)
    return xin, ts, ctx, y


def _unet(net, xin, ts, ctx, y, T):
    return net(xin, ts, ctx, y, num_video_frames=T, image_only_indicator=torch.zeros(xin.shape[0] // T, T))


def test_unet_host_schedule_matches_oracle():
    import emu_ops
    from oracle import ref_unet

    T, hw = 3, 16
    net, sd = _build_unet()
    xin, ts, ctx, y = _unet_inputs(T, hw)
    with emu_ops.patched():
        n0 = emu_ops.launch_count()
        out = _unet(net, xin, ts, ctx, y, T)
        launches = emu_ops.launch_count() - n0
    with torch.no_grad():
        ref = ref_unet.unet_forward(sd, ref_unet.UNetSpec(model_channels=64), xin, ts, ctx, y, T, torch.zeros(2, T))
    r, cs = _rel(out, ref), _cos(out, ref)
    print("unet schedule vs oracle: rel-L2", r, "cos", cs, "launches", launches)
    assert out.shape == ref.shape and torch.isfinite(out).all()
    assert r <= 3e-2 and cs >= 0.999, (r, cs)
    assert_per_sample("unet schedule", out, ref, 3e-2, 0.999)
    assert 600 < launches < 1400          # ~1.1k real launches; the stand-in counts a small_linear (prep + GEMM) once


def test_decoder_host_schedule_matches_oracle():
    import emu_ops
    from oracle import ref_decoder

    T, hw = 3, 8
    dec, sd = _build_decoder()
    z = torch.randn(T, 4, hw, hw, generator=torch.Generator().manual_seed(3))
    calls = []
    with emu_ops.patched(calls):
        out = dec(z, timesteps=T)
    with torch.no_grad():
        ref = ref_decoder.decoder_forward(sd, ref_decoder.DecoderSpec(ch=64), z, T)
    r, cs = _rel(out, ref), _cos(out, ref)
    print("decoder schedule vs oracle: rel-L2", r, "cos", cs, "launches", emu_ops.digest(calls))
    assert out.shape == ref.shape == (T, 3, 8 * hw, 8 * hw)
    assert r <= 3e-2 and cs >= 0.999, (r, cs)
    assert emu_ops.digest(calls) == LAUNCHES["decoder_t3"]


# ---------------------------------------------------------------------------------------------------------------
# frame-sharded schedule vs unsharded schedule, 2 ranks over gloo
# ---------------------------------------------------------------------------------------------------------------
def _shard_worker(rank: int, world: int, port: int, T: int, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    import emu_ops
    from v3d_b200.viewshard import ViewShard

    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    vs = ViewShard.create(T)
    res = {"rank": rank, "block": (vs.t0, vs.tl)}
    pick = torch.cat([torch.arange(vs.t0, vs.t0 + vs.tl), T + torch.arange(vs.t0, vs.t0 + vs.tl)])
    calls, ucalls = [], []
    with emu_ops.patched():
        net, _ = _build_unet()
        xin, ts, ctx, y = _unet_inputs(T, 16)
        full = _unet(net, xin, ts, ctx, y, T)
        tc = torch.stack([ctx[0], ctx[T]])                               # frame 0 of the uc and the c video
        net.view_shard = vs
        try:
            with emu_ops.patched(ucalls):
                part = net(xin[pick], ts[pick], ctx[pick], y[pick], time_context=tc, num_video_frames=vs.tl,
                           image_only_indicator=torch.zeros(2, vs.tl))
        finally:
            net.view_shard = None
        res["unet_launches"] = emu_ops.digest(ucalls)
        res["unet_rel"] = _rel(part, full[pick])
        res["unet_exchanges"] = dict(vs.exchanges)

        dec, _ = _build_decoder()
        z = torch.randn(T, 4, 8, 8, generator=torch.Generator().manual_seed(3))   # the AttnBlock needs h*w % 64 == 0
        full_d = dec(z, timesteps=T)
        dec.view_shard = vs
        try:
            with emu_ops.patched(calls):
                part_d = dec(z[vs.frames].contiguous(), timesteps=vs.tl)
        finally:
            dec.view_shard = None
        res["dec_launches"] = emu_ops.digest(calls)
        res["dec_rel"] = _rel(part_d, full_d[vs.frames])
        res["dec_gathered_rel"] = _rel(vs.gather_frames(part_d), full_d)
    q.put(res)
    dist.barrier()
    dist.destroy_process_group()


def test_view_sharded_host_schedule_matches_unsharded_gloo():
    from mp_util import run_workers

    world, T = 2, 5
    res = sorted(run_workers(_shard_worker, world, (T,), timeout=900), key=lambda r: r["rank"])
    print(res)
    assert [r["block"] for r in res] == [(0, 3), (3, 2)]
    for r in res:
        assert r["unet_rel"] <= 1e-6, r
        assert r["dec_rel"] <= 1e-6 and r["dec_gathered_rel"] <= 1e-6, r
        assert r["dec_launches"] == LAUNCHES[f"decoder_t5_rank{r['rank']}_of_2"], r
        assert r["unet_launches"] == LAUNCHES[f"unet_t5_rank{r['rank']}_of_2"], r
        # UNet: 22 VideoResBlocks x (2 statistics all-reduces + 2 halo exchanges), 16 transformers x 1 K|V gather
        assert r["unet_exchanges"] == {"gn_allreduce": 44, "halo": 44, "kv_allgather": 16}, r


def test_encoder_host_schedule_matches_oracle():
    """SURVEY 8(f)-1: the native first-stage Encoder's schedule (asymmetric-pad stride-2 im2row, mid AttnBlock)."""
    import emu_ops
    from oracle import ref_encoder, synth
    from v3d_b200.encoder import Encoder

    enc = Encoder(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=64, ch_mult=[1, 2, 4, 4],
                  num_res_blocks=2, attn_resolutions=[], dropout=0.0, attn_type="vanilla")
    sd = synth.synth_state_dict(enc.param_shapes(), seed=13)
    enc.load_state_dict(sd, strict=True)
    x = torch.randn(2, 3, 64, 64, generator=torch.Generator().manual_seed(4))
    calls = []
    with emu_ops.patched(calls):
        out = enc.eval()(x)
    with torch.no_grad():
        ref = ref_encoder.encoder_forward(sd, ref_encoder.EncoderSpec(ch=64), x)
    r, cs = _rel(out, ref), _cos(out, ref)
    print("encoder schedule vs oracle: rel-L2", r, "cos", cs, "launches", emu_ops.digest(calls))
    assert out.shape == ref.shape == (2, 8, 8, 8)
    assert r <= 3e-2 and cs >= 0.999, (r, cs)
    assert emu_ops.digest(calls) == LAUNCHES["encoder_64"]


# ---------------------------------------------------------------------------------------------------------------
# the whole hot path (DiffusionEngine.sample_views: sampler loop + CFG + denoiser + UNet + decode) on CPU
# ---------------------------------------------------------------------------------------------------------------
def test_sample_views_host_path_matches_oracle():
    """What __graft_entry__.smoke() checks on the GPU, with the kernels replaced by their CPU stand-ins: 2 Euler-EDM
    steps with per-frame CFG scales through the drop-in sampler / guider / denoiser / wrapper / UNet, then the decode."""
    import cpu_shims
    import emu_ops
    from oracle import ref_decoder, ref_sampling, ref_unet, synth

    T, hw, steps = 3, 8, 2
    eng, sd_u, sd_d = cpu_shims.cpu_engine(T, steps)
    x, c, uc = synth.synth_inputs(T, hw)
    calls = []
    with emu_ops.patched(calls):
        frames = eng.sample_views(x.clone(), c, uc, num_frames=T)
    assert emu_ops.digest(calls) == LAUNCHES["sample_views"], emu_ops.digest(calls)
    u8 = emu_ops.frames_nchw_to_u8(frames, torch.empty(T, 8 * hw, 8 * hw, 3, dtype=torch.uint8))
    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    with torch.no_grad():
        z_ref = ref_sampling.euler_edm_sample(
            lambda i, s, cc: ref_sampling.denoiser(
                lambda xx, tt, cond, **kw: ref_unet.openai_wrapper(sd_u, ref_unet.UNetSpec(model_channels=64), xx, tt,
                                                                   cond, **kw), i, s, cc, **extra),
            x.clone(), c, uc, steps, ref_sampling.guider_scale(1.5, 3.5, T), T)
        img_ref = ref_decoder.decode_first_stage(sd_d, ref_decoder.DecoderSpec(ch=64), z_ref, n_samples_a_time=T)
    r, cs = _rel(frames, img_ref), _cos(frames, img_ref)
    print("sample_views host path vs oracle: rel-L2", r, "cos", cs)
    assert frames.shape == img_ref.shape == (T, 3, 8 * hw, 8 * hw) and torch.isfinite(frames).all()
    assert r <= 5e-2 and cs >= 0.998, (r, cs)                      # the bound smoke() applies on the GPU
    ref_u8 = (torch.clamp((frames + 1.0) / 2.0, 0.0, 1.0) * 255).to(torch.uint8).permute(0, 2, 3, 1)
    assert torch.equal(u8, ref_u8)                                  # V3D_512.py:286-303 wire format


def _engine_shard_worker(rank: int, world: int, port: int, T: int, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    import cpu_shims
    import emu_ops
    from oracle import synth
    from v3d_b200.viewshard import ViewShard

    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    vs = ViewShard.create(T)
    eng, _, _ = cpu_shims.cpu_engine(T, 2)
    x, c, uc = synth.synth_inputs(T, 8)
    g = torch.Generator().manual_seed(5)
    c = dict(c, crossattn=c["crossattn"] + 0.5 * torch.randn(T, 1, 1024, generator=g))   # frames differ
    with emu_ops.patched():
        ref = eng.sample_views(x.clone(), c, uc, num_frames=T)
        mine = eng.sample_views(x.clone(), c, uc, num_frames=T, view_shard=vs)
        gathered = vs.gather_frames(mine)
    q.put({"rank": rank, "block": (vs.t0, vs.tl), "local_rel": _rel(mine, ref[vs.frames]),
           "gathered_rel": _rel(gathered, ref), "shape": tuple(mine.shape), "exchanges": dict(vs.exchanges),
           "guider_frames": eng.sampler.guider.num_frames, "hooks_cleared":
               eng.model.diffusion_model.view_shard is None and eng.first_stage_model.decoder.view_shard is None})
    dist.barrier()
    dist.destroy_process_group()


def test_view_sharded_sample_views_matches_unsharded_gloo():
    """DiffusionEngine.sample_views(view_shard=...) end to end (cond slicing, guider slice, time context, sampler
    state per block, sharded UNet x 2 steps x CFG, sharded decode, frame gather) == the unsharded call, bit for bit."""
    from mp_util import run_workers

    world, T = 2, 5
    res = sorted(run_workers(_engine_shard_worker, world, (T,), timeout=900), key=lambda r: r["rank"])
    print(res)
    assert [r["block"] for r in res] == [(0, 3), (3, 2)]
    for r in res:
        assert r["shape"] == (r["block"][1], 3, 64, 64)
        assert r["local_rel"] <= 1e-6 and r["gathered_rel"] <= 1e-6, r
        assert r["guider_frames"] == T and r["hooks_cleared"], r        # the engine's own sampler is left untouched
        # 2 EDM steps x one CFG-batched forward: 2 x (44 + 44 + 16); decode: 28 norms, 29 halos; one frame gather
        assert r["exchanges"] == {"gn_allreduce": 88 + 28, "halo": 88 + 29, "kv_allgather": 32, "frame_gather": 1}, r


@pytest.mark.parametrize("tag", ["edm_small", "edm_small_heun", "edm_small_central", "edm_small_vanilla"])
def test_sampler_variants_host_path_match_reference_golden(tag):
    """EulerEDMSampler / HeunEDMSampler x LinearPrediction / CentralPrediction / VanillaCFG guiders (SURVEY 8(f)-3)
    through the drop-in classes with the kernels' CPU stand-ins, against the REAL reference's outputs
    (tests/golden/edm_small*.pt, 3 steps at latent 32; bound = the GPU parity tolerance, rel-L2 <= 3e-2)."""
    import json

    import emu_ops
    from oracle import synth
    from v3d_b200 import sampling
    from v3d_b200.unet import VideoUNet

    gold_dir = Path(ROOT) / "tests" / "golden"
    manifest = json.loads((gold_dir / "MANIFEST.json").read_text())
    m, mu = manifest[tag], manifest["unet_small"]
    gold = torch.load(gold_dir / f"{tag}.pt")
    net = VideoUNet(**dict(UNET_KW, model_channels=mu["model_channels"]))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=mu["weight_seed"]), strict=True)
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    base = "v3d_b200.sgm.modules.diffusionmodules."
    kind = m.get("guider", "linear")
    guider = {"linear": {"target": base + "guiders.LinearPredictionGuider",
                         "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}},
              "central": {"target": base + "guiders.CentralPredictionGuider",
                          "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}},
              "vanilla": {"target": base + "guiders.VanillaCFG", "params": {"scale": m.get("vanilla_scale", 2.5)}}}[kind]
    sampler = getattr(sampling, m.get("sampler", "EulerEDMSampler"))(num_steps=m["num_steps"],
        discretization_config={"target": base + "discretizer.EDMDiscretization", "params": {"sigma_max": m["sigma_max"]}},
        guider_config=guider)
    den = sampling.Denoiser({"target": base + "denoiser_scaling.VScalingWithEDMcNoise"})
    model = sampling.OpenAIWrapper(net.eval())
    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    x0 = x.clone()
    with emu_ops.patched():
        n0 = emu_ops.launch_count()
        out = sampler(lambda i, s, cc: den(model, i, s, cc, **extra), x0, cond=c, uc=uc)
        launches = emu_ops.launch_count() - n0
    r = _rel(out, gold["out"])
    print(tag, "host path vs reference golden: rel-L2", r, "launches", launches)
    assert not torch.equal(x0, x)                       # the caller's noise is scaled in place, like sampling.py:50
    # Three Heun steps down from sigma = 700 are an unstable integration (reference output std 14 against 1.4 for
    # Euler): they amplify the network's bf16 rounding (measured 9e-2 with the stand-ins) although the sampler logic
    # is exact (next test).  The Euler variants stay inside the usual parity bound.
    assert r <= (2e-1 if "heun" in tag else 3e-2), (tag, r)


@pytest.mark.parametrize("tag", ["edm_small", "edm_small_heun", "edm_small_central", "edm_small_vanilla"])
def test_sampler_variants_logic_exact_with_fp32_network(tag):
    """The drop-in samplers / guiders / denoiser (their elementwise kernels as CPU stand-ins) around the ORACLE's
    fp32 UNet reproduce the real reference's outputs to fp32 rounding: schedule, CFG batch order, per-frame scales,
    Heun's second evaluation and its first-order last step are all exactly the reference's."""
    import json

    import emu_ops
    from oracle import ref_unet, synth
    from v3d_b200 import sampling

    gold_dir = Path(ROOT) / "tests" / "golden"
    manifest = json.loads((gold_dir / "MANIFEST.json").read_text())
    m, mu = manifest[tag], manifest["unet_small"]
    gold = torch.load(gold_dir / f"{tag}.pt")
    spec = ref_unet.UNetSpec(model_channels=mu["model_channels"])
    sd = synth.synth_state_dict(ref_unet.unet_param_shapes(spec), seed=mu["weight_seed"])
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    base = "v3d_b200.sgm.modules.diffusionmodules."
    kind = m.get("guider", "linear")
    guider = {"linear": {"target": base + "guiders.LinearPredictionGuider",
                         "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}},
              "central": {"target": base + "guiders.CentralPredictionGuider",
                          "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}},
              "vanilla": {"target": base + "guiders.VanillaCFG", "params": {"scale": m.get("vanilla_scale", 2.5)}}}[kind]
    sampler = getattr(sampling, m.get("sampler", "EulerEDMSampler"))(num_steps=m["num_steps"],
        discretization_config={"target": base + "discretizer.EDMDiscretization", "params": {"sigma_max": m["sigma_max"]}},
        guider_config=guider)
    den = sampling.Denoiser({"target": base + "denoiser_scaling.VScalingWithEDMcNoise"})

    class OracleNet(torch.nn.Module):
        def forward(self, xx, t, cond, **kw):
            with torch.no_grad():
                return ref_unet.openai_wrapper(sd, spec, xx, t, cond, **kw)

    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    with emu_ops.patched():
        out = sampler(lambda i, s, cc: den(OracleNet(), i, s, cc, **extra), x.clone(), cond=c, uc=uc)
    r = _rel(out, gold["out"])
    print(tag, "sampler logic with fp32 network vs reference golden: rel-L2", r)
    assert r <= 1e-5, (tag, r)


def test_conditioning_host_path_matches_reference_golden():
    """SURVEY 8(f)-1: GeneralConditioner / ConcatTimestepEmbedderND / get_batch assembly (scripts/pub/V3D_512.py:247-267)
    through the drop-in module with v3d_timestep_embedding's stand-in, against the real reference's (c, uc)."""
    import emu_ops
    from v3d_b200 import conditioning

    gold = torch.load(Path(ROOT) / "tests" / "golden" / "conditioning.pt")
    with emu_ops.patched():
        cond = conditioning.GeneralConditioner(conditioning.V3D_512_EMB_MODELS)
        c, uc = conditioning.assemble_v3d_conditioning(cond, gold["clip_emb"], gold["latent"], 6.0, 127.0, 0.02, 18)
    assert torch.allclose(c["vector"], gold["c"]["vector"], atol=2e-6) and torch.equal(uc["vector"], c["vector"])
    assert torch.equal(c["crossattn"], gold["c"]["crossattn"]) and torch.equal(uc["concat"], gold["uc"]["concat"])
    assert torch.equal(c["concat"], gold["c"]["concat"]) and torch.equal(uc["crossattn"], gold["uc"]["crossattn"])


def test_single_rank_view_shard_schedule_equals_unsharded():
    """world = 1: the frame-sharded schedule (halo'd GroupNorm buffers with zero halos, split-KV attention over its own
    frames, statistics rescaled by 1, halo'd time_mix_conv) needs no process group and must equal the dense schedule."""
    import cpu_shims
    import emu_ops
    from oracle import synth
    from v3d_b200.viewshard import ViewShard

    T = 3
    eng, _, _ = cpu_shims.cpu_engine(T, 2)
    x, c, uc = synth.synth_inputs(T, 8)
    vs = ViewShard(num_frames=T, rank=0, world=1)
    with emu_ops.patched():
        ref = eng.sample_views(x.clone(), c, uc, num_frames=T)
        one = eng.sample_views(x.clone(), c, uc, num_frames=T, view_shard=vs)
    assert torch.equal(one, ref)
    assert vs.exchanges["halo"] == 2 * 44 + 29 and vs.exchanges["kv_allgather"] == 32


def _plan_worker(rank: int, world: int, port: int, T: int, mode: str, q, sampler: str = "euler"):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    import cpu_shims
    import emu_ops
    from oracle import synth
    from v3d_b200.viewshard import ShardPlan

    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    plan = ShardPlan.create(T, mode)
    eng, _, _ = cpu_shims.cpu_engine(T, 2, sampler="HeunEDMSampler" if sampler == "heun" else "EulerEDMSampler")
    x, c, uc = synth.synth_inputs(T, 8)
    g = torch.Generator().manual_seed(5)
    c = dict(c, crossattn=c["crossattn"] + 0.5 * torch.randn(T, 1, 1024, generator=g))
    with emu_ops.patched():
        ref = eng.sample_views(x.clone(), c, uc, num_frames=T)
        mine = eng.sample_views(x.clone(), c, uc, num_frames=T, shard=plan)
        gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "decode_block": (plan.decode.t0, plan.decode.tl), "finite": bool(torch.isfinite(mine).all()),
           "local_rel": _rel(mine, ref[plan.decode.frames]), "gathered_rel": _rel(gathered, ref),
           "plan": plan.describe()})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode,world,T", [("cfg", 2, 4), ("cfg+views", 4, 5)])
def test_cfg_split_plans_match_unsharded_gloo(mode, world, T):
    """ShardPlan 'cfg' (the [uc; c] halves on two ranks, one all-gather per network evaluation, decode on two frame
    blocks) and 'cfg+views' (frame blocks x CFG pairs, decode blocks nested in the sampling blocks) reproduce the
    unsharded DiffusionEngine.sample_views bit for bit."""
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker, world, (T, mode), timeout=900), key=lambda r: r["rank"])
    print(res)
    covered = []
    for r in res:
        covered += list(range(r["decode_block"][0], sum(r["decode_block"])))
        assert r["local_rel"] <= 1e-6 and r["gathered_rel"] <= 1e-6, r
        assert r["plan"]["exchanges"]["cfg_gather"] == 2              # 2 EDM steps x one network evaluation
    assert covered == list(range(T))
    if mode == "cfg":
        assert all("halo" not in r["plan"]["exchanges"] for r in res)  # the UNet runs dense on each CFG half
        assert [r["plan"]["cfg_rank"] for r in res] == [0, 1]
    else:
        assert [r["plan"]["sample_blocks"] for r in res] == [[(0, 3), (3, 2)]] * 4
        assert [r["decode_block"] for r in res] == [(0, 2), (2, 1), (3, 1), (4, 1)]


def _plan_worker_heun(rank, world, port, T, mode, q):
    _plan_worker(rank, world, port, T, mode, q, sampler="heun")


def test_cfg_split_with_heun_sampler_matches_unsharded_gloo():
    """HeunEDMSampler evaluates the network twice per step (once on the last, first-order step): the CFG-pair split
    gathers the halves after every evaluation - 3 gathers for 2 steps - and still reproduces the unsharded result."""
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker_heun, 2, (4, "cfg"), timeout=900), key=lambda r: r["rank"])
    print(res)
    for r in res:
        assert r["finite"] and r["local_rel"] <= 1e-6 and r["gathered_rel"] <= 1e-6, r
        assert r["plan"]["exchanges"]["cfg_gather"] == 3


@pytest.mark.parametrize("tag", ["encoder_small", "encoder_full"])
def test_encoder_host_schedule_matches_reference_golden(tag):
    """The native Encoder's schedule + DiagonalGaussianRegularizer against the REAL reference's moments and sampled
    latent (tests/golden/encoder_*.pt), with the noise the reference drew."""
    import json

    import emu_ops
    from oracle import ref_encoder, synth
    from v3d_b200.encoder import DiagonalGaussianRegularizer, Encoder

    gold_dir = Path(ROOT) / "tests" / "golden"
    m = json.loads((gold_dir / "MANIFEST.json").read_text())[tag]
    gold = torch.load(gold_dir / f"{tag}.pt")
    enc = Encoder(attn_type="vanilla", double_z=True, z_channels=4, resolution=m["image_hw"], in_channels=3, out_ch=3,
                  ch=m["ch"], ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0)
    sd = synth.synth_state_dict(ref_encoder.encoder_param_shapes(ref_encoder.EncoderSpec(ch=m["ch"])),
                                seed=m["weight_seed"])
    enc.load_state_dict(sd)
    with emu_ops.patched():
        mom = enc.eval()(gold["x"])
    z, _ = DiagonalGaussianRegularizer()(mom, noise=gold["noise"])
    r, rz = _rel(mom, gold["moments"]), _rel(z, gold["z"])
    print(tag, "moments rel-L2", r, "z rel-L2", rz)
    assert r <= 3e-2 and rz <= 3e-2


@pytest.mark.parametrize("tag", ["unet_small", "unet_small_t18", "unet_full"])
def test_unet_host_schedule_matches_reference_golden_with_block_taps(tag):
    """The CPU twin of tests/test_parity_gpu.py::test_unet_forward_matches_reference: output AND per-block taps of the
    UNet schedule against the REAL reference's golden outputs (same bounds: taps 2e-2, output 3e-2 / cosine 0.999)."""
    import json

    import emu_ops
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    gold_dir = Path(ROOT) / "tests" / "golden"
    m = json.loads((gold_dir / "MANIFEST.json").read_text())[tag]
    gold = torch.load(gold_dir / f"{tag}.pt")
    net = VideoUNet(**dict(UNET_KW, model_channels=m["model_channels"]))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=m["weight_seed"]), strict=True)
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    taps = {k[4:]: None for k in gold if k.startswith("tap:")}
    net.debug_taps = taps
    with emu_ops.patched():
        out = _unet(net.eval(), xin, gold["timesteps"], ctx, y, T)
    report = [(name, _rel(val[[0, T]][:, ::8], gold["tap:" + name])) for name, val in taps.items()]
    r, cs = _rel(out, gold["out"]), _cos(out, gold["out"])
    print(tag, "rel-L2", r, "cos", cs, "worst tap", max(report, key=lambda t: t[1]))
    assert all(v is not None for v in taps.values()) and len(report) >= 4
    assert all(e <= 2e-2 for _, e in report), report
    assert r <= 3e-2 and cs >= 0.999
    # per sample the taps are only reported: the deepest tap (output_blocks.11.1) of the unconditional sample 0 is at
    # rel-L2 2.1e-2 (unet_small) and 2.2e-2 (unet_small_t18) with these fp64 stand-ins, the accumulated bf16 error of
    # the path itself; tests/test_unet_blocks_fp64_gpu.py bounds every block's own share in fp64
    print(tag, "worst per-sample tap rel-L2", max((max(r for _, r, _ in per_sample(v[[0, T]][:, ::8], gold["tap:" + n])), n)
                                                  for n, v in taps.items()))
    print(tag, "worst sample (rel-L2, cosine)", assert_per_sample(tag, out, gold["out"], 3e-2, 0.999))


@pytest.mark.parametrize("tag", ["decoder_small", "decoder_small_2videos", "decoder_full"])
def test_decoder_host_schedule_matches_reference_golden(tag):
    """Decoder schedule vs the REAL reference's decode; `decoder_small_2videos` decodes two videos in one batch
    (nb = 2: the 3-D norms and temporal convs must not couple them)."""
    import json

    import emu_ops
    from oracle import synth
    from v3d_b200.decoder import VideoDecoder

    gold_dir = Path(ROOT) / "tests" / "golden"
    m = json.loads((gold_dir / "MANIFEST.json").read_text())[tag]
    gold = torch.load(gold_dir / f"{tag}.pt")
    dec = VideoDecoder(**dict(DEC_KW, ch=m["ch"]))
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=m["weight_seed"]), strict=True)
    z = gold["z"] / 0.18215
    B, T = z.shape[0], m["T"]
    with emu_ops.patched():
        out = dec.eval()(z, timesteps=T)
    r, cs = _rel(out, gold["out"]), _cos(out, gold["out"])
    print(tag, "rel-L2", r, "cos", cs)
    assert out.shape == gold["out"].shape and r <= 3e-2 and cs >= 0.999


@pytest.mark.parametrize("T,hw", [(1, 8), (2, 24), (3, 40)])
def test_unet_host_schedule_edge_geometries_match_oracle(T, hw):
    """Edge cases of the schedule against the oracle: a single frame (temporal attention / (3,1,1) convs / 3-D norms
    over T = 1), and latents that do not tile into power-of-two boxes (24 -> 12 -> 6 -> 3 and 40 -> 20 -> 10 -> 5: every
    3x3 convolution then takes the explicit im2row path instead of the TMA gather)."""
    import emu_ops
    from oracle import ref_unet
    from v3d_b200.unet import conv_tiles_ok

    net, sd = _build_unet()
    xin, ts, ctx, y = _unet_inputs(T, hw)
    with emu_ops.patched():
        out = _unet(net, xin, ts, ctx, y, T)
    with torch.no_grad():
        ref = ref_unet.unet_forward(sd, ref_unet.UNetSpec(model_channels=64), xin, ts, ctx, y, T, torch.zeros(2, T))
    r, cs = _rel(out, ref), _cos(out, ref)
    print((T, hw), "rel-L2", r, "cos", cs, "tma-gather geometry:", conv_tiles_ok(hw, hw))
    assert out.shape == ref.shape and torch.isfinite(out).all()
    assert r <= 3e-2 and cs >= 0.999, (r, cs)
    assert_per_sample(f"T={T} hw={hw}", out, ref, 3e-2, 0.999)
    if hw in (24, 40):
        assert not conv_tiles_ok(hw, hw)


def test_unet_rejects_latents_whose_skips_would_not_line_up():
    """12 -> 6 -> 3 -> 2 -> (x2) 4 != 3: the reference dies in th.cat (video_model.py:483); the drop-in raises before
    launching anything (the kernels take raw pointers: a mismatched skip would be an out-of-bounds read)."""
    import emu_ops

    net, _ = _build_unet()
    xin, ts, ctx, y = _unet_inputs(2, 12)
    calls = []
    with pytest.raises(RuntimeError, match="divisible by 8"), emu_ops.patched(calls):
        _unet(net, xin, ts, ctx, y, 2)
    assert calls == []


def test_non_square_latents_match_oracle():
    """H != W through all three schedules (the reference handles any size divisible by the down-sampling factor): a
    swapped height / width anywhere in the conv geometry, the upsample or the layout conversions shows up here."""
    import emu_ops
    from oracle import ref_decoder, ref_encoder, ref_unet, synth
    from v3d_b200.encoder import Encoder

    g = torch.Generator().manual_seed(9)
    T, H, W = 2, 16, 24
    net, sd = _build_unet()
    xin = torch.randn(2 * T, 8, H, W, generator=g)
    ts = torch.linspace(-0.5, 1.0, 2 * T)
    ctx = torch.randn(2 * T, 1, 1024, generator=g)
    y = torch.randn(2 * T, 768, generator=g)
    with emu_ops.patched():
        out = _unet(net, xin, ts, ctx, y, T)
    with torch.no_grad():
        ref = ref_unet.unet_forward(sd, ref_unet.UNetSpec(model_channels=64), xin, ts, ctx, y, T, torch.zeros(2, T))
    r = _rel(out, ref)
    print("unet 16x24 rel-L2", r)
    assert out.shape == ref.shape == (2 * T, 4, H, W) and r <= 3e-2 and _cos(out, ref) >= 0.999

    dec, sdd = _build_decoder()
    z = torch.randn(3, 4, 8, 16, generator=g)
    with emu_ops.patched():
        out = dec(z, timesteps=3)
    with torch.no_grad():
        ref = ref_decoder.decoder_forward(sdd, ref_decoder.DecoderSpec(ch=64), z, 3)
    r = _rel(out, ref)
    print("decoder 8x16 rel-L2", r)
    assert out.shape == ref.shape == (3, 3, 64, 128) and r <= 3e-2 and _cos(out, ref) >= 0.999

    enc = Encoder(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=64, ch_mult=[1, 2, 4, 4],
                  num_res_blocks=2, attn_resolutions=[], dropout=0.0, attn_type="vanilla")
    sde = synth.synth_state_dict(enc.param_shapes(), seed=13)
    enc.load_state_dict(sde, strict=True)
    x = torch.randn(1, 3, 64, 128, generator=g)
    with emu_ops.patched():
        out = enc.eval()(x)
    with torch.no_grad():
        ref = ref_encoder.encoder_forward(sde, ref_encoder.EncoderSpec(ch=64), x)
    r = _rel(out, ref)
    print("encoder 64x128 rel-L2", r)
    assert out.shape == ref.shape == (1, 8, 8, 16) and r <= 3e-2 and _cos(out, ref) >= 0.999


def test_decode_first_stage_chunking_matches_oracle():
    """en_and_decode_n_samples_a_time < T: every chunk is decoded as its own short video (temporal convs zero-pad at
    chunk edges, video_diffusion.py:182-210) - chunks of 2 + 1 frames vs the oracle's chunked decode, and != one chunk."""
    import cpu_shims
    import emu_ops
    from oracle import ref_decoder

    eng, _, sd_d = cpu_shims.cpu_engine(3, 2)
    z = torch.randn(3, 4, 8, 8, generator=torch.Generator().manual_seed(2)) * 0.18215
    with emu_ops.patched():
        eng.en_and_decode_n_samples_a_time = 2
        chunked = eng.decode_first_stage(z)
        eng.en_and_decode_n_samples_a_time = 3
        whole = eng.decode_first_stage(z)
    with torch.no_grad():
        ref = ref_decoder.decode_first_stage(sd_d, ref_decoder.DecoderSpec(ch=64), z, n_samples_a_time=2)
    assert chunked.shape == ref.shape == (3, 3, 64, 64)
    assert _rel(chunked, ref) <= 3e-2 and _cos(chunked, ref) >= 0.999
    assert _rel(chunked, whole) > 1e-2          # the chunk boundary matters, exactly as in the reference


def test_do_sample_call_sequence_runs_against_the_drop_in_engine():
    """SURVEY 8(f)-3, second caller: the body of sgm/inference/helpers.py:do_sample (:121-170) touches
    model.ema_scope(), model.conditioner.get_unconditional_conditioning, model.denoiser(model.model, ...), the sampler
    call and model.decode_first_stage - replayed here statement by statement against the drop-in engine (kernels as
    CPU stand-ins) and compared with sample_views on the same conditioning."""
    import math

    import cpu_shims
    import emu_ops
    from v3d_b200 import conditioning

    T, hw = 3, 8
    eng, _, _ = cpu_shims.cpu_engine(T, 2)
    eng.conditioner = conditioning.GeneralConditioner(conditioning.V3D_512_EMB_MODELS)
    g = torch.Generator().manual_seed(11)
    clip_emb, latent = torch.randn(1, 1, 1024, generator=g), torch.randn(1, 4, hw, hw, generator=g)
    with emu_ops.patched(), torch.no_grad(), eng.ema_scope():
        c, uc = conditioning.assemble_v3d_conditioning(eng.conditioner, clip_emb, latent, 6.0, 127.0, 0.02, T)
        num_samples = [T]
        for k in c:                                                    # helpers.py:143-147
            if not k == "crossattn":
                c[k], uc[k] = map(lambda y: y[k][: math.prod(num_samples)], (c, uc))
        additional_model_inputs = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
        randn = torch.randn((T, 4, hw, hw), generator=g)

        def denoiser(input, sigma, cc):                                # helpers.py:156-159
            return eng.denoiser(eng.model, input, sigma, cc, **additional_model_inputs)

        samples_z = eng.sampler(denoiser, randn.clone(), cond=c, uc=uc)
        eng.en_and_decode_n_samples_a_time = T
        samples_x = eng.decode_first_stage(samples_z)
        samples = torch.clamp((samples_x + 1.0) / 2.0, min=0.0, max=1.0)
        ref = eng.sample_views(randn.clone(), c, uc, num_frames=T)
    assert samples.shape == (T, 3, 8 * hw, 8 * hw) and float(samples.min()) >= 0.0 and float(samples.max()) <= 1.0
    assert torch.equal(samples_x, ref)


def test_encode_first_stage_matches_oracle():
    """DiffusionEngine.encode_first_stage (video_diffusion.py:212-237) with the native Encoder: chunked encode of a
    [b, t, c, h, w] video, posterior sample drawn on the CPU generator like the reference (distributions.py:37-41),
    times scale_factor - against the oracle encoder + Gaussian sample with the same draws."""
    import emu_ops
    from oracle import ref_encoder, synth
    from v3d_b200 import engine

    cfg = engine.v3d_512_config(num_frames=2, num_steps=1)
    cfg["network_config"]["params"]["model_channels"] = 64
    fs = cfg["first_stage_config"]["params"]
    fs["decoder_config"]["params"]["ch"] = 64
    fs["encoder_config"] = {"target": "v3d_b200.sgm.modules.diffusionmodules.model.Encoder",
                            "params": dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256,
                                           in_channels=3, out_ch=3, ch=64, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                                           attn_resolutions=[], dropout=0.0)}
    fs["regularizer_config"] = {"target": "v3d_b200.encoder.DiagonalGaussianRegularizer", "params": {"sample": True}}
    eng = engine.DiffusionEngine(**cfg).eval()
    enc = eng.first_stage_model.encoder
    assert enc is not None, "native encoder not built"
    sd = synth.synth_state_dict(enc.param_shapes(), seed=21)
    enc.load_state_dict(sd, strict=True)
    x = torch.randn(1, 3, 3, 64, 64, generator=torch.Generator().manual_seed(6))     # [b, t, c, h, w]
    eng.en_and_decode_n_samples_a_time = 2                                            # chunks of 2 + 1 frames
    with emu_ops.patched():
        torch.manual_seed(77)
        z = eng.encode_first_stage(x)
    torch.manual_seed(77)
    with torch.no_grad():
        flat = x.reshape(-1, 3, 64, 64)
        zs = []
        for chunk in (flat[:2], flat[2:]):
            mom = ref_encoder.encoder_forward(sd, ref_encoder.EncoderSpec(ch=64), chunk)
            zs.append(ref_encoder.gaussian_sample(mom, torch.randn(chunk.shape[0], 4, 8, 8)))
        ref = 0.18215 * torch.cat(zs)
    r = _rel(z, ref)
    print("encode_first_stage vs oracle: rel-L2", r)
    assert z.shape == ref.shape == (3, 4, 8, 8) and r <= 3e-2


def test_views_from_image_matches_oracle_composition():
    """sample_one from the conditioning image to the decoded views (V3D_512.py:235-285), CLIP embedding given: native
    encoder -> cond_aug noise -> conditioner + per-frame repeat -> latent noise -> sampler + decode, with the reference's
    order of random draws - against the same composition of the oracle's pieces under the same seed."""
    import emu_ops
    from oracle import ref_conditioning, ref_decoder, ref_encoder, ref_sampling, ref_unet, synth
    from v3d_b200 import conditioning, engine, pipeline

    T, steps, side = 3, 2, 64
    cfg = engine.v3d_512_config(num_frames=T, num_steps=steps, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    fs = cfg["first_stage_config"]["params"]
    fs["decoder_config"]["params"]["ch"] = 64
    fs["encoder_config"] = {"target": "v3d_b200.sgm.modules.diffusionmodules.model.Encoder",
                            "params": dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256,
                                           in_channels=3, out_ch=3, ch=64, ch_mult=[1, 2, 4, 4], num_res_blocks=2,
                                           attn_resolutions=[], dropout=0.0)}
    fs["regularizer_config"] = {"target": "v3d_b200.encoder.DiagonalGaussianRegularizer", "params": {"sample": True}}
    eng = engine.DiffusionEngine(**cfg).eval()
    eng.conditioner = conditioning.GeneralConditioner(conditioning.V3D_512_EMB_MODELS)
    unet, dec, enc = eng.model.diffusion_model, eng.first_stage_model.decoder, eng.first_stage_model.encoder
    sd_u = synth.synth_state_dict(unet.param_shapes(), seed=11)
    sd_d = synth.synth_state_dict(dec.param_shapes(), seed=12)
    sd_e = synth.synth_state_dict(enc.param_shapes(), seed=13)
    unet.load_state_dict(sd_u, strict=True)
    dec.load_state_dict(sd_d, strict=True)
    enc.load_state_dict(sd_e, strict=True)
    g = torch.Generator().manual_seed(31)
    image = torch.rand(1, 3, side, side, generator=g) * 2 - 1
    clip_emb = torch.randn(1, 1, 1024, generator=g)

    torch.manual_seed(23)
    with emu_ops.patched():
        frames = pipeline.views_from_image(eng, image, clip_emb, num_frames=T, fps_id=6, motion_bucket_id=127,
                                           cond_aug=0.02)
    torch.manual_seed(23)
    with torch.no_grad():
        mom = ref_encoder.encoder_forward(sd_e, ref_encoder.EncoderSpec(ch=64), image)
        latent = ref_encoder.gaussian_sample(mom, torch.randn(1, 4, side // 8, side // 8))   # posterior draw
        latent = latent + 0.02 * torch.randn_like(latent)                                   # cond_aug noise
        c, uc = ref_conditioning.v3d_conditioning(clip_emb, latent, 6, 127, 0.02, T)
        randn = torch.randn(T, 4, side // 8, side // 8)                                       # latent noise
        extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
        z = ref_sampling.euler_edm_sample(
            lambda i, s, cc: ref_sampling.denoiser(
                lambda xx, tt, cond, **kw: ref_unet.openai_wrapper(sd_u, ref_unet.UNetSpec(model_channels=64), xx, tt,
                                                                   cond, **kw), i, s, cc, **extra),
            randn, c, uc, steps, ref_sampling.guider_scale(1.5, 3.5, T), T)
        ref = ref_decoder.decode_first_stage(sd_d, ref_decoder.DecoderSpec(ch=64), z, n_samples_a_time=T)
    r, cs = _rel(frames, ref), _cos(frames, ref)
    print("views_from_image vs oracle composition: rel-L2", r, "cos", cs)
    assert frames.shape == ref.shape == (T, 3, side, side)
    assert r <= 5e-2 and cs >= 0.998


@pytest.mark.parametrize("channel_mult,num_res_blocks,attention_resolutions", [
    ((1, 2, 4), 1, (2, 1)),        # three levels, one block per level, no attention at the coarsest level
    ((1, 1, 2, 2), 2, (4,)),       # repeated widths (no 1x1 skip convs in places), attention only at ds = 4
])
def test_unet_host_schedule_other_architectures_match_oracle(channel_mult, num_res_blocks, attention_resolutions):
    """The execution plan is derived from the constructor arguments like the reference's loops
    (video_model.py:186-440): other members of the SVD configuration family go through the same code and must agree
    with the oracle built from the same arguments."""
    import emu_ops
    from oracle import ref_unet, synth
    from v3d_b200.unet import VideoUNet

    kw = dict(UNET_KW, channel_mult=list(channel_mult), num_res_blocks=num_res_blocks,
              attention_resolutions=list(attention_resolutions))
    net = VideoUNet(**kw)
    sd = synth.synth_state_dict(net.param_shapes(), seed=17)
    net.load_state_dict(sd, strict=True)
    spec = ref_unet.UNetSpec(model_channels=64, channel_mult=channel_mult, num_res_blocks=num_res_blocks,
                             attention_resolutions=attention_resolutions)
    assert set(ref_unet.unet_param_shapes(spec)) == set(net.param_shapes())        # same state_dict keys
    T, hw = 2, 16
    xin, ts, ctx, y = _unet_inputs(T, hw)
    with emu_ops.patched():
        out = _unet(net.eval(), xin, ts, ctx, y, T)
    with torch.no_grad():
        ref = ref_unet.unet_forward(sd, spec, xin, ts, ctx, y, T, torch.zeros(2, T))
    r, cs = _rel(out, ref), _cos(out, ref)
    print(channel_mult, num_res_blocks, attention_resolutions, "rel-L2", r, "cos", cs)
    assert out.shape == ref.shape and r <= 3e-2 and cs >= 0.999
    assert_per_sample(str(channel_mult), out, ref, 3e-2, 0.999)


def test_decoder_and_encoder_other_architectures_match_oracle():
    """Three-level, one-block-per-level first stage (ch_mult [1, 2, 4], num_res_blocks 1): decoder and encoder
    schedules vs the oracle built from the same arguments."""
    import emu_ops
    from oracle import ref_decoder, ref_encoder, synth
    from v3d_b200.decoder import VideoDecoder
    from v3d_b200.encoder import Encoder

    dec = VideoDecoder(**dict(DEC_KW, ch_mult=[1, 2, 4], num_res_blocks=1))
    sd = synth.synth_state_dict(dec.param_shapes(), seed=19)
    dec.load_state_dict(sd, strict=True)
    spec = ref_decoder.DecoderSpec(ch=64, ch_mult=(1, 2, 4), num_res_blocks=1)
    assert set(ref_decoder.decoder_param_shapes(spec)) == set(dec.param_shapes())
    z = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(8))
    with emu_ops.patched():
        out = dec.eval()(z, timesteps=2)
    with torch.no_grad():
        ref = ref_decoder.decoder_forward(sd, spec, z, 2)
    r = _rel(out, ref)
    print("decoder [1,2,4] x1: rel-L2", r)
    assert out.shape == ref.shape == (2, 3, 32, 32) and r <= 3e-2 and _cos(out, ref) >= 0.999

    enc = Encoder(double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=64, ch_mult=[1, 2, 4],
                  num_res_blocks=1, attn_resolutions=[], dropout=0.0, attn_type="vanilla")
    sde = synth.synth_state_dict(enc.param_shapes(), seed=20)
    enc.load_state_dict(sde, strict=True)
    espec = ref_encoder.EncoderSpec(ch=64, ch_mult=(1, 2, 4), num_res_blocks=1)
    assert set(ref_encoder.encoder_param_shapes(espec)) == set(enc.param_shapes())
    x = torch.randn(2, 3, 32, 32, generator=torch.Generator().manual_seed(9))
    with emu_ops.patched():
        out = enc.eval()(x)
    with torch.no_grad():
        ref = ref_encoder.encoder_forward(sde, espec, x)
    r = _rel(out, ref)
    print("encoder [1,2,4] x1: rel-L2", r)
    assert out.shape == ref.shape == (2, 8, 8, 8) and r <= 3e-2 and _cos(out, ref) >= 0.999


def test_clip_tower_host_schedule_matches_oracle():
    """The native CLIP image tower through FrozenOpenCLIPImagePredictionEmbedder.forward with the kernels' stand-ins,
    against oracle/ref_clip.py on the clip_small weights and image (the bound of test_parity_gpu.py's
    test_clip_tower_matches_oracle: rel-L2 3e-2, cosine 0.999).  load_state_dict and .to() drop the packed weights, as
    for the other kernel modules."""
    import json

    import emu_ops
    from oracle import ref_clip, synth
    from v3d_b200.sgm.modules.encoders.modules import FrozenOpenCLIPImagePredictionEmbedder

    m = json.loads((Path(ROOT) / "tests" / "golden" / "MANIFEST.json").read_text())["clip_small"]
    spec = ref_clip.ClipSpec(**m["spec"])
    emb = FrozenOpenCLIPImagePredictionEmbedder(
        {"target": "v3d_b200.sgm.modules.encoders.modules.FrozenOpenCLIPImageEmbedder",
         "params": {"freeze": True, "vision_cfg": m["spec"]}}, n_cond_frames=1, n_copies=1)
    sd = synth.synth_state_dict(ref_clip.clip_visual_param_shapes(spec), seed=m["weight_seed"])
    keys = set(emb.state_dict())
    emb.load_state_dict({"open_clip.model.visual." + k: v for k, v in sd.items()}, strict=False)
    assert set(emb.state_dict()) == keys
    g = torch.Generator().manual_seed(m["x_seed"])
    x = torch.rand(m["B"], 3, m["image_hw"], m["image_hw"], generator=g) * 2.0 - 1.0
    with emu_ops.patched():
        out = emb.eval()(x)
    ref = ref_clip.clip_visual_forward(sd, spec, ref_clip.preprocess(x, spec.image_size))
    r, cs = _rel(out[:, 0], ref), _cos(out[:, 0], ref)
    print("clip_small tower vs oracle: rel-L2", r, "cos", cs)
    assert out.shape == (m["B"], 1, spec.embed_dim) and r <= 3e-2 and cs >= 0.999, (r, cs)

    clip = emb.open_clip
    packed = clip._packed
    assert packed is not None
    clip.load_state_dict(clip.state_dict())
    assert clip._packed is None
    with emu_ops.patched():
        clip.packed()
    assert clip._packed is not None and clip._packed is not packed
    clip.to(torch.float32)
    assert clip._packed is None
