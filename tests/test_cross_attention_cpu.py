"""Cross-attention over contexts of more than one token (the M > 1 schedule of VideoUNet), on CPU with the kernels'
stand-ins (tests/emu_ops.py):

  * the stand-in of v3d_attention_cross against an fp64 softmax attention written out by hand, over the key counts and
    key-set strides the GPU edge test runs;
  * the UNet schedule against fixtures of the REAL reference with 3, 4 and 77 context tokens (tests/golden/
    unet_*_ctx*.pt), at the bounds of the single-token fixtures;
  * DiffusionEngine.sample_views with M = 3 against the oracle composition, and the views / cfg / cfg+views plans over
    gloo against the unsharded engine, bit for bit;
  * the single-token forward issues exactly the launch sequence it issued before this path existed;
  * assemble_v3d_conditioning with a k-token CLIP embedding against the oracle's conditioning, bit for bit.
"""
import hashlib
import json
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = str(Path(__file__).resolve().parent.parent)
sys.path.insert(0, str(Path(__file__).resolve().parent))

from framewise import assert_per_sample  # noqa: E402

UNET_KW = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
               model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
               num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
               spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
               merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])

# sha256 of the ops call sequence (entry point, tensor shapes / dtypes, scalar arguments) of one single-token forward
# of the width-64 UNet at T = 3, latent 16x16, recorded before the multi-token path was added
SINGLE_TOKEN_LAUNCHES = 744
SINGLE_TOKEN_DIGEST = "3d4721d20e3db6570438b7f97fa2f145dbe99d6ccd2a7ac2171a73d2a06b9dcc"


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _cos(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-12)).item()


def _digest(calls):
    return hashlib.sha256(repr(calls).encode()).hexdigest()


def _single_token_forward():
    import emu_ops
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**UNET_KW)
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=11), strict=True)
    T, hw = 3, 16
    x, c, uc = synth.synth_inputs(T, hw)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    ts = torch.linspace(-0.5, 1.2, 2 * T)

    calls = []
    with emu_ops.patched(calls):
        net(xin, ts, ctx, y, num_video_frames=T, image_only_indicator=torch.zeros(2, T))
    return calls


def test_single_token_forward_launch_sequence_is_unchanged():
    calls = _single_token_forward()
    print("single-token forward:", len(calls), "ops calls, digest", _digest(calls))
    assert len(calls) == SINGLE_TOKEN_LAUNCHES
    assert _digest(calls) == SINGLE_TOKEN_DIGEST
    assert not any(n == "attention_cross" for n, _, _ in calls)


# ---------------------------------------------------------------------------------------------------------------
# the stand-in of v3d_attention_cross
# ---------------------------------------------------------------------------------------------------------------
def cross_reference(q, kv, nbatch, nq, nk, nheads, scale, kv_bstride):
    """softmax(q k^T scale) v in fp64 written out by hand (no SDPA): item b's queries against rows b*kv_bstride + j."""
    c = nheads * 64
    out = torch.empty(nbatch * nq, c, dtype=torch.float64)
    for b in range(nbatch):
        qb = q[b * nq:(b + 1) * nq, :c].double().cpu()
        keys = kv[b * kv_bstride:b * kv_bstride + nk].double().cpu()
        for h in range(nheads):
            s = qb[:, h * 64:(h + 1) * 64] @ keys[:, h * 64:(h + 1) * 64].t() * scale
            p = torch.exp(s - s.max(dim=1, keepdim=True).values)
            out[b * nq:(b + 1) * nq, h * 64:(h + 1) * 64] = (p / p.sum(dim=1, keepdim=True)) @ \
                keys[:, c + h * 64:c + (h + 1) * 64]
    return out


def cross_operands(nbatch, nq, nk, nheads, gap, seed=0, amp=1.0, device="cpu"):
    """q / kv / out with row strides ld_q != ld_kv != ld_o and padded margins; `gap` extra rows between key sets hold
    NaN, which a read would spread into the output."""
    g = torch.Generator().manual_seed(seed)
    c = nheads * 64
    bs = nk + gap
    qbuf = torch.randn(nbatch * nq, c + 24, generator=g) * amp
    kvbuf = torch.randn(nbatch * bs, 2 * c + 40, generator=g)
    kvbuf[:, :c] *= amp
    for b in range(nbatch):
        kvbuf[b * bs + nk:(b + 1) * bs] = float("nan")
    q = qbuf.to(device=device, dtype=torch.bfloat16)[:, 8:8 + c]
    kv = kvbuf.to(device=device, dtype=torch.bfloat16)[:, 16:16 + 2 * c]
    obuf = torch.full((nbatch * nq, c + 56), 7.0, device=device, dtype=torch.bfloat16)
    return q, kv, obuf, bs


@pytest.mark.parametrize("nk", [1, 2, 63, 64, 65, 77, 257])
@pytest.mark.parametrize("gap", [0, 3])
def test_attention_cross_standin_matches_fp64(nk, gap):
    import emu_ops

    nbatch, nq, nheads = 3, 37, 2
    c = nheads * 64
    q, kv, obuf, bs = cross_operands(nbatch, nq, nk, nheads, gap, seed=nk, amp=4.0)
    out = obuf[:, 24:24 + c]
    emu_ops.attention_cross(q, kv, out, nbatch, nq, nk, nheads, 64 ** -0.5, kv_bstride=bs)
    ref = cross_reference(q, kv, nbatch, nq, nk, nheads, 64 ** -0.5, bs)
    assert torch.isfinite(out.float()).all()
    assert ((out.double() - ref).abs() <= 2.0 ** -8 * ref.abs()).all()                # fp64, one bf16 rounding
    assert (obuf[:, :24] == 7.0).all() and (obuf[:, 24 + c:] == 7.0).all()           # margins untouched


# ---------------------------------------------------------------------------------------------------------------
# the UNet schedule against the real reference with M > 1
# ---------------------------------------------------------------------------------------------------------------
def ctx_case(tag):
    sys.path.insert(0, str(Path(ROOT) / "tools"))
    from make_golden_ctx import ctx_inputs

    gold_dir = Path(ROOT) / "tests" / "golden"
    m = json.loads((gold_dir / "CTX.json").read_text())[tag]
    gold = torch.load(gold_dir / f"{tag}.pt")
    xin, ts, ctx, y = ctx_inputs(m["T"], m["latent_hw"], m["context_tokens"], m["sigma"])
    assert torch.equal(ts, gold["timesteps"])
    return m, gold, xin, ts, ctx, y


CTX_TAGS = ["unet_small_ctx3", "unet_small_t18_ctx77", "unet_full_t18_16_ctx4"]


# Block taps of the M-token fixtures are held to 2.5e-2 instead of the single-token fixtures' 2e-2.  Measured with these
# stand-ins at the deepest tap (output_blocks.11.1): the uc sample, whose context is zero, is at 2.19e-2 on
# unet_small_ctx3, the same as the single-token path's own uc sample on the same inputs (2.1e-2, unet_small); the c
# sample reaches 1.8-2.1e-2, about twice the single-token fixtures' c sample, because attn2 over M tokens rounds its
# q, K, V and attention output to bf16 where the single-token path adds attn2 as an fp32 epilogue bias.  That the
# schedule itself is right is pinned at the single-token bounds by the next test.
CTX_TAP_TOL = 2.5e-2


@pytest.mark.parametrize("tag", CTX_TAGS)
def test_unet_multi_token_schedule_matches_reference_golden(tag):
    """Output and block taps of the M-token schedule against the real reference (output rel-L2 3e-2 / cosine 0.999 for
    the whole tensor and every sample, like the single-token fixtures; taps CTX_TAP_TOL)."""
    import emu_ops
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    m, gold, xin, ts, ctx, y = ctx_case(tag)
    T = m["T"]
    net = VideoUNet(**dict(UNET_KW, model_channels=m["model_channels"]))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=m["weight_seed"]), strict=True)
    taps = {k[4:]: None for k in gold if k.startswith("tap:")}
    net.debug_taps = taps
    with emu_ops.patched():
        n0 = emu_ops.launch_count()
        out = net.eval()(xin, ts, ctx, y, num_video_frames=T, image_only_indicator=torch.zeros(xin.shape[0] // T, T))
        launches = emu_ops.launch_count() - n0
    report = [(name, _rel(val[[0, T]][:, ::8], gold["tap:" + name])) for name, val in taps.items()]
    r, cs = _rel(out, gold["out"]), _cos(out, gold["out"])
    print(tag, "rel-L2", r, "cos", cs, "worst tap", max(report, key=lambda t: t[1]), "launches", launches)
    assert all(v is not None for v in taps.values()) and len(report) == 6
    assert all(e <= CTX_TAP_TOL for _, e in report), report
    assert r <= 3e-2 and cs >= 0.999
    assert_per_sample(tag, out, gold["out"], 3e-2, 0.999)


def test_duplicated_tokens_match_single_token_golden():
    """Softmax over M copies of one key is that key: the M-token schedule fed the single-token fixture's context
    repeated twice must meet that fixture's own bounds (taps 2e-2, output 3e-2 / 0.999), through norm2, to_q, the
    attention kernel's stand-in, to_out and the frame-0 key sets of the temporal attn2."""
    import emu_ops
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    gold_dir = Path(ROOT) / "tests" / "golden"
    m = json.loads((gold_dir / "MANIFEST.json").read_text())["unet_small_t18"]
    gold = torch.load(gold_dir / "unet_small_t18.pt")
    net = VideoUNet(**dict(UNET_KW, model_channels=m["model_channels"]))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=m["weight_seed"]), strict=True)
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]]).repeat(1, 2, 1)
    y = torch.cat([uc["vector"], c["vector"]])
    taps = {k[4:]: None for k in gold if k.startswith("tap:")}
    net.debug_taps = taps
    calls = []
    with emu_ops.patched(calls):
        out = net(xin, gold["timesteps"], ctx, y, num_video_frames=T, image_only_indicator=torch.zeros(2, T))
    report = [(name, _rel(val[[0, T]][:, ::8], gold["tap:" + name])) for name, val in taps.items()]
    print("duplicated tokens: rel-L2", _rel(out, gold["out"]), "worst tap", max(report, key=lambda t: t[1]))
    assert sum(n == "attention_cross" for n, _, _ in calls) == 32              # 16 transformers x (spatial, temporal)
    assert all(e <= 2e-2 for _, e in report), report
    assert _rel(out, gold["out"]) <= 3e-2 and _cos(out, gold["out"]) >= 0.999


def test_multi_token_schedule_reads_the_right_key_sets():
    """The fixtures above would not notice a key-set mix-up that leaves the output within tolerance; here the same
    forward is repeated with one context perturbed at a time.  Changing frame 1's tokens must change frame 1 and leave
    the other samples bit-identical except through the temporal mixing of the same video (frame 1 is not frame 0);
    changing frame 0 of the c half must change every frame of the c half and no frame of the uc half."""
    import emu_ops
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**UNET_KW)
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=11), strict=True)
    T, hw, M = 3, 8, 3
    g = torch.Generator().manual_seed(4)
    xin, ts = torch.randn(2 * T, 8, hw, hw, generator=g), torch.linspace(-0.5, 1.0, 2 * T)
    ctx, y = torch.randn(2 * T, M, 1024, generator=g), torch.randn(2 * T, 768, generator=g)

    def run(cx):
        with emu_ops.patched():
            return net.eval()(xin, ts, cx, y, num_video_frames=T, image_only_indicator=torch.zeros(2, T))

    base = run(ctx)
    c0 = ctx.clone()
    c0[T, 2] += 1.0                                   # last token of frame 0 of the c half
    d0 = (run(c0) - base).flatten(1).abs().amax(1)
    assert (d0[:T] == 0).all() and (d0[T:] > 0).all(), d0
    c1 = ctx.clone()
    c1[1, 0] += 1.0                                   # first token of frame 1 of the uc half
    d1 = (run(c1) - base).flatten(1).abs().amax(1)
    assert (d1[T:] == 0).all() and (d1[:T] > 0).all(), d1


def test_prepare_accepts_tokens_and_keys_graphs_by_token_count():
    """_prepare flattens an M-token context to one row per sample; a frame-sharded call needs an M-token time context;
    a CUDA graph captured for one token count is never replayed for another.  `_prepare` is called directly: what is
    checked is the context matrix it hands the schedule, which forward() does not return."""
    from v3d_b200.unet import VideoUNet
    from v3d_b200.viewshard import ViewShard

    with torch.device("meta"):
        net = VideoUNet(**UNET_KW)
    T, hw = 2, 16
    xin, ts, y = torch.zeros(2 * T, 8, hw, hw), torch.zeros(2 * T), torch.zeros(2 * T, 768)
    args, dims, _ = net._prepare(xin, ts, torch.ones(2 * T, 5, 1024), y, None, T, torch.zeros(2, T))
    assert args[2].shape == (2 * T, 5 * 1024) and dims == (2 * T, T, 2, hw, hw)
    with pytest.raises(AssertionError):
        net._prepare(xin, ts, torch.ones(2 * T, 5, 768), y, None, T, torch.zeros(2, T))
    net.view_shard = ViewShard(num_frames=T, rank=0, world=1)
    try:
        args, _, _ = net._prepare(xin, ts, torch.ones(2 * T, 5, 1024), y, torch.ones(2, 5, 1024), T,
                                  torch.zeros(2, T))
        assert args[2].shape == (2 * T + 2, 5 * 1024)
        with pytest.raises(AssertionError):
            net._prepare(xin, ts, torch.ones(2 * T, 5, 1024), y, torch.ones(2, 1, 1024), T, torch.zeros(2, T))
    finally:
        net.view_shard = None
    dev = torch.device("cuda", 0)
    assert net._graph_key(36, 18, 64, 64, dev) == net._graph_key(36, 18, 64, 64, dev, 1)
    assert len({net._graph_key(36, 18, 64, 64, dev, m) for m in (1, 2, 4, 77)}) == 4


# ---------------------------------------------------------------------------------------------------------------
# the whole hot path with a multi-token context, and the sharded plans
# ---------------------------------------------------------------------------------------------------------------
def _ctx_cond(T, hw, M):
    """synth_inputs with an M-token context that differs per frame and per CFG half."""
    from oracle import synth

    x, c, uc = synth.synth_inputs(T, hw)
    g = torch.Generator().manual_seed(41)
    c = dict(c, crossattn=torch.randn(T, M, 1024, generator=g))
    uc = dict(uc, crossattn=torch.randn(T, M, 1024, generator=g))
    return x, c, uc


def test_sample_views_multi_token_matches_oracle():
    """DiffusionEngine.sample_views with a 3-token context (2 Euler-EDM steps, per-frame CFG, decode) against the oracle
    composition, at the bound smoke() applies."""
    import cpu_shims
    import emu_ops
    from oracle import ref_decoder, ref_sampling, ref_unet

    T, hw, steps = 3, 8, 2
    eng, sd_u, sd_d = cpu_shims.cpu_engine(T, steps)
    x, c, uc = _ctx_cond(T, hw, 3)
    with emu_ops.patched():
        frames = eng.sample_views(x.clone(), c, uc, num_frames=T)
    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    with torch.no_grad():
        z_ref = ref_sampling.euler_edm_sample(
            lambda i, s, cc: ref_sampling.denoiser(
                lambda xx, tt, cond, **kw: ref_unet.openai_wrapper(sd_u, ref_unet.UNetSpec(model_channels=64), xx, tt,
                                                                   cond, **kw), i, s, cc, **extra),
            x.clone(), c, uc, steps, ref_sampling.guider_scale(1.5, 3.5, T), T)
        img_ref = ref_decoder.decode_first_stage(sd_d, ref_decoder.DecoderSpec(ch=64), z_ref, n_samples_a_time=T)
    r, cs = _rel(frames, img_ref), _cos(frames, img_ref)
    print("sample_views, 3 context tokens, vs oracle composition: rel-L2", r, "cos", cs)
    assert frames.shape == img_ref.shape == (T, 3, 8 * hw, 8 * hw) and torch.isfinite(frames).all()
    assert r <= 5e-2 and cs >= 0.998, (r, cs)


def _plan_worker(rank: int, world: int, port: int, T: int, mode: str, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    import cpu_shims
    import emu_ops
    from v3d_b200.viewshard import ShardPlan

    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    plan = ShardPlan.create(T, mode)
    eng, _, _ = cpu_shims.cpu_engine(T, 2)
    x, c, uc = _ctx_cond(T, 8, 3)
    with emu_ops.patched():
        ref = eng.sample_views(x.clone(), c, uc, num_frames=T)
        mine = eng.sample_views(x.clone(), c, uc, num_frames=T, shard=plan)
        gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "equal": bool(torch.equal(gathered, ref)), "finite": bool(torch.isfinite(mine).all()),
           "gathered_rel": _rel(gathered, ref), "plan": plan.describe()})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode,world,T", [("views", 2, 5), ("cfg", 2, 4), ("cfg+views", 4, 5)])
def test_sharded_plans_with_multi_token_context_match_unsharded_gloo(mode, world, T):
    """The frame-sharded plan (the M-token time context of frame 0 travels as `time_context` and is appended to the
    context rows), the CFG split and both together reproduce the unsharded sample_views with a 3-token context bit for
    bit."""
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker, world, (T, mode), timeout=900), key=lambda r: r["rank"])
    print(res)
    for r in res:
        assert r["finite"] and r["equal"], r


# ---------------------------------------------------------------------------------------------------------------
# front end: a k-token CLIP embedding
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 4])
def test_assemble_conditioning_with_k_token_clip_embedding_matches_oracle(k):
    """get_batch + GeneralConditioner + per-frame repeat (V3D_512.py:247-267) with a [1, k, 1024] embedding give
    crossattn [T, k, 1024] (every frame the same k tokens, uc zeros) and the concat latent of the one conditioning
    image, bit for bit as the oracle's conditioning."""
    import emu_ops
    from oracle import ref_conditioning
    from v3d_b200 import conditioning

    T = 5
    g = torch.Generator().manual_seed(43)
    clip_emb, latent = torch.randn(1, k, 1024, generator=g), torch.randn(1, 4, 8, 8, generator=g)
    with emu_ops.patched():
        cond = conditioning.GeneralConditioner(conditioning.V3D_512_EMB_MODELS)
        c, uc = conditioning.assemble_v3d_conditioning(cond, clip_emb, latent, 6.0, 127.0, 0.02, T)
    oc, ouc = ref_conditioning.v3d_conditioning(clip_emb, latent, 6.0, 127.0, 0.02, T)
    assert c["crossattn"].shape == (T, k, 1024) and c["concat"].shape == (T, 4, 8, 8)
    for key in ("crossattn", "concat"):
        assert torch.equal(c[key], oc[key]) and torch.equal(uc[key], ouc[key]), key
    assert torch.allclose(c["vector"], oc["vector"], atol=2e-6) and torch.equal(uc["vector"], c["vector"])
    assert all(torch.equal(c["crossattn"][t], clip_emb[0]) for t in range(T))
