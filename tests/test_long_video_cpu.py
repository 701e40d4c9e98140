"""Videos of more than 32 view-frames (up to 128), on CPU with the kernels' stand-ins (tests/emu_ops.py):

  * the temporal attention stand-ins against an fp64 softmax attention written out per sequence, dense and
    through a shuffled, padded, rank-major row table;
  * the UNet schedule and a 3-step Euler-EDM trajectory against fixtures of the REAL reference at T = 40 and T = 48
    (tests/golden/unet_small_t40.pt, unet_full_t48_16.pt, edm_small_t40.pt), at the bounds of the T <= 32 fixtures;
  * the views / cfg / cfg+views plans over gloo at T = 40 and T = 48 against the unsharded engine, bit for bit;
  * more than 128 frames are refused with a ValueError before any kernel of the schedule is launched, also when the
    video is frame-sharded and the local block is short;
  * forwards at T = 18 and T = 32 issue exactly the launch sequence they issued before long videos existed.
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
sys.path.insert(0, str(Path(ROOT) / "tools"))

from framewise import assert_per_sample  # noqa: E402

GOLD = Path(ROOT) / "tests" / "golden"
UNET_KW = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
               model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
               num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
               spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
               merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])

# (ops calls, sha256 of the call sequence: entry point, tensor shapes / dtypes / strides, scalar arguments) of one
# forward of the width-64 UNet at latent 8x8, recorded on the commit before the long-sequence kernel was added
SHORT_T_LAUNCHES = {18: (683, "5b2ddb63ed1d0ab3aa2f00a60964086080ce677c9f006d2513eb2f843a94c001"),
                    32: (683, "1bd01fef55b81feb4f8d9eccc5c2f0bbe49f33c61d56b11c1c1a1fb2865ba2a2")}


def _rel(a, b):
    return ((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-12)).item()


def _cos(a, b):
    a, b = a.float().flatten(), b.float().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-12)).item()


# ---------------------------------------------------------------------------------------------------------------
# the stand-ins
# ---------------------------------------------------------------------------------------------------------------
def shuffled_table(blocks, nb, s, rank_order):
    """Row table of a rank-major K|V buffer whose slots are padded to the largest block and laid out in `rank_order`
    (a permutation of the ranks): -> (row, bstride, buffer rows).  Key frames stay in video order."""
    tmax = max(n for _, n in blocks)
    slot = nb * tmax * s
    row, bstride = [], []
    for r, (_, n) in enumerate(blocks):
        for j in range(n):
            row.append(rank_order.index(r) * slot + j * s)
            bstride.append(n * s)
    return row, bstride, len(blocks) * slot


def pack_kv(qkv, c, blocks, nb, T, s, row, bstride, nrows, pad_cols=0):
    """The K|V columns of the dense [nb*T*s, 3c] matrix scattered through the table into a NaN-filled buffer."""
    buf = torch.full((nrows, 2 * c + pad_cols), float("nan"), device=qkv.device, dtype=qkv.dtype)
    v = qkv.view(nb, T, s, -1)
    for f in range(T):
        for b in range(nb):
            buf[row[f] + b * bstride[f]: row[f] + b * bstride[f] + s, :2 * c] = v[b, f, :, c:3 * c]
    return buf


def sequence_reference(qkv, nb, T, s, heads, scale):
    """fp64 softmax attention of every (video, pixel, head) sequence, one at a time -> [nb*T*s, c]."""
    c = heads * 64
    v = qkv.double().view(nb, T, s, 3, heads, 64)
    out = torch.empty(nb, T, s, heads, 64, dtype=torch.float64)
    for b in range(nb):
        for p in range(s):
            for h in range(heads):
                q, k, val = v[b, :, p, 0, h], v[b, :, p, 1, h], v[b, :, p, 2, h]
                out[b, :, p, h] = torch.softmax(q @ k.t() * scale, dim=-1) @ val
    return out.reshape(nb * T * s, c)


@pytest.mark.parametrize("T,blocks,rank", [(33, [(0, 1), (1, 32)], 0), (40, [(0, 14), (14, 13), (27, 13)], 1),
                                           (48, [(0, 12), (12, 12), (24, 12), (36, 12)], 3),
                                           (128, [(0, 16)] + [(16 * i, 16) for i in range(1, 8)], 5)])
def test_temporal_standins_match_fp64(T, blocks, rank):
    import emu_ops

    nb, s, heads = 2, 3, 2
    c = heads * 64
    g = torch.Generator().manual_seed(T)
    qkv = (torch.randn(nb * T * s, 3 * c, generator=g) * 2.0).to(torch.bfloat16)
    ref = sequence_reference(qkv, nb, T, s, heads, 0.125)
    dense = torch.zeros(nb * T * s, c, dtype=torch.bfloat16)
    emu_ops.attention_temporal(qkv, dense, nb, T, s, heads, 0.125)
    assert ((dense.double() - ref).abs() <= 2.0 ** -8 * ref.abs()).all()                    # fp64, one bf16 rounding
    order = list(range(len(blocks)))[::-1]
    row, bstride, nrows = shuffled_table(blocks, nb, s, order)
    buf = pack_kv(qkv, c, blocks, nb, T, s, row, bstride, nrows, pad_cols=8)[:, :2 * c]
    t0, tl = blocks[rank]
    ql = qkv.view(nb, T, s, 3 * c)[:, t0:t0 + tl].reshape(nb * tl * s, 3 * c)
    out = torch.zeros(nb * tl * s, c, dtype=torch.bfloat16)
    emu_ops.attention_temporal_kv(ql, buf, out, nb, tl, s, heads, row, bstride, 0.125)
    assert torch.equal(out, dense.view(nb, T, s, c)[:, t0:t0 + tl].reshape(nb * tl * s, c))


# ---------------------------------------------------------------------------------------------------------------
# the host schedule against the real reference at T = 40 and T = 48
# ---------------------------------------------------------------------------------------------------------------
def _manifest(tag):
    return json.loads((GOLD / "LONGT.json").read_text())[tag]


def _net(m):
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**dict(UNET_KW, model_channels=m["model_channels"]))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=m["weight_seed"]), strict=True)
    return net.eval()


@pytest.mark.parametrize("tag", ["unet_small_t40", "unet_full_t48_16"])
def test_unet_long_video_schedule_matches_reference_golden(tag):
    """Output rel-L2 3e-2 / cosine 0.999 for the whole tensor and every sample, block taps 2e-2: the bounds of the
    T <= 32 fixtures."""
    import emu_ops
    from make_golden_longt import unet_inputs

    m = _manifest(tag)
    gold = torch.load(GOLD / f"{tag}.pt")
    T = m["T"]
    xin, ts, ctx, y = unet_inputs(T, m["latent_hw"], m["sigma"])
    assert torch.equal(ts, gold["timesteps"])
    net = _net(m)
    taps = {k[4:]: None for k in gold if k.startswith("tap:")}
    net.debug_taps = taps
    with emu_ops.patched():
        n0 = emu_ops.launch_count()
        out = net(xin, ts, ctx, y, num_video_frames=T, image_only_indicator=torch.zeros(xin.shape[0] // T, T))
        launches = emu_ops.launch_count() - n0
    report = [(name, _rel(val[[0, T]][:, ::8], gold["tap:" + name])) for name, val in taps.items()]
    r, cs = _rel(out, gold["out"]), _cos(out, gold["out"])
    print(tag, "rel-L2", r, "cos", cs, "worst tap", max(report, key=lambda t: t[1]), "launches", launches)
    assert all(v is not None for v in taps.values()) and len(report) == 6
    assert all(e <= 2e-2 for _, e in report), report
    assert r <= 3e-2 and cs >= 0.999
    assert_per_sample(tag, out, gold["out"], 3e-2, 0.999)


def test_edm_long_video_trajectory_matches_reference_golden():
    """3 Euler-EDM steps under LinearPredictionGuider(num_frames=40) through the drop-in sampler / denoiser / wrapper."""
    import emu_ops
    from oracle import synth
    from v3d_b200 import sampling

    m = _manifest("edm_small_t40")
    gold = torch.load(GOLD / "edm_small_t40.pt")
    net = _net(_manifest(m["unet"]))
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    sampler = sampling.EulerEDMSampler(
        num_steps=m["num_steps"],
        discretization_config={"target": "v3d_b200.sgm.modules.diffusionmodules.discretizer.EDMDiscretization",
                               "params": {"sigma_max": m["sigma_max"]}},
        guider_config={"target": "v3d_b200.sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                       "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}})
    den = sampling.Denoiser({"target": "v3d_b200.sgm.modules.diffusionmodules.denoiser_scaling.VScalingWithEDMcNoise"})
    model = sampling.OpenAIWrapper(net)
    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    with emu_ops.patched():
        out = sampler(lambda i, s, cc: den(model, i, s, cc, **extra), x.clone(), cond=c, uc=uc)
    r = _rel(out, gold["out"])
    print("edm_small_t40 rel-L2", r)
    assert r <= 3e-2
    assert_per_sample("edm_small_t40", out, gold["out"], 3e-2)


# ---------------------------------------------------------------------------------------------------------------
# the sharded plans
# ---------------------------------------------------------------------------------------------------------------
def test_shard_plans_partition_long_videos():
    from v3d_b200.viewshard import ViewShard, partition_frames

    assert [n for _, n in partition_frames(48, 8)] == [6] * 8
    assert [n for _, n in partition_frames(40, 3)] == [14, 13, 13]
    assert [n for _, n in partition_frames(128, 8)] == [16] * 8
    vs = ViewShard(num_frames=40, rank=2, world=3)
    row, bstride = vs.kv_table(nb=2, rows_per_frame=4)
    assert len(row) == 40 and (vs.t0, vs.tl, vs.tmax) == (27, 13, 14)
    slot = 2 * 14 * 4                                       # every rank's slot is padded to the largest block
    assert row[:2] == [0, 4] and row[14] == slot and row[27] == 2 * slot and row[39] == 2 * slot + 12 * 4
    assert bstride[0] == 14 * 4 and bstride[14] == bstride[39] == 13 * 4


def _plan_worker(rank: int, world: int, port: int, T: int, mode: str, q):
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
    eng, _, _ = cpu_shims.cpu_engine(T, 1)
    x, c, uc = synth.synth_inputs(T, 8)
    with emu_ops.patched():
        ref = eng.sample_views(x.clone(), c, uc, num_frames=T, decoding_t=T)    # a sharded video decodes as one chunk
        mine = eng.sample_views(x.clone(), c, uc, num_frames=T, shard=plan)
        gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "equal": bool(torch.equal(gathered, ref)), "finite": bool(torch.isfinite(mine).all()),
           "gathered_rel": _rel(gathered, ref), "plan": plan.describe()})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode,world,T", [("views", 2, 40), ("views", 3, 40), ("views", 4, 48), ("cfg", 2, 40),
                                          ("cfg+views", 4, 48)])
def test_sharded_plans_match_unsharded_long_video_gloo(mode, world, T):
    """Each rank's frames attend to all 40 / 48 key frames through the row table (blocks of 20, 14/13/13 and 12, and
    24 split 12/12 for the decode): the gathered frames equal the unsharded sample_views bit for bit.  The unsharded
    call decodes the video as one chunk (decoding_t = T), as every sharded plan does; its default of 24 frames per chunk
    cuts the decoder's temporal convolutions at the chunk borders once T > 24."""
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker, world, (T, mode), timeout=1500), key=lambda r: r["rank"])
    print(res)
    for r in res:
        assert r["finite"] and r["equal"], r


# ---------------------------------------------------------------------------------------------------------------
# the frame limit
# ---------------------------------------------------------------------------------------------------------------
def test_more_than_128_frames_is_refused_before_any_launch():
    import emu_ops
    from v3d_b200 import ops
    from v3d_b200.unet import VideoUNet
    from v3d_b200.viewshard import ViewShard

    assert ops.MAX_TEMPORAL_FRAMES == 128
    with torch.device("meta"):
        net = VideoUNet(**UNET_KW)

    def call(T, total=None, tc=None):
        xin, ts, y = torch.zeros(2 * T, 8, 8, 8), torch.zeros(2 * T), torch.zeros(2 * T, 768)
        return net(xin, ts, torch.zeros(2 * T, 1, 1024), y, tc, T, torch.zeros(2, T))

    with emu_ops.patched():
        n0 = emu_ops.launch_count()
        with pytest.raises(ValueError, match="temporal attention supports at most 128 frames, got 129"):
            call(129)
        # frame-sharded: this rank's 33 frames are fine on their own, the 132 key frames of the video are not
        net.view_shard = ViewShard(num_frames=132, rank=0, world=4)
        try:
            with pytest.raises(ValueError, match="at most 128 frames, got 132"):
                call(33, tc=torch.zeros(2, 1, 1024))
        finally:
            net.view_shard = None
        assert emu_ops.launch_count() == n0
    # the argument checks alone: forward() would go on to pack the meta-device weights this test builds
    net._prepare(torch.zeros(256, 8, 8, 8), torch.zeros(256), torch.zeros(256, 1, 1024), torch.zeros(256, 768), None,
                 128, torch.zeros(2, 128))


def test_front_end_takes_48_frames():
    """The public helpers a 48-view orbit passes through carry no frame assumption."""
    from v3d_b200 import engine, wire

    cfg = engine.v3d_512_config(num_frames=48)
    assert cfg["sampler_config"]["params"]["guider_config"]["params"]["num_frames"] == 48
    poses = wire.orbit_poses(48)
    assert len(poses) == 48


# ---------------------------------------------------------------------------------------------------------------
# T <= 32 is untouched
# ---------------------------------------------------------------------------------------------------------------
def short_forward_calls(T, hw=8):
    """Every ops launch ([(name, args, kwargs)], tensors as shapes) of one forward of the width-64 UNet."""
    import emu_ops
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**UNET_KW)
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=11), strict=True)
    x, c, uc = synth.synth_inputs(T, hw)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    ts = torch.linspace(-0.5, 1.2, 2 * T)
    calls = []
    with emu_ops.patched(calls):
        net(xin, ts, ctx, y, num_video_frames=T, image_only_indicator=torch.zeros(2, T))
    return calls


@pytest.mark.parametrize("T", [18, 32])
def test_short_video_launch_sequence_is_unchanged(T):
    calls = short_forward_calls(T)
    digest = hashlib.sha256(repr(calls).encode()).hexdigest()
    print(f"T = {T}:", len(calls), "ops calls, digest", digest)
    assert (len(calls), digest) == SHORT_T_LAUNCHES[T]
    assert sum(n == "attention_temporal" for n, _, _ in calls) == 16
