"""Videos of more than 32 view-frames on the H100: attn_temporal_long_kernel (33 <= T <= 128) in fp64 at its tile
edges, its frame-sharded form against the dense one bit for bit, which kernel each T launches, the stand-ins of
tests/emu_ops.py against the kernel, and the native UNet / sampler / engine at T = 40 and T = 48 against the
real reference's fixtures, under CUDA graphs, in deterministic mode and frame-sharded over the peer transport.  The
CPU twins are in tests/test_long_video_cpu.py."""
import json
import os
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = str(Path(__file__).resolve().parent.parent)
sys.path.insert(0, str(Path(__file__).resolve().parent))
sys.path.insert(0, str(Path(ROOT) / "tools"))

from framewise import assert_per_sample  # noqa: E402

DEV = "cuda"
BF, F64 = torch.bfloat16, torch.float64
SCALE = 64 ** -0.5
C_ATTN = 2.0 ** -8 + 2.0 ** -12        # the bound of the other attention entry points' fp64 edge tests
SENTINEL = -3.0
GOLD = Path(ROOT) / "tests" / "golden"


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _cos(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-12)).item()


# --------------------------------------------------------------------------------------------------------------
# kernel edges, fp64
# --------------------------------------------------------------------------------------------------------------
def _qkv(nb, T, S, heads, seed, pad=16):
    """Packed projection [nb*T*S, 3C + pad] bf16: every third row's q and k are 6x larger (scores of O(100) nats),
    the `pad` columns beyond 3C hold NaN."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = heads * 64
    rows = nb * T * S
    buf = torch.randn(rows, 3 * c + pad, device=DEV, generator=g)
    buf[::3, :2 * c] *= 6.0
    buf[:, 3 * c:] = float("nan")
    return buf.to(BF)


def _reference(qkv, nb, T, S, heads, t0=0, tq=None):
    """softmax(q k^T scale) v and mag = sum p |v| per (video, pixel, head) sequence in fp64, queries = frames
    [t0, t0 + tq) -> two [nb*tq*S, C] matrices in the kernel's row order.  Chunked over pixels."""
    c = heads * 64
    tq = T if tq is None else tq
    v5 = qkv[:, :3 * c].view(nb, T, S, 3, heads, 64)
    ref = torch.empty(nb, tq, S, heads, 64, dtype=F64, device=DEV)
    mag = torch.empty_like(ref)
    step = max(1, (1 << 22) // (T * T * heads))
    for s0 in range(0, S, step):
        blk = v5[:, :, s0:s0 + step].double().permute(3, 0, 2, 4, 1, 5)          # [3, b, s, h, t, 64]
        q, k, v = blk[0][..., t0:t0 + tq, :], blk[1], blk[2]
        p = torch.softmax(q @ k.transpose(-1, -2) * SCALE, dim=-1)
        ref[:, :, s0:s0 + step] = (p @ v).permute(0, 3, 1, 2, 4)
        mag[:, :, s0:s0 + step] = (p @ v.abs()).permute(0, 3, 1, 2, 4)
    return ref.reshape(nb * tq * S, c), mag.reshape(nb * tq * S, c)


def _check(what, got, ref, mag, c_mag=C_ATTN):
    err = (got.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + c_mag * mag
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isfinite(got.double()), ratio, torch.full_like(err, float("inf")))
    worst = float(ratio.max())
    print(f"EDGE attn_temporal_long {what} ratio={worst:.3g}")
    assert worst <= 1.0, f"{what}: worst |err| / (2^-8 |ref| + {c_mag:.3g} mag) = {worst:.3g}"


ALL_T = [33, 40, 47, 48, 49, 63, 64, 65, 96, 127, 128]
# every T at S = 64, 5 heads, two videos; the other pixel counts, head counts and the single video spread over the T's
CASES = [(T, 64, 5, 2) for T in ALL_T] + [
    (33, 1, 20, 2), (48, 1, 10, 1), (65, 1, 5, 2), (128, 1, 20, 1),
    (40, 64, 20, 1), (64, 64, 10, 2), (96, 64, 10, 1), (127, 64, 20, 2),
    (33, 4096, 5, 2), (48, 4096, 5, 2), (49, 4096, 10, 1), (64, 4096, 5, 1), (128, 4096, 5, 1),
]


@pytest.mark.parametrize("T,S,heads,nb", CASES)
def test_attention_temporal_long_edges(T, S, heads, nb):
    """v3d_attention_temporal for 33 <= T <= 128: the ragged last 16-query tile, the masked keys of the last 16-key
    tile, both key capacities (64 / 128), row strides wider than 3C / C with NaN padding that must not be read and
    sentinel margins and tail rows that must not be written; the other video's rows turned to NaN must not change this
    video's output.  The torch stand-in runs on the same operands where they are small."""
    import emu_ops
    from v3d_b200 import ops

    c = heads * 64
    rows = nb * T * S
    qkv = _qkv(nb, T, S, heads, seed=T * 131 + S + heads)
    ref, mag = _reference(qkv, nb, T, S, heads)
    impls = [("kernel", ops.attention_temporal)] + ([("standin", emu_ops.attention_temporal)] if S <= 64 else [])
    for impl, fn in impls:
        obuf = torch.full((rows + 8, c + 16), SENTINEL, device=DEV, dtype=BF)
        fn(qkv, obuf, nb, T, S, heads, SCALE)
        torch.cuda.synchronize()
        # the stand-in is fp64 with one bf16 rounding: no share of the magnitude term
        _check(f"{impl} T={T} S={S} heads={heads} nb={nb}", obuf[:rows, :c], ref, mag, C_ATTN if impl == "kernel" else 0.0)
        assert (obuf[:, c:] == SENTINEL).all() and (obuf[rows:] == SENTINEL).all(), "margin or tail rows written"
        if impl == "kernel":
            clean = obuf[:rows, :c].clone()
    if nb == 2:
        poisoned = qkv.clone()
        poisoned[:T * S] = float("nan")
        obuf = torch.full((rows + 8, c + 16), SENTINEL, device=DEV, dtype=BF)
        ops.attention_temporal(poisoned, obuf, nb, T, S, heads, SCALE)
        torch.cuda.synchronize()
        assert torch.equal(obuf[T * S:rows, :c], clean[T * S:]), "video 0's NaNs reached video 1"


@pytest.mark.parametrize("tq,tk,blocks,rank", [(12, 48, [12] * 4, 2), (10, 40, [10] * 4, 3), (14, 40, [14, 13, 13], 0),
                                               (16, 128, [16] * 8, 5), (1, 33, [1, 32], 0)])
@pytest.mark.parametrize("S,heads", [(64, 5), (1024, 10)])
def test_split_kv_equals_dense_bit_for_bit(tq, tk, blocks, rank, S, heads):
    """The frame-sharded form through a rank-major K|V buffer (slots padded to the largest block, laid out in shuffled
    rank order, NaN wherever no key row lives, wider row stride) gives the dense kernel's bits for this rank's frames,
    and both are within the fp64 bound."""
    from test_long_video_cpu import pack_kv, shuffled_table
    from v3d_b200 import ops

    nb = 2
    c = heads * 64
    bl, t0 = [], 0
    for n in blocks:
        bl.append((t0, n))
        t0 += n
    assert t0 == tk and bl[rank][1] == tq
    qkv = _qkv(nb, tk, S, heads, seed=tq * 7 + tk, pad=0)
    dense = torch.empty(nb * tk * S, c, device=DEV, dtype=BF)
    ops.attention_temporal(qkv, dense, nb, tk, S, heads, SCALE)
    order = list(range(len(blocks)))
    order = order[1::2] + order[0::2]
    row, bstride, nrows = shuffled_table(bl, nb, S, order)
    buf = pack_kv(qkv, c, bl, nb, tk, S, row, bstride, nrows, pad_cols=24)[:, :2 * c]
    f0 = bl[rank][0]
    ql = qkv.view(nb, tk, S, 3 * c)[:, f0:f0 + tq].reshape(nb * tq * S, 3 * c).contiguous()
    obuf = torch.full((nb * tq * S, c + 8), SENTINEL, device=DEV, dtype=BF)
    ops.attention_temporal_kv(ql, buf, obuf, nb, tq, S, heads, row, bstride, SCALE)
    torch.cuda.synchronize()
    want = dense.view(nb, tk, S, c)[:, f0:f0 + tq].reshape(nb * tq * S, c)
    assert torch.equal(obuf[:, :c], want)
    assert (obuf[:, c:] == SENTINEL).all()
    ref, mag = _reference(qkv, nb, tk, S, heads, f0, tq)
    _check(f"split Tq={tq} Tk={tk} S={S} heads={heads}", obuf[:, :c], ref, mag)
    if S == 64:
        import emu_ops

        sbuf = torch.full_like(obuf, SENTINEL)
        emu_ops.attention_temporal_kv(ql, buf, sbuf, nb, tq, S, heads, row, bstride, SCALE)
        _check(f"split standin Tq={tq} Tk={tk}", sbuf[:, :c], ref, mag, 0.0)
        assert (sbuf[:, c:] == SENTINEL).all()


def _kernels_launched(fn):
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return [e.key for e in prof.key_averages()]


def test_each_frame_count_launches_its_kernel():
    """T <= 32 still runs attn_temporal_kernel, exactly as before; 33 and up run attn_temporal_long_kernel; beyond 128
    the entry points refuse on the host and launch nothing."""
    from v3d_b200 import ops

    S, heads = 16, 2
    c = heads * 64
    for T, want, other in [(18, "attn_temporal_kernel", "attn_temporal_long_kernel"),
                           (32, "attn_temporal_kernel", "attn_temporal_long_kernel"),
                           (33, "attn_temporal_long_kernel", "attn_temporal_kernel"),
                           (128, "attn_temporal_long_kernel", "attn_temporal_kernel")]:
        qkv = _qkv(1, T, S, heads, seed=T, pad=0)
        out = torch.empty(T * S, c, device=DEV, dtype=BF)
        row, bstride = [f * S for f in range(T)], [T * S] * T
        for name, fn in (("dense", lambda: ops.attention_temporal(qkv, out, 1, T, S, heads, SCALE)),
                         ("split", lambda: ops.attention_temporal_kv(qkv, qkv[:, c:], out, 1, T, S, heads, row, bstride,
                                                                     SCALE))):
            names = _kernels_launched(fn)
            print(T, name, names)
            assert any(want in n for n in names) and not any(other in n for n in names), (T, name, names)
    qkv = _qkv(1, 129, S, heads, seed=1, pad=0)
    out = torch.empty(129 * S, c, device=DEV, dtype=BF)
    with pytest.raises(RuntimeError, match="1..128"):
        ops.attention_temporal(qkv, out, 1, 129, S, heads, SCALE)
    with pytest.raises(RuntimeError, match="<= 128"):
        ops.attention_temporal_kv(qkv, qkv[:, c:], out, 1, 129, S, heads, [0] * 129, [0] * 129, SCALE)


# --------------------------------------------------------------------------------------------------------------
# the native UNet and sampler against the real reference
# --------------------------------------------------------------------------------------------------------------
UNET_KW = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
               model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
               num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
               spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
               merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])


def _manifest(tag):
    return json.loads((GOLD / "LONGT.json").read_text())[tag]


def _net(m):
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**dict(UNET_KW, model_channels=m["model_channels"]))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=m["weight_seed"]), strict=True)
    return net.to(DEV).eval()


@pytest.mark.parametrize("tag", ["unet_small_t40", "unet_full_t48_16"])
def test_unet_long_video_forward_matches_reference(tag):
    """Eager forward (block taps) and the CUDA-graph replay of the same shape against the reference's output, at the
    bounds of the T <= 32 fixtures."""
    from make_golden_longt import unet_inputs

    m = _manifest(tag)
    gold = torch.load(GOLD / f"{tag}.pt")
    net = _net(m)
    T = m["T"]
    xin, ts, ctx, y = (t.to(DEV) for t in unet_inputs(T, m["latent_hw"], m["sigma"]))
    ind = torch.zeros(2, T, device=DEV)
    taps = {k[4:]: None for k in gold if k.startswith("tap:")}
    net.debug_taps = taps
    try:
        out = net(xin, ts, ctx, y, None, T, ind)
    finally:
        net.debug_taps = None
    report = [(n, _rel(v[[0, T]][:, ::8], gold["tap:" + n])) for n, v in taps.items()]
    r, cs = _rel(out, gold["out"]), _cos(out, gold["out"])
    print(tag, "rel-L2", r, "cos", cs, "taps", report)
    assert torch.isfinite(out).all()
    assert all(e <= 2e-2 for _, e in report), report
    assert r <= 3e-2 and cs >= 0.999
    assert_per_sample(tag, out, gold["out"], 3e-2, 0.999)
    for _ in range(2):                              # warm -> capture + replay -> replay
        g = net(xin, ts, ctx, y, None, T, ind)
    assert net.replayed_launches > 0
    assert _rel(g, gold["out"]) <= 3e-2 and _cos(g, gold["out"]) >= 0.999


def test_edm_long_video_trajectory_matches_reference():
    from oracle import synth
    from v3d_b200 import sampling

    m = _manifest("edm_small_t40")
    gold = torch.load(GOLD / "edm_small_t40.pt")
    net = _net(_manifest(m["unet"]))
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    c, uc = ({k: v.to(DEV) for k, v in d.items()} for d in (c, uc))
    sampler = sampling.EulerEDMSampler(
        num_steps=m["num_steps"],
        discretization_config={"target": "v3d_b200.sgm.modules.diffusionmodules.discretizer.EDMDiscretization",
                               "params": {"sigma_max": m["sigma_max"]}},
        guider_config={"target": "v3d_b200.sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                       "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}})
    den = sampling.Denoiser({"target": "v3d_b200.sgm.modules.diffusionmodules.denoiser_scaling.VScalingWithEDMcNoise"})
    model = sampling.OpenAIWrapper(net)
    extra = {"image_only_indicator": torch.zeros(2, T, device=DEV), "num_video_frames": T}
    out = sampler(lambda i, s, cc: den(model, i, s, cc, **extra), x.clone().to(DEV), cond=c, uc=uc)
    torch.cuda.synchronize()
    r = _rel(out, gold["out"])
    print("edm_small_t40 rel-L2", r)
    assert r <= 3e-2
    assert_per_sample("edm_small_t40", out, gold["out"], 3e-2)


# --------------------------------------------------------------------------------------------------------------
# the engine: CUDA graphs, deterministic mode, frame-sharded
# --------------------------------------------------------------------------------------------------------------
def _small_engine(T, dev=DEV):
    from oracle import synth
    from v3d_b200 import engine

    cfg = engine.v3d_512_config(num_frames=T, num_steps=2, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = 64
    eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    unet.load_state_dict(synth.synth_state_dict(unet.param_shapes(), seed=11), strict=True)
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=12), strict=True)
    return eng.to(dev).eval()


def _cond(T, hw, dev=DEV):
    from oracle import synth

    x, c, uc = synth.synth_inputs(T, hw)
    g = torch.Generator().manual_seed(5)
    c = dict(c, crossattn=c["crossattn"] + 0.5 * torch.randn(T, 1, 1024, generator=g))     # frames differ
    return x.to(dev), {k: v.to(dev) for k, v in c.items()}, {k: v.to(dev) for k, v in uc.items()}


def test_sample_views_48_frames_graphs_equal_eager(monkeypatch):
    """sample_views at T = 48 (reduced width, deterministic mode so that equality is exact): the eager run, the run that
    captures the graphs and the run that replays them give the same frames."""
    monkeypatch.setenv("V3D_DETERMINISTIC", "1")
    T = 48
    eng = _small_engine(T)
    unet = eng.model.diffusion_model
    x, c, uc = _cond(T, 16)
    unet.cuda_graphs = False
    eager = eng.sample_views(x.clone(), c, uc, num_frames=T)
    unet.cuda_graphs = True
    runs = [eng.sample_views(x.clone(), c, uc, num_frames=T) for _ in range(3)]
    assert unet.replayed_launches > 0
    assert eager.shape == (T, 3, 128, 128) and torch.isfinite(eager).all() and eager.float().std() > 1e-3
    for r in runs:
        assert torch.equal(r, eager)


def test_deterministic_mode_40_frames_is_reproducible(monkeypatch):
    monkeypatch.setenv("V3D_DETERMINISTIC", "1")
    T = 40
    x, c, uc = _cond(T, 16)
    a = _small_engine(T).sample_views(x.clone(), c, uc, num_frames=T)
    b = _small_engine(T).sample_views(x.clone(), c, uc, num_frames=T)
    assert torch.isfinite(a).all() and torch.equal(a, b)


def _views_worker(rank: int, world: int, port: int, T: int, det: bool, q):
    sys.path.insert(0, ROOT)
    os.environ["V3D_SHARD_TRANSPORT"] = "peer"
    if det:
        os.environ["V3D_DETERMINISTIC"] = "1"
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    from v3d_b200.viewshard import ShardPlan

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    eng = _small_engine(T, dev)
    x, c, uc = _cond(T, 16, dev)
    plan = ShardPlan.create(T, "views")
    ref = eng.sample_views(x.clone(), c, uc, num_frames=T, decoding_t=T)        # a sharded video decodes as one chunk
    mine = eng.sample_views(x.clone(), c, uc, num_frames=T, shard=plan)
    torch.cuda.synchronize()
    plan.check_status()
    gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "peer": plan.describe()["transport"].startswith("peer"),
           "finite": bool(torch.isfinite(mine).all()), "equal": bool(torch.equal(gathered.cpu(), ref.cpu())),
           "gathered_rel": _rel(gathered, ref), "kv_allgather": plan.sample.exchanges.get("kv_allgather", 0)})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("det", [False, True])
def test_views_plan_40_frames_peer_transport_one_gpu(det):
    """sample_views at T = 40 frame-sharded over two processes sharing cuda:0 through the one-sided peer transport (20
    query frames against 40 key frames per rank): within 3e-2 of the unsharded engine, and exactly equal in
    deterministic mode."""
    from mp_util import run_workers

    res = sorted(run_workers(_views_worker, 2, (40, det), timeout=900), key=lambda r: r["rank"])
    print(res)
    for r in res:
        assert r["peer"] and r["finite"] and r["kv_allgather"] > 0, r
        assert r["gathered_rel"] <= 3e-2, r
        assert r["equal"] or not det, r
