"""Cross-attention over contexts of more than one token on the H100: the v3d_attention_cross kernel at its edges in
fp64, the native UNet against the real reference's multi-token fixtures, the deterministic mode and the frame-sharded
plan over the peer transport.  The CPU twins are in tests/test_cross_attention_cpu.py."""
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


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _cos(a, b):
    a, b = a.float().cpu().flatten(), b.float().cpu().flatten()
    return (a @ b / (a.norm() * b.norm()).clamp_min(1e-12)).item()


# --------------------------------------------------------------------------------------------------------------
# kernel edges, fp64
# --------------------------------------------------------------------------------------------------------------
def _operands(nbatch, nq, nk, heads, gap, amp, seed):
    """q [nbatch*nq, C] in a row-strided buffer (ld_q = C + 24), K | V in another (ld_kv = 2C + 40), key set b at rows
    b*(nk + gap) with NaN rows between sets; output window of a sentinel-filled buffer with ld_o = C + 56."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    c = heads * 64
    bs = nk + gap
    qbuf = (torch.randn(nbatch * nq, c + 24, device=DEV, generator=g) * amp).to(BF)
    kvbuf = torch.randn(nbatch * bs, 2 * c + 40, device=DEV, generator=g)
    kvbuf[:, 16:16 + c] *= amp
    kvbuf = kvbuf.to(BF)
    for b in range(nbatch):
        kvbuf[b * bs + nk:(b + 1) * bs] = float("nan")
    obuf = torch.full((nbatch * nq, c + 56), SENTINEL, device=DEV, dtype=BF)
    return qbuf[:, 8:8 + c], kvbuf[:, 16:16 + 2 * c], obuf, bs


def _reference(q, kv, nbatch, nq, nk, heads, bs):
    """softmax(q k^T scale) v and mag = sum p |v| / sum p, fp64, per (item, head)."""
    c = heads * 64
    ref = torch.empty(nbatch * nq, c, dtype=F64, device=DEV)
    mag = torch.empty_like(ref)
    for b in range(nbatch):
        qb = q[b * nq:(b + 1) * nq].double()
        keys = kv[b * bs:b * bs + nk].double()
        for h in range(heads):
            sl = slice(h * 64, (h + 1) * 64)
            p = torch.softmax(qb[:, sl] @ keys[:, sl].t() * SCALE, dim=-1)
            v = keys[:, c + h * 64:c + (h + 1) * 64]
            ref[b * nq:(b + 1) * nq, sl] = p @ v
            mag[b * nq:(b + 1) * nq, sl] = p @ v.abs()
    return ref, mag


def _check(what, got, ref, mag):
    err = (got.double() - ref).abs()
    bound = 2.0 ** -8 * ref.abs() + C_ATTN * mag
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isfinite(got.double()), ratio, torch.full_like(err, float("inf")))
    worst = float(ratio.max())
    print(f"EDGE attn_cross {what} ratio={worst:.3g}")
    assert worst <= 1.0, f"{what}: worst |err| / (2^-8 |ref| + {C_ATTN:.3g} mag) = {worst:.3g}"


NQ = [1, 127, 128, 129, 4096, 73728]
NK = [1, 2, 63, 64, 65, 77, 257]
HEADS = [1, 5, 20]


@pytest.mark.parametrize("heads", HEADS)
@pytest.mark.parametrize("nk", NK)
@pytest.mark.parametrize("nq", NQ)
def test_attention_cross_edges(nq, nk, heads):
    """v3d_attention_cross: query tiles with tails, key counts below, at and past one 64-key tile (the tail keys come
    zero-filled from TMA and must be masked), key sets packed (kv_bstride = nk) and spaced with NaN rows that must not
    be read, distinct row strides and untouched margins; scores of O(1) and of O(100) nats (the running maximum).  The
    torch stand-in runs on the same operands."""
    import emu_ops
    from v3d_b200 import ops

    nbatch = 1 if nq == 73728 else 2
    c = heads * 64
    for gap in (0, 5):
        for amp in (1.0, 6.0):
            seed = nq * 7 + nk * 131 + heads * 3 + gap + int(amp)
            q, kv, obuf, bs = _operands(nbatch, nq, nk, heads, gap, amp, seed)
            ref, mag = _reference(q, kv, nbatch, nq, nk, heads, bs)
            impls = [("kernel", ops.attention_cross)] + ([("standin", emu_ops.attention_cross)] if nq <= 4096 else [])
            for impl, fn in impls:
                obuf.fill_(SENTINEL)
                out = obuf[:, 24:24 + c]
                fn(q, kv, out, nbatch, nq, nk, heads, SCALE, kv_bstride=bs)
                torch.cuda.synchronize()
                _check(f"{impl} nq={nq} nk={nk} heads={heads} gap={gap} amp={amp}", out, ref, mag)
                assert (obuf[:, :24] == SENTINEL).all() and (obuf[:, 24 + c:] == SENTINEL).all(), "margin written"


def test_attention_cross_rejects_bad_arguments():
    from v3d_b200 import ops

    q = torch.zeros(8, 64, device=DEV, dtype=BF)
    kv = torch.zeros(8, 128, device=DEV, dtype=BF)
    out = torch.zeros(8, 64, device=DEV, dtype=BF)
    for args in ((q, kv, out, 2, 4, 0, 1), (q, kv, out, 2, 4, 5, 1), (q, kv, out, 0, 4, 2, 1)):
        with pytest.raises(RuntimeError, match="attention_cross"):
            ops.attention_cross(*args, SCALE, kv_bstride=4 if args[5] == 5 else None)


# --------------------------------------------------------------------------------------------------------------
# the native UNet against the real reference
# --------------------------------------------------------------------------------------------------------------
UNET_KW = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
               model_channels=64, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
               num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
               spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
               merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])
GOLD = Path(ROOT) / "tests" / "golden"
CTX_TAP_TOL = 2.5e-2          # why it is not 2e-2: tests/test_cross_attention_cpu.py, CTX_TAP_TOL


def _net(mc, wseed):
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**dict(UNET_KW, model_channels=mc))
    net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=wseed), strict=True)
    return net.to(DEV).eval()


@pytest.mark.parametrize("tag", ["unet_small_ctx3", "unet_small_t18_ctx77", "unet_full_t18_16_ctx4"])
def test_unet_multi_token_forward_matches_reference(tag):
    """Eager forward (block taps) and the CUDA-graph replay of the same shape against the reference's output."""
    from make_golden_ctx import ctx_inputs

    m = json.loads((GOLD / "CTX.json").read_text())[tag]
    gold = torch.load(GOLD / f"{tag}.pt")
    net = _net(m["model_channels"], m["weight_seed"])
    T = m["T"]
    xin, ts, ctx, y = (t.to(DEV) for t in ctx_inputs(T, m["latent_hw"], m["context_tokens"], m["sigma"]))
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
    assert all(e <= CTX_TAP_TOL for _, e in report), report
    assert r <= 3e-2 and cs >= 0.999
    assert_per_sample(tag, out, gold["out"], 3e-2, 0.999)
    for _ in range(2):                              # warm -> capture + replay -> replay
        g = net(xin, ts, ctx, y, None, T, ind)
    assert net.replayed_launches > 0
    assert _rel(g, gold["out"]) <= 3e-2 and _cos(g, gold["out"]) >= 0.999


def test_multi_token_graph_is_not_replayed_for_another_token_count(monkeypatch):
    """One shape, two token counts, alternated: each gets its own graph (a graph captured for M = 4 replayed with M = 1
    inputs would read the context rows as 4 tokens).  In the deterministic mode every call of a token count, eager or
    replayed, gives the same bytes."""
    from make_golden_ctx import ctx_inputs

    monkeypatch.setenv("V3D_DETERMINISTIC", "1")
    net = _net(64, 1)
    T = 2
    xin, ts, ctx, y = (t.to(DEV) for t in ctx_inputs(T, 16, 4, 3.0))
    ind = torch.zeros(2, T, device=DEV)
    outs = {}
    for M in (4, 1, 4, 1, 4, 1):
        outs.setdefault(M, []).append(net(xin, ts, ctx[:, :M].contiguous(), y, None, T, ind))
    assert len(net._graphs) == 2 and net.replayed_launches > 0
    for M, o in outs.items():
        assert all(torch.equal(oi, o[0]) for oi in o[1:]), M
    assert _rel(outs[4][-1], outs[1][-1]) > 1e-2


def test_multi_token_forward_is_deterministic(monkeypatch):
    """V3D_DETERMINISTIC=1: the same M = 4 forward twice gives the same bytes (eager, then graph replays)."""
    from make_golden_ctx import ctx_inputs

    monkeypatch.setenv("V3D_DETERMINISTIC", "1")
    net = _net(64, 2)
    T = 5
    xin, ts, ctx, y = (t.to(DEV) for t in ctx_inputs(T, 16, 4, 3.0))
    ind = torch.zeros(2, T, device=DEV)
    outs = [net(xin, ts, ctx, y, None, T, ind) for _ in range(4)]
    for o in outs[1:]:
        assert torch.equal(o, outs[0])


# --------------------------------------------------------------------------------------------------------------
# frame-sharded over the peer transport: two processes on one GPU
# --------------------------------------------------------------------------------------------------------------
def _views_worker(rank: int, world: int, port: int, T: int, M: int, q):
    sys.path.insert(0, ROOT)
    os.environ["V3D_SHARD_TRANSPORT"] = "peer"
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    from oracle import synth
    from v3d_b200 import engine
    from v3d_b200.viewshard import ViewShard

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    hw = 16
    cfg = engine.v3d_512_config(num_frames=T, num_steps=2, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = 64
    eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    unet.load_state_dict(synth.synth_state_dict(unet.param_shapes(), seed=11), strict=True)
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=12), strict=True)
    eng = eng.to(dev).eval()
    x, c, uc = synth.synth_inputs(T, hw)
    g = torch.Generator().manual_seed(47)
    c = dict(c, crossattn=torch.randn(T, M, 1024, generator=g))          # every frame its own M tokens
    uc = dict(uc, crossattn=torch.zeros(T, M, 1024))
    c, uc = ({k: v.to(dev) for k, v in d.items()} for d in (c, uc))
    vs = ViewShard.create(T)
    ref = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T)
    mine = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T, view_shard=vs)
    gathered = vs.gather_frames(mine)
    torch.cuda.synchronize()
    q.put({"rank": rank, "peer": vs.peer is not None, "finite": bool(torch.isfinite(mine).all()),
           "frames_rel": _rel(mine, ref[vs.frames]), "gathered_rel": _rel(gathered, ref),
           "kv_allgather": vs.exchanges.get("kv_allgather", 0)})
    dist.barrier()
    dist.destroy_process_group()


def test_view_sharded_engine_multi_token_peer_transport_one_gpu():
    """sample_views with a 4-token context, frame-sharded over two processes sharing cuda:0 through the one-sided peer
    transport, against the unsharded engine (the bound of the single-token peer test: the fp64 GroupNorm statistics
    sum in another order)."""
    from mp_util import run_workers

    res = sorted(run_workers(_views_worker, 2, (5, 4), timeout=900), key=lambda r: r["rank"])
    print(res)
    for r in res:
        assert r["peer"] and r["finite"] and r["kv_allgather"] > 0, r
        assert r["frames_rel"] <= 3e-2 and r["gathered_rel"] <= 3e-2, r
