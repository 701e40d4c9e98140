"""Frame-sharded (view-sharded) CUDA path vs the unsharded CUDA path (SURVEY.md 8(e)).

Kernel level (one process): the halo'd-operand mode of the tap GEMM and the split-KV temporal attention must give the
SAME BITS as the dense kernels on the frames they own (same K order, same tile arithmetic).
Model level: two processes run `DiffusionEngine.sample_views(view_shard=...)` on an uneven 3/2 split of T=5 frames
and compare with the unsharded engine - over gloo with both ranks on cuda:0 (exchanges staged through the host, so it
runs on a one-GPU box) and over NCCL on two GPUs when the box has them.  The only arithmetic difference is the
summation order of the fp64 GroupNorm statistics (atomics: the unsharded path is not run-to-run deterministic
either); where that flips a bf16 rounding, this random-weight network amplifies the flip to its bf16 noise floor
within a few blocks (measured with the CPU stand-ins: one flip -> rel-L2 1e-2 at the output), so the model-level
bound is the parity tolerance of SURVEY.md App. C (rel-L2 <= 3e-2); the schedule itself is proven bit-exact against
the unsharded schedule in tests/test_host_schedule_cpu.py and the kernels bit-exact above.
"""
import os
import sys
from pathlib import Path

import pytest
import torch

pytestmark = [pytest.mark.gpu]

ROOT = str(Path(__file__).resolve().parent.parent)
DEV = "cuda"

# The gloo-staged variants (exchanges copied through host memory, all ranks on cuda:0) spawn 2-4 model-building
# processes each.  The frame-block plan stays in the default suite (it covers the torch.distributed fallback transport on
# a one-GPU box); the CFG-pair and the 4-process composite duplicates exercise no device code that the peer-transport
# variants below do not (same kernels, same schedules), their host logic is proven bit-exact over gloo in the CPU suite
# (tests/test_host_schedule_cpu.py) and they add ~2 minutes, so they run on request only.
slow = pytest.mark.skipif(os.environ.get("V3D_SLOW_TESTS") != "1", reason="gloo-staged duplicate of the peer-transport "
                          "test (set V3D_SLOW_TESTS=1)")


def _rel(a, b):
    a, b = a.float().cpu(), b.float().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


# --------------------------------------------------------------------------------------------------------------
# kernel level
# --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("hw,c,T,blocks", [(64, 320, 5, [(0, 3), (3, 2)]), (256, 128, 6, [(0, 2), (2, 2), (4, 2)]),
                                           (4, 64, 5, [(0, 3), (3, 2)]), (1024, 64, 4, [(0, 1), (1, 3)])])
def test_tap_gemm_halo_mode_equals_dense(hw, c, T, blocks):
    from v3d_b200 import ops

    nb = 2
    g = torch.Generator(device=DEV).manual_seed(hw + c)
    a = torch.randn(nb, T, hw, c, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(c, 3 * c, device=DEV, generator=g) / (3 * c) ** 0.5).to(torch.bfloat16)
    bias = torch.randn(c, device=DEV, generator=g)
    r1 = torch.randn(nb, T, hw, c, device=DEV, generator=g).to(torch.bfloat16)
    dense = torch.empty(nb * T * hw, c, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a.view(-1, c), w, dense, K=c, N=c, rows_per_batch=T * hw, batch=nb, a_batch_stride=T * hw * c, bias=bias,
             ntaps=3, tap_shift=hw, r1=r1.view(-1, c), s1=1.0, s0=0.5)
    dense = dense.view(nb, T, hw, c)
    for t0, tl in blocks:
        pad = torch.zeros(nb, tl + 2, hw, c, device=DEV, dtype=torch.bfloat16)
        lo, hi = max(t0 - 1, 0), min(t0 + tl + 1, T)
        pad[:, lo - (t0 - 1): hi - (t0 - 1)] = a[:, lo:hi]            # halos from the neighbours, zeros at the ends
        out = torch.empty(nb * tl * hw, c, device=DEV, dtype=torch.bfloat16)
        r1l = r1[:, t0:t0 + tl].contiguous()
        ops.gemm(pad.view(-1, c), w, out, K=c, N=c, rows_per_batch=tl * hw, batch=nb,
                 a_batch_stride=(tl + 2) * hw * c, bias=bias, ntaps=3, tap_shift=hw, r1=r1l.view(-1, c), s1=1.0,
                 s0=0.5, a_rows=(tl + 2) * hw, a_row0=hw)
        torch.cuda.synchronize()
        assert torch.equal(out.view(nb, tl, hw, c), dense[:, t0:t0 + tl]), f"block {(t0, tl)} differs from dense"


@pytest.mark.parametrize("hw,heads,T,world", [(64, 5, 5, 2), (16, 20, 18, 8), (256, 10, 18, 4), (4, 1, 7, 3)])
def test_temporal_attention_split_kv_equals_dense(hw, heads, T, world):
    from v3d_b200 import ops
    from v3d_b200.viewshard import ViewShard

    nb, c = 2, heads * 64
    g = torch.Generator(device=DEV).manual_seed(T * hw)
    qkv = torch.randn(nb, T, hw, 3 * c, device=DEV, generator=g).to(torch.bfloat16)
    dense = torch.empty(nb * T * hw, c, device=DEV, dtype=torch.bfloat16)
    ops.attention_temporal(qkv.view(-1, 3 * c), dense, nb, T, hw, heads, 0.125)
    dense = dense.view(nb, T, hw, c)
    shards = [ViewShard(num_frames=T, rank=r, world=world) for r in range(world)]
    tmax = shards[0].tmax
    # what all_gather_into_tensor would deliver: rank-major slots of nb*tmax*hw rows, each filled from row 0
    buf = torch.full((world * nb * tmax * hw, 2 * c), float("nan"), device=DEV, dtype=torch.bfloat16)
    for vs in shards:
        rows = nb * vs.tl * hw
        buf[vs.rank * nb * tmax * hw: vs.rank * nb * tmax * hw + rows] = \
            qkv[:, vs.frames].reshape(rows, 3 * c)[:, c:]
    for vs in shards:
        ql = qkv[:, vs.frames].reshape(nb * vs.tl * hw, 3 * c).contiguous()
        out = torch.empty(nb * vs.tl * hw, c, device=DEV, dtype=torch.bfloat16)
        row, bstride = vs.kv_table(nb, hw)
        ops.attention_temporal_kv(ql, buf, out, nb, vs.tl, hw, heads, row, bstride, 0.125)
        torch.cuda.synchronize()
        assert torch.equal(out.view(nb, vs.tl, hw, c), dense[:, vs.frames]), f"rank {vs.rank} differs from dense"


def test_single_rank_view_shard_equals_unsharded_engine():
    """world = 1 needs no process group: the frame-sharded code path (halo'd operands with zero halos, split-KV
    attention over its own frames, halo'd time_mix_conv) on one GPU must reproduce the dense path."""
    sys.path.insert(0, ROOT)
    from oracle import synth  # seeded weights / inputs only
    from v3d_b200 import engine
    from v3d_b200.viewshard import ViewShard

    T, hw = 5, 16
    cfg = engine.v3d_512_config(num_frames=T, num_steps=2, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = 64
    eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    unet.load_state_dict(synth.synth_state_dict(unet.param_shapes(), seed=11), strict=True)
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=12), strict=True)
    eng = eng.to(DEV).eval()
    x, c, uc = synth.synth_inputs(T, hw)
    c, uc = {k: v.to(DEV) for k, v in c.items()}, {k: v.to(DEV) for k, v in uc.items()}
    vs = ViewShard(num_frames=T, rank=0, world=1)
    ref = eng.sample_views(x.clone().to(DEV), c, uc, num_frames=T)
    one = eng.sample_views(x.clone().to(DEV), c, uc, num_frames=T, view_shard=vs)
    torch.cuda.synchronize()
    r = _rel(one, ref)
    print("world-1 shard vs dense: rel-L2", r, vs.exchanges)
    assert torch.isfinite(one).all() and r <= 3e-2, r      # fp64-atomic statistics order is the only difference


@pytest.mark.parametrize("M,K,C", [(1000, 320, 320), (16384, 640, 640), (4608, 1280, 1280)])
def test_gemm_kv_scatter_equals_output_columns(M, K, C):
    """Fused projection GEMM -> all-gather: the epilogue stores the K|V columns (>= C of the packed q|k|v output) a second
    time into every destination matrix - here two local buffers, one with a wider row stride; across GPUs the same
    stores go to IPC-mapped peer memory.  The copies must be bit-identical to the output columns, the output itself
    unchanged, rows past M untouched."""
    from v3d_b200 import ops

    g = torch.Generator(device=DEV).manual_seed(M + C)
    a = torch.randn(M, K, device=DEV, generator=g).to(torch.bfloat16)
    w = (torch.randn(3 * C, K, device=DEV, generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = torch.randn(3 * C, device=DEV, generator=g)
    ref = torch.empty(M, 3 * C, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, ref, K=K, N=3 * C, rows_per_batch=M, bias=bias)
    out = torch.empty_like(ref)
    d0 = torch.full((M + 64, 2 * C), 7.0, device=DEV, dtype=torch.bfloat16)
    d1 = torch.full((M + 64, 2 * C), 7.0, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, out, K=K, N=3 * C, rows_per_batch=M, bias=bias, kv=(C, [d0.data_ptr(), d1.data_ptr()], 2 * C))
    torch.cuda.synchronize()
    assert torch.equal(out, ref)
    for d in (d0, d1):
        assert torch.equal(d[:M], ref[:, C:]) and (d[M:] == 7.0).all()


# --------------------------------------------------------------------------------------------------------------
# model level
# --------------------------------------------------------------------------------------------------------------
def _engine_worker(rank: int, world: int, port: int, backend: str, one_gpu: bool, T: int, transport: str, q):
    sys.path.insert(0, ROOT)
    os.environ["V3D_SHARD_TRANSPORT"] = transport
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    from oracle import synth  # seeded weights / inputs only (test infrastructure)
    from v3d_b200 import engine
    from v3d_b200.viewshard import ViewShard

    dev = torch.device("cuda", 0 if one_gpu else rank)
    torch.cuda.set_device(dev)
    kw = {"device_id": dev} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    hw, steps = 16, 2
    cfg = engine.v3d_512_config(num_frames=T, num_steps=steps, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = 64
    eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    unet.load_state_dict(synth.synth_state_dict(unet.param_shapes(), seed=11), strict=True)
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=12), strict=True)
    eng = eng.to(dev).eval()
    x, c, uc = synth.synth_inputs(T, hw)
    to = lambda d: {k: v.to(dev) for k, v in d.items()}
    c, uc = to(c), to(uc)
    vs = ViewShard.create(T)
    res = {"rank": rank, "block": (vs.t0, vs.tl), "peer": vs.peer is not None}

    # one UNet forward, sharded vs unsharded
    xin = torch.cat([torch.cat([x.to(dev)] * 2), torch.cat([uc["concat"], c["concat"]])], 1)   # [2T, 8, hw, hw]
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    ts = torch.full((2 * T,), 0.7, device=dev)
    full = unet(xin, ts, ctx, y, None, T, torch.zeros(2, T, device=dev))
    pick = torch.cat([torch.arange(vs.t0, vs.t0 + vs.tl), T + torch.arange(vs.t0, vs.t0 + vs.tl)]).to(dev)
    unet.view_shard = vs
    try:
        part = unet(xin[pick], ts[pick], ctx[pick], y[pick], vs.time_context(c, uc), vs.tl,
                    torch.zeros(2, vs.tl, device=dev))
    finally:
        unet.view_shard = None
    res["unet_rel"] = _rel(part, full[pick])

    # the whole hot path: sampler loop + decode
    ref = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T)
    mine = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T, view_shard=vs)
    torch.cuda.synchronize()
    res["frames_rel"] = _rel(mine, ref[vs.frames])
    gathered = vs.gather_frames(mine)
    res["gathered_rel"] = _rel(gathered, ref)
    res["finite"] = bool(torch.isfinite(mine).all())
    res["exchanges"] = dict(vs.exchanges)
    q.put(res)
    dist.barrier()
    dist.destroy_process_group()


def _run_engine_pair(backend: str, one_gpu: bool, T: int = 5, world: int = 2, transport: str = "auto"):
    """transport: "auto" = one-sided peer memory over NCCL groups, torch.distributed collectives over gloo;
    "peer" / "nccl" force one (peer works between two processes on ONE GPU too: IPC-mapped memory of the same device)"""
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    from mp_util import run_workers

    res = sorted(run_workers(_engine_worker, world, (backend, one_gpu, T, transport), timeout=900),
                 key=lambda r: r["rank"])
    print(backend, transport, res)
    assert [r["block"] for r in res] == [(0, 3), (3, 2)]
    want_peer = transport == "peer" or (transport == "auto" and backend == "nccl")
    for r in res:
        assert r["peer"] == want_peer, r
        assert r["finite"]
        assert r["unet_rel"] <= 3e-2, r
        assert r["frames_rel"] <= 3e-2 and r["gathered_rel"] <= 3e-2, r
        # per forward: 2 norms + 2 halos per VideoResBlock, one K|V gather per SpatialVideoTransformer
        assert r["exchanges"]["kv_allgather"] > 0 and r["exchanges"]["halo"] >= r["exchanges"]["gn_allreduce"] > 0


def test_view_sharded_engine_matches_unsharded_one_gpu_gloo():
    _run_engine_pair("gloo", one_gpu=True)


def test_view_sharded_engine_peer_transport_one_gpu():
    """The one-sided peer-memory transport (csrc/peer.cu: IPC-mapped arenas, epoch flags, the sharded forward captured
    into a CUDA graph) between two processes that share cuda:0 - the arenas are mapped through the same IPC handles as
    across NVLink, so the whole protocol (sites, rotation, flags, statistics all-reduce) runs on a one-GPU box."""
    _run_engine_pair("gloo", one_gpu=True, transport="peer")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_view_sharded_engine_matches_unsharded_nccl():
    _run_engine_pair("nccl", one_gpu=False)                       # default transport over NCCL groups: peer memory


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_view_sharded_engine_matches_unsharded_nccl_collectives():
    _run_engine_pair("nccl", one_gpu=False, transport="nccl")    # torch.distributed collectives on the data path


# --------------------------------------------------------------------------------------------------------------
# CFG-pair split and composite plans (ShardPlan)
# --------------------------------------------------------------------------------------------------------------
def _plan_worker(rank: int, world: int, port: int, backend: str, one_gpu: bool, T: int, mode: str, transport: str, q):
    sys.path.insert(0, ROOT)
    os.environ["V3D_SHARD_TRANSPORT"] = transport
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    import torch.distributed as dist

    from oracle import synth  # seeded weights / inputs only (test infrastructure)
    from v3d_b200 import engine
    from v3d_b200.viewshard import ShardPlan

    dev = torch.device("cuda", 0 if one_gpu else rank)
    torch.cuda.set_device(dev)
    kw = {"device_id": dev} if backend == "nccl" else {}
    dist.init_process_group(backend, rank=rank, world_size=world, **kw)
    cfg = engine.v3d_512_config(num_frames=T, num_steps=2, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = 64
    eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    unet.load_state_dict(synth.synth_state_dict(unet.param_shapes(), seed=11), strict=True)
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=12), strict=True)
    eng = eng.to(dev).eval()
    x, c, uc = synth.synth_inputs(T, 16)
    c, uc = {k: v.to(dev) for k, v in c.items()}, {k: v.to(dev) for k, v in uc.items()}
    plan = ShardPlan.create(T, mode)
    ref = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T)
    mine = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T, shard=plan)
    torch.cuda.synchronize()
    gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "decode_block": (plan.decode.t0, plan.decode.tl), "finite": bool(torch.isfinite(mine).all()),
           "local_rel": _rel(mine, ref[plan.decode.frames]), "gathered_rel": _rel(gathered, ref),
           "plan": plan.describe()})
    dist.barrier()
    dist.destroy_process_group()


def _run_plan(mode: str, world: int, backend: str, one_gpu: bool, T: int = 5, transport: str = "auto"):
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker, world, (backend, one_gpu, T, mode, transport), timeout=900),
                 key=lambda r: r["rank"])
    print(mode, backend, transport, res)
    covered = []
    want_peer = transport == "peer" or (transport == "auto" and backend == "nccl")
    for r in res:
        assert r["plan"]["transport"].startswith("peer") == want_peer, r
        covered += list(range(r["decode_block"][0], sum(r["decode_block"])))
        assert r["finite"] and r["local_rel"] <= 3e-2 and r["gathered_rel"] <= 3e-2, r
        assert r["plan"]["exchanges"]["cfg_gather"] == 2
    assert covered == list(range(T))


@slow
def test_cfg_split_engine_matches_unsharded_one_gpu_gloo():
    _run_plan("cfg", 2, "gloo", one_gpu=True)


@slow
def test_cfg_views_engine_matches_unsharded_one_gpu_gloo():
    _run_plan("cfg+views", 4, "gloo", one_gpu=True)


def test_cfg_split_engine_peer_transport_one_gpu():
    _run_plan("cfg", 2, "gloo", one_gpu=True, transport="peer")


@pytest.mark.skipif(torch.cuda.device_count() < 4, reason="needs four GPUs: four processes that "
                    "spin-wait on each other's signals do not make progress under the time-slicing of ONE GPU")
def test_cfg_views_engine_peer_transport():
    _run_plan("cfg+views", 4, "nccl", one_gpu=False, transport="peer")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_cfg_split_engine_matches_unsharded_nccl():
    _run_plan("cfg", 2, "nccl", one_gpu=False)


@pytest.mark.skipif(torch.cuda.device_count() < 4, reason="needs four GPUs")
def test_cfg_views_engine_matches_unsharded_nccl():
    _run_plan("cfg+views", 4, "nccl", one_gpu=False)
