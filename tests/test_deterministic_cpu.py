"""Deterministic mode on the CPU: the C-ABI surface of the deterministic GroupNorm, the mode switch, and the HOST
SCHEDULES in deterministic mode with the kernels' CPU stand-ins (tests/emu_ops.py):

  * against the oracle, within the usual bf16 parity bound;
  * frame-sharded ('views') and CFG-split ('cfg') plans over gloo against the unsharded deterministic schedule:
    torch.equal (the statistics are block partials that depend on a block's rows only, all-gathered and folded in one
    fixed order, so no summation order depends on the plan).
"""
import os
import sys
from pathlib import Path

import pytest
import torch

ROOT = str(Path(__file__).resolve().parent.parent)
sys.path.insert(0, str(Path(__file__).resolve().parent))

from test_host_schedule_cpu import LAUNCHES, _build_decoder, _build_unet, _cos, _rel, _unet, _unet_inputs  # noqa: E402

NEW_SYMBOLS = ["v3d_groupnorm_det_blocks", "v3d_groupnorm_det_workspace_bytes", "v3d_groupnorm_partials",
               "v3d_groupnorm_fold_apply", "v3d_groupnorm_det"]


@pytest.fixture
def det_mode(monkeypatch):
    monkeypatch.setenv("V3D_DETERMINISTIC", "1")


def test_new_entry_points_are_declared_exported_and_bound():
    import ctypes

    from v3d_b200 import _lib

    header = (Path(ROOT) / "include" / "v3d_b200.h").read_text()
    raw = ctypes.CDLL(str(_lib.lib_path()))
    for n in NEW_SYMBOLS:
        assert n + "(" in header, n
        assert hasattr(raw, n), f"{n} not exported"
        assert n in _lib.SIGNATURES, f"{n} has no ctypes prototype"
    assert _lib.load().v3d_abi_version() == 1                      # additive: the ABI version is unchanged


@pytest.mark.parametrize("rows,hw", [(4096, 4096), (18 * 4096, 4096), (18 * 576, 576), (5 * 64, 64), (3 * 300, 300),
                                     (2 * 262144, 262144), (7, 7)])
def test_block_geometry_and_workspace_size_match_the_library(rows, hw):
    import emu_ops
    from v3d_b200 import ops

    assert ops.groupnorm_det_blocks(rows, hw) == emu_ops.groupnorm_det_blocks(rows, hw)
    assert ops.groupnorm_det_workspace_bytes(rows, hw, 3) == emu_ops.groupnorm_det_workspace_bytes(rows, hw, 3)
    r = min(256, hw)
    assert ops.groupnorm_det_blocks(rows, hw) == rows // hw * -(-hw // r)


def test_block_geometry_rejects_frames_that_do_not_tile():
    from v3d_b200 import _lib, ops

    assert _lib.load().v3d_groupnorm_det_blocks(1000, 300) == -1
    with pytest.raises(RuntimeError, match="does not divide"):
        ops.groupnorm_det_blocks(1000, 300)


def test_mode_switch(monkeypatch):
    from v3d_b200 import ops

    monkeypatch.delenv("V3D_DETERMINISTIC", raising=False)
    assert not torch.are_deterministic_algorithms_enabled() and not ops.deterministic()
    monkeypatch.setenv("V3D_DETERMINISTIC", "1")
    assert ops.deterministic()
    monkeypatch.setenv("V3D_DETERMINISTIC", "0")
    assert not ops.deterministic()
    try:
        torch.use_deterministic_algorithms(True)
        assert ops.deterministic()
    finally:
        torch.use_deterministic_algorithms(False)


def test_graph_cache_key_includes_the_mode(monkeypatch):
    net, _ = _build_unet()
    dev = torch.device("cpu")
    monkeypatch.delenv("V3D_DETERMINISTIC", raising=False)
    default = net._graph_key(36, 18, 64, 64, dev)
    assert default == (36, 18, 64, 64, None)                      # unchanged in the default mode
    monkeypatch.setenv("V3D_DETERMINISTIC", "1")
    assert net._graph_key(36, 18, 64, 64, dev) != default


def test_frame_subset_partials_equal_the_whole_tensors():
    import emu_ops

    g = torch.Generator().manual_seed(3)
    nb, T, hw, c = 2, 5, 300, 64                                   # blocks of 256 + 44 rows per frame
    x = torch.randn(nb, T, hw, c, generator=g).to(torch.bfloat16)
    full = emu_ops.block_pairs(x.view(-1, c), T * hw, hw, nb, c)
    sub = emu_ops.block_pairs(x[:, 2:4].contiguous().view(-1, c), 2 * hw, hw, nb, c)
    assert full.shape == (nb, T * 2, 32, 2)
    assert torch.equal(sub, full[:, 4:8])


def test_det_schedule_selects_the_deterministic_kernels(det_mode):
    """In deterministic mode no norm takes the atomic statistics; the 2-D norms take the single launch, the 3-D norms
    the pair (the same selection as the default mode), and V3D_GN_FUSED=0 moves everything to the pair."""
    import emu_ops

    T, hw = 4, 8                                                  # B = 8 samples: the 2-D norms take one launch
    net, _ = _build_unet()
    xin, ts, ctx, y = _unet_inputs(T, hw)
    names = ["groupnorm_stats", "groupnorm", "groupnorm_det", "groupnorm_partials", "groupnorm_fold_apply"]

    def norm_calls(since):
        return {n: k for n, k in (launches - since).items() if n in names}

    with emu_ops.patched() as launches:
        n0 = launches.copy()
        _unet(net, xin, ts, ctx, y, T)
        first = norm_calls(n0)
        n1 = launches.copy()
        os.environ["V3D_GN_FUSED"] = "0"
        try:
            _unet(net, xin, ts, ctx, y, T)
        finally:
            del os.environ["V3D_GN_FUSED"]
        calls = norm_calls(n1)
    assert first == {"groupnorm_det": 61, "groupnorm_partials": 44, "groupnorm_fold_apply": 44}, first
    assert calls == {"groupnorm_partials": 105, "groupnorm_fold_apply": 105}, calls


def test_det_unet_and_decoder_schedules_match_oracle(det_mode):
    import emu_ops
    from oracle import ref_decoder, ref_unet

    T, hw = 3, 16
    net, sd = _build_unet()
    xin, ts, ctx, y = _unet_inputs(T, hw)
    calls = []
    with emu_ops.patched(calls):
        out = _unet(net, xin, ts, ctx, y, T)
    with torch.no_grad():
        ref = ref_unet.unet_forward(sd, ref_unet.UNetSpec(model_channels=64), xin, ts, ctx, y, T, torch.zeros(2, T))
    r, cs = _rel(out, ref), _cos(out, ref)
    print("det unet schedule vs oracle: rel-L2", r, "cos", cs, "launches", emu_ops.digest(calls))
    assert r <= 3e-2 and cs >= 0.999, (r, cs)
    assert emu_ops.digest(calls) == LAUNCHES["unet_t3_deterministic"]

    dec, sdd = _build_decoder()
    z = torch.randn(T, 4, 8, 8, generator=torch.Generator().manual_seed(3))
    calls = []
    with emu_ops.patched(calls):
        out = dec(z, timesteps=T)
    with torch.no_grad():
        ref = ref_decoder.decoder_forward(sdd, ref_decoder.DecoderSpec(ch=64), z, T)
    r, cs = _rel(out, ref), _cos(out, ref)
    print("det decoder schedule vs oracle: rel-L2", r, "cos", cs, "launches", emu_ops.digest(calls))
    assert r <= 3e-2 and cs >= 0.999, (r, cs)
    assert emu_ops.digest(calls) == LAUNCHES["decoder_t3_deterministic"]


# ---------------------------------------------------------------------------------------------------------------
# sharded plans vs the unsharded schedule, deterministic mode, over gloo
# ---------------------------------------------------------------------------------------------------------------
def _views_worker(rank: int, world: int, port: int, T: int, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port), V3D_DETERMINISTIC="1")
    import torch.distributed as dist

    import emu_ops
    from v3d_b200.viewshard import ViewShard

    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    vs = ViewShard.create(T)
    res = {"rank": rank, "block": (vs.t0, vs.tl)}
    pick = torch.cat([torch.arange(vs.t0, vs.t0 + vs.tl), T + torch.arange(vs.t0, vs.t0 + vs.tl)])
    with emu_ops.patched():
        net, _ = _build_unet()
        xin, ts, ctx, y = _unet_inputs(T, 16)
        full = _unet(net, xin, ts, ctx, y, T)
        tc = torch.stack([ctx[0], ctx[T]])
        net.view_shard = vs
        try:
            part = net(xin[pick], ts[pick], ctx[pick], y[pick], time_context=tc, num_video_frames=vs.tl,
                       image_only_indicator=torch.zeros(2, vs.tl))
        finally:
            net.view_shard = None
        res["unet_equal"] = torch.equal(part, full[pick])
        res["unet_exchanges"] = dict(vs.exchanges)

        dec, _ = _build_decoder()
        z = torch.randn(T, 4, 8, 8, generator=torch.Generator().manual_seed(3))
        full_d = dec(z, timesteps=T)
        dec.view_shard = vs
        try:
            part_d = dec(z[vs.frames].contiguous(), timesteps=vs.tl)
        finally:
            dec.view_shard = None
        res["dec_equal"] = torch.equal(vs.gather_frames(part_d), full_d)
    q.put(res)
    dist.barrier()
    dist.destroy_process_group()


def test_det_view_sharded_schedules_equal_unsharded_gloo():
    from mp_util import run_workers

    world, T = 2, 5
    res = sorted(run_workers(_views_worker, world, (T,), timeout=900), key=lambda r: r["rank"])
    print(res)
    assert [r["block"] for r in res] == [(0, 3), (3, 2)]
    for r in res:
        assert r["unet_equal"] and r["dec_equal"], r
        # the statistics all-reduce becomes an all-gather of the block partials: one per 3-D norm
        assert r["unet_exchanges"] == {"gn_allgather": 44, "halo": 44, "kv_allgather": 16}, r


def _plan_worker(rank: int, world: int, port: int, T: int, mode: str, q):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, str(Path(ROOT) / "tests"))
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port), V3D_DETERMINISTIC="1")
    import torch.distributed as dist

    import cpu_shims
    import emu_ops
    from oracle import synth
    from v3d_b200.viewshard import ShardPlan

    torch.set_num_threads(2)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    plan = ShardPlan.create(T, mode)
    eng, _, _ = cpu_shims.cpu_engine(T, 2)
    x, c, uc = synth.synth_inputs(T, 8)
    g = torch.Generator().manual_seed(5)
    c = dict(c, crossattn=c["crossattn"] + 0.5 * torch.randn(T, 1, 1024, generator=g))
    with emu_ops.patched():
        ref = eng.sample_views(x.clone(), c, uc, num_frames=T)
        mine = eng.sample_views(x.clone(), c, uc, num_frames=T, shard=plan)
        gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "equal": torch.equal(gathered, ref), "plan": plan.describe()})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("mode,T", [("views", 5), ("cfg", 4)])
def test_det_plans_equal_unsharded_sample_views_gloo(mode, T):
    """sample_views under the 'views' and 'cfg' plans (CFG split: the 2-D norms see half the samples, the 3-D norms
    one video instead of two) gives exactly the unsharded deterministic frames."""
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker, 2, (T, mode), timeout=900), key=lambda r: r["rank"])
    print(res)
    for r in res:
        assert r["equal"], r
        if mode == "views":
            assert r["plan"]["exchanges"]["gn_allgather"] == 2 * 44 + 28 and "gn_allreduce" not in r["plan"]["exchanges"]
