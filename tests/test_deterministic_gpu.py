"""Deterministic mode on the GPU (V3D_DETERMINISTIC=1 or torch.use_deterministic_algorithms(True)).

Kernels: the block partials and the fold against fp64; the partials of a frame subset equal those of the same frames
inside the whole tensor; the single launch equals the pair; the output does not change with nsamples or V3D_GN_WAVES.
Engine: sample_views and views_from_image give the same bytes run to run and in a fresh process; the 'views' and 'cfg'
plans (two processes sharing cuda:0, over the peer transport and over gloo) give exactly the unsharded frames; parity
against the golden fixtures holds in this mode too.
"""
import os
import subprocess
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

pytestmark = [pytest.mark.gpu]

ROOT = str(Path(__file__).resolve().parent.parent)
TESTS = str(Path(__file__).resolve().parent)
sys.path[:0] = [ROOT, TESTS]
DEV = "cuda"


@pytest.fixture
def det_mode(monkeypatch):
    monkeypatch.setenv("V3D_DETERMINISTIC", "1")


def _x(ns, rows, c, seed, ldx=None):
    g = torch.Generator(device=DEV).manual_seed(seed)
    ld = c if ldx is None else ldx
    x = (torch.randn(ns * rows, ld, device=DEV, generator=g) * 1.5 + 0.3).to(torch.bfloat16)
    return x if ldx is None else x[:, :c]


def _affine(c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed + 1)
    return 1 + 0.1 * torch.randn(c, device=DEV, generator=g), 0.1 * torch.randn(c, device=DEV, generator=g)


def _pairs_f64(x, rows, hw, ns, c):
    """fp64 (sum, sumsq) per (block, group), blocks of min(256, hw) rows inside each frame"""
    frames, r = rows // hw, min(256, hw)
    nbf = -(-hw // r)
    v = x.reshape(ns, frames, hw, c).double()
    v = F.pad(v, (0, 0, 0, nbf * r - hw)).reshape(ns, frames * nbf, r, 32, c // 32)
    return v.sum(dim=(2, 4)), (v * v).sum(dim=(2, 4)), v.abs().sum(dim=(2, 4))


SHAPES = [(2, 18, 4096, 320), (36, 1, 4096, 320), (8, 1, 1024, 640), (2, 5, 576, 1280), (3, 4, 64, 2560),
          (2, 3, 300, 64)]


@pytest.mark.parametrize("ns,T,hw,c", SHAPES)
def test_partials_and_fold_match_fp64(ns, T, hw, c):
    from v3d_b200 import ops

    rows = T * hw
    x = _x(ns, rows, c, seed=hw + c)
    nblk = ops.groupnorm_det_blocks(rows, hw)
    part = torch.empty(ns, nblk, 32, 2, device=DEV)
    ops.groupnorm_partials(x, part, rows, hw, ns, c)
    s, q, a = _pairs_f64(x, rows, hw, ns, c)
    es = ((part[..., 0].double() - s).norm() / a.norm()).item()
    eq = ((part[..., 1].double() - q).norm() / q.norm()).item()
    print((ns, T, hw, c), "partials: sum", es, "sumsq", eq)
    assert es <= 1e-6 and eq <= 1e-6
    # fold + apply against fp32 ATen GroupNorm over the same rows (bf16 output)
    gamma, beta = _affine(c, hw)
    y = torch.empty(ns * rows, c, device=DEV, dtype=torch.bfloat16)
    ops.groupnorm_fold_apply(x, y, part, gamma, beta, rows, ns, c, 1e-5, False, nblk)
    ref = F.group_norm(x.float().view(ns, rows, c).permute(0, 2, 1), 32, gamma, beta, 1e-5).permute(0, 2, 1)
    ref = ref.reshape(-1, c)
    err = ((y.float() - ref).norm() / ref.norm()).item()
    assert err <= 4e-3 and (y.float() - ref).abs().max().item() <= 0.05, err


@pytest.mark.parametrize("hw,c,T", [(4096, 320, 18), (576, 640, 5), (64, 1280, 7), (300, 128, 4)])
def test_frame_subset_partials_bit_identical(hw, c, T):
    from v3d_b200 import ops

    nb = 2
    x = _x(nb, T * hw, c, seed=7 * T)
    nbf = ops.groupnorm_det_blocks(hw, hw)
    full = torch.empty(nb, T * nbf, 32, 2, device=DEV)
    ops.groupnorm_partials(x, full, T * hw, hw, nb, c)
    for t0, tl in [(0, 1), (1, T - 2), (T - 2, 2)]:
        sub = x.view(nb, T, hw, c)[:, t0:t0 + tl].contiguous().view(-1, c)
        got = torch.full_like(full, float("nan"))
        ops.groupnorm_partials(sub, got[:, t0 * nbf:], tl * hw, hw, nb, c, ldp=T * nbf)   # at the global offset
        assert torch.equal(got[:, t0 * nbf:(t0 + tl) * nbf], full[:, t0 * nbf:(t0 + tl) * nbf]), (t0, tl)
        assert torch.isnan(got[:, :t0 * nbf]).all() and torch.isnan(got[:, (t0 + tl) * nbf:]).all()


def _pair(ops, x, rows, hw, ns, c, gamma, beta, silu, ldx=None):
    nblk = ops.groupnorm_det_blocks(rows, hw)
    part = torch.empty(ns, nblk, 32, 2, device=DEV)
    ops.groupnorm_partials(x, part, rows, hw, ns, c, ldx=ldx)
    y = torch.empty(ns * rows, c, device=DEV, dtype=torch.bfloat16)
    return ops.groupnorm_fold_apply(x, y, part, gamma, beta, rows, ns, c, 1e-5, silu, nblk, ldx=ldx)


def _fused(ops, x, rows, hw, ns, c, gamma, beta, silu, ldx=None, ws=None):
    if ws is None:
        ws = ops.groupnorm_det_workspace(DEV, ops.groupnorm_det_workspace_bytes(rows, hw, ns))
    y = torch.empty(ns * rows, c, device=DEV, dtype=torch.bfloat16)
    return ops.groupnorm_det(x, y, gamma, beta, rows, hw, ns, c, 1e-5, silu, ws, ldx=ldx)


@pytest.mark.parametrize("ns,T,hw,c", SHAPES)
@pytest.mark.parametrize("silu", [False, True])
def test_single_launch_equals_pair(ns, T, hw, c, silu):
    from v3d_b200 import ops

    rows = T * hw
    gamma, beta = _affine(c, c)
    x = _x(ns, rows, c, seed=c + ns)
    ws = ops.groupnorm_det_workspace(DEV, ops.groupnorm_det_workspace_bytes(rows, hw, ns))
    a = _fused(ops, x, rows, hw, ns, c, gamma, beta, silu, ws=ws)
    b = _pair(ops, x, rows, hw, ns, c, gamma, beta, silu)
    again = _fused(ops, x, rows, hw, ns, c, gamma, beta, silu, ws=ws)      # the barrier state is reused
    assert torch.equal(a, b) and torch.equal(a, again)
    xs = _x(ns, rows, c, seed=c + ns, ldx=c + 64)                            # row stride > C
    assert torch.equal(_fused(ops, xs, rows, hw, ns, c, gamma, beta, silu, ldx=c + 64),
                       _pair(ops, xs.contiguous(), rows, hw, ns, c, gamma, beta, silu))


def test_output_does_not_depend_on_nsamples():
    from v3d_b200 import ops

    c, hw = 320, 4096
    gamma, beta = _affine(c, 1)
    x = _x(36, hw, c, seed=5)
    whole = _fused(ops, x, hw, hw, 36, c, gamma, beta, True)
    assert torch.equal(whole, _pair(ops, x, hw, hw, 36, c, gamma, beta, True))
    for s0, n in [(0, 18), (18, 18), (5, 1), (9, 8)]:
        xs = x[s0 * hw:(s0 + n) * hw]
        ref = whole[s0 * hw:(s0 + n) * hw]
        assert torch.equal(_pair(ops, xs, hw, hw, n, c, gamma, beta, True), ref), (s0, n)
        assert torch.equal(_fused(ops, xs, hw, hw, n, c, gamma, beta, True), ref), (s0, n)
    # a 3-D norm's two videos, together and one at a time
    x3 = _x(2, 18 * hw, c, seed=6)
    both = _pair(ops, x3, 18 * hw, hw, 2, c, gamma, beta, True)
    one = _pair(ops, x3[18 * hw:], 18 * hw, hw, 1, c, gamma, beta, True)
    assert torch.equal(both[18 * hw:], one)


_WAVES_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import test_deterministic_gpu as t
from v3d_b200 import ops
out = {{}}
for ns, T, hw, c in [(2, 18, 4096, 320), (36, 1, 4096, 320), (8, 1, 1024, 640)]:
    gamma, beta = t._affine(c, c)
    x = t._x(ns, T * hw, c, seed=c + ns)
    out[(ns, c, "pair")] = t._pair(ops, x, T * hw, hw, ns, c, gamma, beta, True).cpu()
    out[(ns, c, "fused")] = t._fused(ops, x, T * hw, hw, ns, c, gamma, beta, True).cpu()
torch.save(out, sys.argv[1])
"""


def test_output_does_not_depend_on_gn_waves(tmp_path):
    """V3D_GN_WAVES (read once per process) sets the row chunking of the apply grid: a fresh process per value."""
    script = _WAVES_SCRIPT.format(root=ROOT, tests=TESTS)
    results = []
    for waves in ("1", "4", "9"):
        path = tmp_path / f"w{waves}.pt"
        env = dict(os.environ, V3D_GN_WAVES=waves)
        subprocess.run([sys.executable, "-c", script, str(path)], check=True, env=env, cwd=ROOT, timeout=600)
        results.append(torch.load(path))
    for k in results[0]:
        assert torch.equal(results[0][k], results[0][(k[0], k[1], "pair")]), k
        for r in results[1:]:
            assert torch.equal(results[0][k], r[k]), k


# --------------------------------------------------------------------------------------------------------------
# engine level
# --------------------------------------------------------------------------------------------------------------
T_FULL, LAT = 18, 64


def _full_engine(native_encoder: bool, steps: int):
    from v3d_b200 import conditioning, engine

    cfg = engine.v3d_512_config(num_frames=T_FULL, num_steps=steps)
    if native_encoder:
        fs = cfg["first_stage_config"]["params"]
        fs["encoder_config"] = {"target": "v3d_b200.sgm.modules.diffusionmodules.model.Encoder",
                                "params": dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256,
                                               in_channels=3, out_ch=3, ch=128, ch_mult=[1, 2, 4, 4],
                                               num_res_blocks=2, attn_resolutions=[], dropout=0.0)}
        fs["regularizer_config"] = {"target": "v3d_b200.encoder.DiagonalGaussianRegularizer",
                                    "params": {"sample": True}}
    with torch.device("meta"):
        eng = engine.DiffusionEngine(**cfg)
    dev = torch.device(DEV, 0)
    eng.model.diffusion_model.init_random_(dev, seed=100)
    eng.first_stage_model.decoder.init_random_(dev, seed=101)
    if native_encoder:
        eng.first_stage_model.encoder.init_random_(dev, seed=102)
        eng.conditioner = conditioning.GeneralConditioner(conditioning.V3D_512_EMB_MODELS).to(dev)
    return eng.eval()


def _capture_latents(eng):
    seen = []
    decode = eng.decode_first_stage

    def recording(z):
        seen.append(z.clone())
        return decode(z)
    eng.decode_first_stage = recording
    return seen


def _u8(frames):
    from v3d_b200 import ops

    t, _, h, w = frames.shape
    return ops.frames_nchw_to_u8(frames.float().contiguous(), torch.empty(t, h, w, 3, device=frames.device,
                                                                         dtype=torch.uint8))


def _views_once(eng=None, seen=None):
    """sample_views, T = 18, latent 64 x 64, 25 steps, random weights -> (latents, uint8 frames) on the CPU"""
    from oracle import synth

    if eng is None:
        eng = _full_engine(False, 25)
        seen = _capture_latents(eng)
    x, c, uc = synth.synth_inputs(T_FULL, LAT)
    to = lambda d: {k: v.to(DEV) for k, v in d.items()}
    frames = eng.sample_views(x.to(DEV), to(c), to(uc), num_frames=T_FULL)
    return seen[-1].cpu(), _u8(frames).cpu()


def _from_image_once(eng=None):
    from v3d_b200 import pipeline

    if eng is None:
        eng = _full_engine(True, 4)
    g = torch.Generator().manual_seed(31)
    image = (torch.rand(1, 3, 8 * LAT, 8 * LAT, generator=g) * 2 - 1).to(DEV)
    clip_emb = torch.randn(1, 1, 1024, generator=g).to(DEV)
    torch.manual_seed(23)
    frames = pipeline.views_from_image(eng, image, clip_emb, num_frames=T_FULL, fps_id=6, motion_bucket_id=127,
                                       cond_aug=0.02)
    return _u8(frames).cpu()


_FRESH_SCRIPT = r"""
import sys, torch
sys.path[:0] = [{root!r}, {tests!r}]
import test_deterministic_gpu as t
torch.save({{"views": t._views_once(), "from_image": t._from_image_once()}}, sys.argv[1])
"""


def test_same_seed_same_bytes_across_runs_and_processes(det_mode, tmp_path):
    eng = _full_engine(False, 25)
    seen = _capture_latents(eng)
    z1, f1 = _views_once(eng, seen)
    z2, f2 = _views_once(eng, seen)              # the second call replays captured CUDA graphs
    eng_img = _full_engine(True, 4)
    i1, i2 = _from_image_once(eng_img), _from_image_once(eng_img)
    path = tmp_path / "fresh.pt"
    subprocess.run([sys.executable, "-c", _FRESH_SCRIPT.format(root=ROOT, tests=TESTS), str(path)], check=True,
                   env=dict(os.environ, V3D_DETERMINISTIC="1"), cwd=ROOT, timeout=1200)
    fresh = torch.load(path)
    assert torch.isfinite(z1).all() and f1.float().std() > 1.0
    assert torch.equal(z1, z2) and torch.equal(f1, f2)
    assert torch.equal(z1, fresh["views"][0]) and torch.equal(f1, fresh["views"][1])
    assert torch.equal(i1, i2) and torch.equal(i1, fresh["from_image"])


def test_torch_switch_selects_the_mode():
    """torch.use_deterministic_algorithms(True) alone gives the same bytes as V3D_DETERMINISTIC=1."""
    from oracle import synth
    from v3d_b200 import engine

    T = 4
    cfg = engine.v3d_512_config(num_frames=T, num_steps=2, min_cfg=1.5, max_cfg=3.5)
    cfg["network_config"]["params"]["model_channels"] = 64
    cfg["first_stage_config"]["params"]["decoder_config"]["params"]["ch"] = 64
    eng = engine.DiffusionEngine(**cfg)
    unet, dec = eng.model.diffusion_model, eng.first_stage_model.decoder
    unet.load_state_dict(synth.synth_state_dict(unet.param_shapes(), seed=11), strict=True)
    dec.load_state_dict(synth.synth_state_dict(dec.param_shapes(), seed=12), strict=True)
    eng = eng.to(DEV).eval()
    x, c, uc = synth.synth_inputs(T, 16)
    to = lambda d: {k: v.to(DEV) for k, v in d.items()}
    os.environ["V3D_DETERMINISTIC"] = "1"
    try:
        a = eng.sample_views(x.clone().to(DEV), to(c), to(uc), num_frames=T)
    finally:
        del os.environ["V3D_DETERMINISTIC"]
    torch.use_deterministic_algorithms(True, warn_only=True)
    try:
        b = eng.sample_views(x.clone().to(DEV), to(c), to(uc), num_frames=T)
    finally:
        torch.use_deterministic_algorithms(False)
    assert torch.equal(a, b)


def _plan_worker(rank: int, world: int, port: int, backend: str, one_gpu: bool, T: int, mode: str, transport: str, q):
    sys.path.insert(0, ROOT)
    os.environ["V3D_SHARD_TRANSPORT"] = transport
    os.environ.update(RANK=str(rank), LOCAL_RANK=str(rank), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port), V3D_DETERMINISTIC="1")
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
    g = torch.Generator().manual_seed(5)
    c = dict(c, crossattn=c["crossattn"] + 0.5 * torch.randn(T, 1, 1024, generator=g))     # frames differ
    c, uc = {k: v.to(dev) for k, v in c.items()}, {k: v.to(dev) for k, v in uc.items()}
    plan = ShardPlan.create(T, mode)
    ref = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T)
    mine = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T, shard=plan)
    again = eng.sample_views(x.clone().to(dev), c, uc, num_frames=T, shard=plan)       # graph replay (peer transport)
    torch.cuda.synchronize()
    plan.check_status()
    gathered = plan.gather_frames(mine)
    q.put({"rank": rank, "equal": torch.equal(gathered.cpu(), ref.cpu()), "again": torch.equal(again, mine),
           "plan": plan.describe()})
    dist.barrier()
    dist.destroy_process_group()


def _run_plan(mode: str, world: int, backend: str, one_gpu: bool, transport: str, T: int = 5):
    from mp_util import run_workers

    res = sorted(run_workers(_plan_worker, world, (backend, one_gpu, T, mode, transport), timeout=900),
                 key=lambda r: r["rank"])
    print(mode, backend, transport, res)
    want_peer = transport == "peer" or (transport == "auto" and backend == "nccl")
    for r in res:
        assert r["plan"]["transport"].startswith("peer") == want_peer, r
        assert r["equal"] and r["again"], r
        if mode == "views":
            assert r["plan"]["exchanges"]["gn_allgather"] > 0 and "gn_allreduce" not in r["plan"]["exchanges"], r


@pytest.mark.parametrize("mode", ["views", "cfg"])
@pytest.mark.parametrize("transport", ["peer", "auto"])
def test_plans_equal_unsharded_one_gpu(mode, transport):
    """Two processes sharing cuda:0: 'peer' = the one-sided IPC transport, 'auto' over gloo = torch.distributed
    collectives staged through the host."""
    _run_plan(mode, 2, "gloo", one_gpu=True, transport=transport)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
@pytest.mark.parametrize("mode", ["views", "cfg"])
@pytest.mark.parametrize("transport", ["auto", "nccl"])
def test_plans_equal_unsharded_nccl(mode, transport):
    _run_plan(mode, 2, "nccl", one_gpu=False, transport=transport)


@pytest.mark.skipif(torch.cuda.device_count() < 4, reason="needs four GPUs")
def test_cfg_views_plan_equals_unsharded_nccl():
    _run_plan("cfg+views", 4, "nccl", one_gpu=False, transport="auto")


# --------------------------------------------------------------------------------------------------------------
# parity against the golden fixtures, in deterministic mode
# --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["unet_small", "unet_full", "unet_v3d512"])
def test_det_unet_parity(det_mode, tag):
    import test_parity_gpu

    test_parity_gpu.test_unet_forward_matches_reference(tag)


@pytest.mark.parametrize("tag", ["decoder_small_2videos", "decoder_full"])
def test_det_decoder_parity(det_mode, tag):
    import test_parity_gpu

    test_parity_gpu.test_decoder_matches_reference(tag)


def test_det_decoder_v3d512_and_encoder_parity(det_mode):
    import test_parity_gpu

    test_parity_gpu.test_decoder_matches_reference_v3d512()
    test_parity_gpu.test_encoder_matches_reference("encoder_full")
