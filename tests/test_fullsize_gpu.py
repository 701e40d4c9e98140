"""Size-independent properties at BASELINE.json's FULL sizes (V3D_512: T = 18, B = 36, latent 64 x 64, width 320;
decode to 512 x 512), where the oracle is far too slow to be the checker:

  * the implicit 3x3 convolution (TMA gather, 9 taps) equals the explicit im2row + linear GEMM path on the same input -
    two independent operand-gather implementations of one contraction, same K order;
  * the wgmma flash attention equals its mma.sync twin at N = 4096 keys;
  * the halo'd-operand temporal conv over 8 uneven frame blocks equals the dense temporal conv, bit for bit;
  * a CFG-batched UNet forward (B = 36 = [uc; c]) equals two B = 18 forwards of its halves (nothing may leak between
    the two videos of a batch; exercises 32-bit row / offset arithmetic at the largest shapes);
  * the frame-sharded path with world = 1 equals the dense path for a full UNet forward and a full decode.
Random weights are generated on the device (init_random_), as in bench.py.
"""
import os
import sys
from pathlib import Path

import pytest
import torch

pytestmark = [pytest.mark.gpu]

ROOT = str(Path(__file__).resolve().parent.parent)
sys.path.insert(0, ROOT)
DEV = "cuda"
T, LAT = 18, 64


def _rel(a, b):
    a, b = a.float(), b.float()
    return ((a - b).norm() / b.norm().clamp_min(1e-12)).item()


def _bf(*shape, seed=0, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return (torch.randn(*shape, device=DEV, generator=g) * scale).to(torch.bfloat16)


@pytest.mark.parametrize("hw,cin,cout", [(64, 320, 320), (32, 640, 640), (16, 1280, 1280), (64, 960, 320)])
def test_implicit_conv_equals_im2row_gemm_full_size(hw, cin, cout):
    from v3d_b200 import ops

    n = 2 * T
    x = _bf(n * hw * hw, cin, seed=hw + cin)
    w = _bf(cout, 9 * cin, seed=1, scale=(9 * cin) ** -0.5)
    bias = torch.randn(cout, device=DEV)
    rows = n * hw * hw
    a = torch.empty(rows, cout, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, w, a, K=cin, N=cout, rows_per_batch=rows, bias=bias, conv=(n, hw, hw))
    col = torch.empty(rows, 9 * cin, device=DEV, dtype=torch.bfloat16)
    ops.im2col3x3(x, col, n, hw, hw, cin, 1, 1, hw, hw, 9 * cin)
    b = torch.empty(rows, cout, device=DEV, dtype=torch.bfloat16)
    ops.gemm(col, w, b, K=9 * cin, N=cout, rows_per_batch=rows, bias=bias)
    torch.cuda.synchronize()
    r = _rel(a, b)
    print("implicit vs im2row", (hw, cin, cout), "rel-L2", r, "equal", torch.equal(a, b))
    assert r <= 1e-3


def test_flash_attention_equals_mma_twin_full_size():
    from v3d_b200 import ops

    n, heads, ntok = 2 * T, 5, LAT * LAT
    qkv = _bf(n * ntok, 3 * heads * 64, seed=3)
    a = torch.empty(n * ntok, heads * 64, device=DEV, dtype=torch.bfloat16)
    b = torch.empty_like(a)
    ops.attention_spatial(qkv, a, n, ntok, heads, 0.125)
    ops.attention_spatial_mma(qkv, b, n, ntok, heads, 0.125)
    torch.cuda.synchronize()
    r = _rel(a, b)
    print("wgmma vs mma.sync attention at N=4096: rel-L2", r)
    assert r <= 1e-2                                   # two softmax formulations; bf16 P and output


def test_halo_temporal_conv_equals_dense_full_size():
    from v3d_b200 import ops
    from v3d_b200.viewshard import partition_frames

    nb, hw, c = 2, LAT * LAT, 320
    a = _bf(nb, T, hw, c, seed=5)
    w = _bf(c, 3 * c, seed=6, scale=(3 * c) ** -0.5)
    bias = torch.randn(c, device=DEV)
    dense = torch.empty(nb * T * hw, c, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a.view(-1, c), w, dense, K=c, N=c, rows_per_batch=T * hw, batch=nb, a_batch_stride=T * hw * c, bias=bias,
             ntaps=3, tap_shift=hw)
    dense = dense.view(nb, T, hw, c)
    for t0, tl in partition_frames(T, 8):
        pad = torch.zeros(nb, tl + 2, hw, c, device=DEV, dtype=torch.bfloat16)
        lo, hi = max(t0 - 1, 0), min(t0 + tl + 1, T)
        pad[:, lo - (t0 - 1): hi - (t0 - 1)] = a[:, lo:hi]
        out = torch.empty(nb * tl * hw, c, device=DEV, dtype=torch.bfloat16)
        ops.gemm(pad.view(-1, c), w, out, K=c, N=c, rows_per_batch=tl * hw, batch=nb,
                 a_batch_stride=(tl + 2) * hw * c, bias=bias, ntaps=3, tap_shift=hw, a_rows=(tl + 2) * hw, a_row0=hw)
        torch.cuda.synchronize()
        assert torch.equal(out.view(nb, tl, hw, c), dense[:, t0:t0 + tl]), (t0, tl)


def _full_unet():
    from v3d_b200 import engine
    from v3d_b200.unet import VideoUNet

    with torch.device("meta"):
        net = VideoUNet(**engine.v3d_512_config()["network_config"]["params"])
    return net.init_random_(torch.device(DEV), seed=100).eval()


def _unet_inputs(seed=23):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(2 * T, 8, LAT, LAT, device=DEV, generator=g)
    ts = torch.full((2 * T,), 0.9, device=DEV)
    ctx = torch.randn(2 * T, 1, 1024, device=DEV, generator=g)
    y = torch.randn(2 * T, 768, device=DEV, generator=g)
    return x, ts, ctx, y


def test_cfg_batched_forward_equals_its_halves_full_size():
    net = _full_unet()
    net.cuda_graphs = False
    x, ts, ctx, y = _unet_inputs()
    both = net(x, ts, ctx, y, None, T, torch.zeros(2, T, device=DEV))
    halves = [net(x[s], ts[s], ctx[s], y[s], None, T, torch.zeros(1, T, device=DEV))
              for s in (slice(0, T), slice(T, 2 * T))]
    torch.cuda.synchronize()
    r = _rel(torch.cat(halves), both)
    print("B=36 forward vs two B=18 forwards: rel-L2", r)
    assert torch.isfinite(both).all() and r <= 3e-2   # identical arithmetic up to the fp64-atomic statistics order


def test_single_rank_view_shard_equals_dense_full_size():
    from v3d_b200 import engine
    from v3d_b200.decoder import VideoDecoder
    from v3d_b200.viewshard import ViewShard

    vs = ViewShard(num_frames=T, rank=0, world=1)
    net = _full_unet()
    net.cuda_graphs = False
    x, ts, ctx, y = _unet_inputs()
    ind = torch.zeros(2, T, device=DEV)
    dense = net(x, ts, ctx, y, None, T, ind)
    net.view_shard = vs
    try:
        shard = net(x, ts, ctx, y, torch.stack([ctx[0], ctx[T]]), T, ind)
    finally:
        net.view_shard = None
    torch.cuda.synchronize()
    r = _rel(shard, dense)
    print("UNet, world-1 shard vs dense: rel-L2", r, vs.exchanges)
    assert r <= 3e-2
    del net
    torch.cuda.empty_cache()
    with torch.device("meta"):
        dec = VideoDecoder(**engine.v3d_512_config()["first_stage_config"]["params"]["decoder_config"]["params"])
    dec = dec.init_random_(torch.device(DEV), seed=200).eval()
    z = torch.randn(T, 4, LAT, LAT, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7))
    dense = dec(z, timesteps=T)
    dec.view_shard = vs
    try:
        shard = dec(z, timesteps=T)
    finally:
        dec.view_shard = None
    torch.cuda.synchronize()
    r = _rel(shard, dense)
    print("decoder, world-1 shard vs dense: rel-L2", r)
    assert shard.shape == (T, 3, 8 * LAT, 8 * LAT) and r <= 3e-2
