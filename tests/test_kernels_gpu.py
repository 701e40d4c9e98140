"""Per-kernel parity tests on the GPU, every call through the C ABI (v3d_b200.ops -> libv3d_b200.so).

The checker for a single op is the fp32 ATen implementation of the same op on the same bf16-rounded
inputs (the reference's own kernels on this path are ATen calls, SURVEY.md §2.1); block- and model-level
parity against the reference modules lives in test_parity_gpu.py with committed golden fixtures.
Tolerances: outputs are bf16 (8 mantissa bits) -> |err| <= 2^-8 * |ref| + small absolute slack, stated per test.
"""
import math
import os

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

ops = None


@pytest.fixture(scope="module", autouse=True)
def _load():
    global ops
    from v3d_b200 import ops as _ops

    ops = _ops
    torch.manual_seed(0)
    yield


DEV = "cuda"


def bf(x):
    return x.to(torch.bfloat16)


def rnd(*shape, scale=1.0):
    return bf(torch.randn(*shape, device=DEV) * scale)


def assert_close(got, ref, rtol=1.0 / 128, atol=2e-2, what=""):
    got = got.float()
    ref = ref.float()
    err = (got - ref).abs()
    tol = atol + rtol * ref.abs()
    bad = err > tol
    if bad.any():
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(
            f"{what}: {int(bad.sum())}/{bad.numel()} elements out of tolerance; max err {err.max().item():.4g}; "
            f"first bad at {idx}: got {got[tuple(idx)].item():.5g} ref {ref[tuple(idx)].item():.5g}; "
            f"rel-l2 {((got - ref).norm() / ref.norm().clamp_min(1e-12)).item():.3g}")


# --------------------------------------------------------------------------------------------
# tensor-core (wgmma) GEMM: linear mode
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,K,N", [
    (128, 64, 16), (128, 64, 64), (128, 128, 128), (256, 320, 320), (384, 1280, 1280),
    (200, 64, 32),      # M tail
    (2304, 1280, 640),  # persistent multi-tile per CTA
    (36, 320, 1280),    # M < one tile
    (1024, 2560, 1280),
])
def test_gemm_linear(M, K, N):
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, out, K=K, N=N, rows_per_batch=M, bias=bias)
    ref = a.float() @ w.float().t() + bias
    assert_close(out, ref, what=f"gemm {M}x{K}x{N}")


@pytest.mark.parametrize("bn", [16, 32, 64, 128, 160, 256])
def test_gemm_block_n_variants(bn):
    M, K = 512, 192
    N = bn * 3
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    out = torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, out, K=K, N=N, rows_per_batch=M, block_n=bn)
    assert_close(out, a.float() @ w.float().t(), what=f"gemm bn={bn}")


def test_gemm_epilogue_full():
    """bias + per-frame bias + scaled residuals + strided output slice + fp32 output."""
    M, K, N, rpf = 768, 128, 320, 256
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    fbias = torch.randn(M // rpf, N, device=DEV)
    r1, r2 = rnd(M, N), rnd(M, N + 64)
    core = a.float() @ w.float().t() + bias + fbias.repeat_interleave(rpf, 0)
    ref = 0.3 * core + 1.0 * r1.float() + 0.7 * r2.float()[:, :N]
    big = torch.zeros(M, N + 128, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, big[:, 64:], K=K, N=N, rows_per_batch=M, ldd=N + 128, bias=bias, fbias=fbias,
             rows_per_frame=rpf, r1=r1, ldr1=N, r2=r2, ldr2=N + 64, s0=0.3, s1=1.0, s2=0.7)
    assert_close(big[:, 64:64 + N], ref, what="epilogue bf16")
    assert big[:, :64].abs().max() == 0 and big[:, 64 + N:].abs().max() == 0
    o32 = torch.empty(M, N, device=DEV, dtype=torch.float32)
    ops.gemm(a, w, o32, K=K, N=N, rows_per_batch=M, bias=bias, act=ops.ACT_SILU)
    assert_close(o32, F.silu(a.float() @ w.float().t() + bias), rtol=1e-3, atol=1e-3, what="epilogue fp32 silu")


@pytest.mark.parametrize("N", [320, 256, 128, 64])
@pytest.mark.parametrize("inplace", [False, True])
def test_gemm_single_residual_many_tiles(N, inplace):
    """bf16 output + one residual over far more tiles than SMs (every CTA walks several tiles and reuses its staging
    buffer once the previous tile's TMA stores have read it; N = 320 gives an odd number of 32-column sub-tiles), residual
    separate or in place (out is r1, the transformer's `t = t + f(t)` pattern), row tail included."""
    M, K = 128 * 500 + 40, 64
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    r1 = rnd(M, N)
    ref = 0.5 * (a.float() @ w.float().t() + bias) + 0.75 * r1.float()
    out = r1.clone() if inplace else torch.empty(M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, out, K=K, N=N, rows_per_batch=M, bias=bias, r1=out if inplace else r1, s0=0.5, s1=0.75)
    assert_close(out, ref, what=f"single residual N={N} inplace={inplace}")


@pytest.mark.parametrize("n_out", [1280, 2560, 256])
def test_gemm_geglu(n_out):
    M, K = 512, 320
    proj = torch.randn(2 * n_out, K, device=DEV) * K ** -0.5
    pb = torch.randn(2 * n_out, device=DEV)
    a = rnd(M, K)
    bn = ops.pick_block_n(2 * n_out, ops.ACT_GEGLU)
    perm = ops.geglu_perm(n_out, bn).to(DEV)
    wp, bp = bf(proj[perm]).contiguous(), pb[perm].contiguous()
    out = torch.empty(M, n_out, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, wp, out, K=K, N=2 * n_out, rows_per_batch=M, bias=bp, act=ops.ACT_GEGLU)
    y = a.float() @ bf(proj).float().t() + pb
    v, g = y.chunk(2, dim=-1)
    assert_close(out, v * F.gelu(g), what="geglu")


def test_gemm_geglu_large_gates():
    """The epilogue's erf-GELU is x * Phi(x) with Phi = 0.5 (1 + tanh(x P(x^2))), P fitted on [-8, 8]: outside the fit
    the polynomial must be range-guarded (Phi -> exactly 0 / 1), or outlier gate pre-activations of a real checkpoint
    zero a channel / let a large negative value through.  Gates swept over +-[0, 100] via the bias (zero gate weights)."""
    M, K, n_out = 256, 64, 320
    proj = torch.randn(2 * n_out, K, device=DEV) * K ** -0.5
    proj[n_out:] = 0.0
    pb = torch.zeros(2 * n_out, device=DEV)
    sweep = torch.cat([torch.linspace(-100.0, -8.0, n_out // 4), torch.linspace(-12.0, 12.0, n_out // 2),
                       torch.linspace(8.0, 100.0, n_out - n_out // 4 - n_out // 2)]).to(DEV)
    pb[n_out:] = sweep
    a = rnd(M, K)
    bn = ops.pick_block_n(2 * n_out, ops.ACT_GEGLU)
    perm = ops.geglu_perm(n_out, bn).to(DEV)
    wp, bp = bf(proj[perm]).contiguous(), pb[perm].contiguous()
    out = torch.empty(M, n_out, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, wp, out, K=K, N=2 * n_out, rows_per_batch=M, bias=bp, act=ops.ACT_GEGLU)
    y = a.float() @ bf(proj).float().t() + pb
    v, g = y.chunk(2, dim=-1)
    assert_close(out, v * F.gelu(g), what="geglu large gates")
    big = sweep > 12.0
    assert_close(out[:, big], v[:, big] * g[:, big], what="geglu gate >> 0 is the identity")
    assert out[:, sweep < -12.0].abs().max().item() == 0.0


def test_gemm_batched_b():
    """decoder AttnBlock shape: S_b = Q_b K_b^T, B operand batched."""
    Bn, M, K, N = 3, 256, 512, 256
    q, k = rnd(Bn, M, K, scale=0.2), rnd(Bn, N, K, scale=0.2)
    out = torch.empty(Bn, M, N, device=DEV, dtype=torch.bfloat16)
    ops.gemm(q, k, out, K=K, N=N, rows_per_batch=M, batch=Bn, a_batch_stride=M * K, b_batch_stride=N * K,
             s0=K ** -0.5)
    assert_close(out, torch.einsum("bmk,bnk->bmn", q.float(), k.float()) * K ** -0.5, what="batched")


def test_gemm_batch_tail_rows():
    """rows_per_batch not a multiple of 128: tiles must not bleed across batch items."""
    Bn, M, K, N = 4, 72, 64, 64
    a, w = rnd(Bn, M, K), rnd(N, K, scale=K ** -0.5)
    out = torch.full((Bn, M, N), 7.0, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, out, K=K, N=N, rows_per_batch=M, batch=Bn, a_batch_stride=M * K)
    assert_close(out, a.float() @ w.float().t(), what="batch tail")


# --------------------------------------------------------------------------------------------
# temporal (3,1,1) conv as a 3-tap shifted GEMM
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("b,T,HW,C,Co", [(2, 4, 64, 64, 64), (2, 18, 64, 128, 160), (1, 5, 16, 64, 32), (2, 18, 256, 320, 320)])
def test_temporal_conv(b, T, HW, C, Co):
    x = rnd(b, T, HW, C)
    w3 = torch.randn(Co, C, 3, 1, 1, device=DEV) * (3 * C) ** -0.5
    bias = torch.randn(Co, device=DEV)
    wp = bf(w3[:, :, :, 0, 0].permute(0, 2, 1).reshape(Co, 3 * C)).contiguous()  # [Co][tap][C]
    out = torch.empty(b * T * HW, Co, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, wp, out, K=C, N=Co, rows_per_batch=T * HW, batch=b, a_batch_stride=T * HW * C, bias=bias,
             ntaps=3, tap_shift=HW)
    xin = x.float().permute(0, 3, 1, 2).reshape(b, C, T, HW, 1)
    ref = F.conv3d(xin, bf(w3).float(), bias, padding=(1, 0, 0))
    ref = ref.reshape(b, Co, T, HW).permute(0, 2, 3, 1).reshape(b * T * HW, Co)
    assert_close(out, ref, what="temporal conv")


# --------------------------------------------------------------------------------------------
# implicit-GEMM 3x3 conv
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n,h,w,c,co", [
    (2, 64, 64, 64, 64), (3, 32, 32, 128, 160), (5, 8, 8, 64, 128), (4, 16, 16, 192, 64),
    (1, 128, 128, 64, 16), (9, 4, 4, 64, 64), (2, 256, 256, 64, 32), (36, 8, 8, 1280, 1280),
])
def test_conv3x3(n, h, w, c, co):
    x = rnd(n, h, w, c)
    wt = torch.randn(co, c, 3, 3, device=DEV) * (9 * c) ** -0.5
    bias = torch.randn(co, device=DEV)
    wp = bf(wt.permute(0, 2, 3, 1).reshape(co, 9 * c)).contiguous()  # [Co][ky][kx][C]
    out = torch.empty(n * h * w, co, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, wp, out, K=c, N=co, rows_per_batch=n * h * w, bias=bias, conv=(n, h, w))
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), bf(wt).float(), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, co)
    assert_close(out, ref, what=f"conv3x3 {n}x{h}x{w}x{c}->{co}")


@pytest.mark.parametrize("co", [320, 256])
def test_conv3x3_residual_many_tiles(co):
    """Implicit 3x3 conv + residual (the ResBlock's `conv(.) + skip`) over several tiles per CTA: 10 images of 64 x 64,
    64 x 2-pixel boxes -> 320 pixel tiles x 2 (or 1) channel tiles, i.e. 2-4 tiles per CTA."""
    n, h, w, c = 10, 64, 64, 64
    x = rnd(n, h, w, c)
    wt = torch.randn(co, c, 3, 3, device=DEV) * (9 * c) ** -0.5
    bias = torch.randn(co, device=DEV)
    wp = bf(wt.permute(0, 2, 3, 1).reshape(co, 9 * c)).contiguous()
    r1 = rnd(n * h * w, co)
    out = torch.empty(n * h * w, co, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, wp, out, K=c, N=co, rows_per_batch=n * h * w, bias=bias, conv=(n, h, w), r1=r1, s1=1.0)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), bf(wt).float(), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, co) + r1.float()
    assert_close(out, ref, what=f"conv3x3 + residual, {co} channels, many tiles")


def test_conv3x3_strided_input_and_residual():
    n, h, w, c, co, ld = 2, 32, 32, 64, 64, 192
    buf = rnd(n, h, w, ld)
    x = buf[..., 64:128]
    wt = torch.randn(co, c, 3, 3, device=DEV) * (9 * c) ** -0.5
    wp = bf(wt.permute(0, 2, 3, 1).reshape(co, 9 * c)).contiguous()
    r1 = rnd(n * h * w, co)
    out = torch.empty(n * h * w, co, device=DEV, dtype=torch.bfloat16)
    ops.gemm(x, wp, out, K=c, N=co, rows_per_batch=n * h * w, lda=ld, conv=(n, h, w), r1=r1, s1=1.0)
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), bf(wt).float(), None, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(n * h * w, co) + r1.float()
    assert_close(out, ref, what="conv3x3 strided + residual")


# --------------------------------------------------------------------------------------------
# normalisation
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("ns,rows,c,eps,silu", [(4, 4096, 320, 1e-5, True), (6, 256, 1280, 1e-6, False),
                                                (2, 64, 2560, 1e-5, True), (3, 1000, 64, 1e-5, True),
                                                (2, 18 * 64, 640, 1e-5, True)])
def test_groupnorm(ns, rows, c, eps, silu):
    x = bf(torch.randn(ns, rows, c, device=DEV) * 2.0 + 0.5)
    gamma, beta = torch.randn(c, device=DEV), torch.randn(c, device=DEV)
    stats = torch.empty(ns, 32, 2, device=DEV, dtype=torch.float64)
    y = torch.empty_like(x)
    ops.groupnorm_stats(x, stats, rows, ns, c)
    ops.groupnorm_apply(x, y, stats, gamma, beta, rows, ns, c, eps, silu)
    ref = F.group_norm(x.float().permute(0, 2, 1), 32, gamma, beta, eps).permute(0, 2, 1)
    if silu:
        ref = F.silu(ref)
    assert_close(y, ref, what="groupnorm")
    # the single-launch form (statistics -> grid barrier -> apply): same contract, and bit-reproducible
    ws = ops.groupnorm_workspace(DEV)
    y1, y2 = torch.empty_like(x), torch.empty_like(x)
    ops.groupnorm(x, y1, gamma, beta, rows, ns, c, eps, silu, ws)
    assert_close(y1, ref, what="groupnorm (one launch)")
    for _ in range(3):      # back-to-back launches share the barrier words: the sense reversal must hold
        ops.groupnorm(x, y2, gamma, beta, rows, ns, c, eps, silu, ws)
    assert torch.equal(y1, y2)


@pytest.mark.parametrize("ns,rows,c", [(36, 4096, 320), (2, 18 * 4096, 320), (36, 64, 1280), (18, 16384, 128),
                                       (36, 1024, 1920), (1, 18 * 1024, 640)])
def test_groupnorm_one_launch_model_shapes(ns, rows, c):
    """V3D_512 shapes (2-D per-frame and 3-D time_stack norms, skip-concat widths, a strided input view) through the
    single-launch kernel against the statistics + apply pair; the two must agree to the rounding of the output."""
    x = bf(torch.randn(ns * rows, c, device=DEV) * 1.5 + 0.25)
    gamma, beta = torch.randn(c, device=DEV), torch.randn(c, device=DEV)
    stats = torch.empty(ns, 32, 2, device=DEV, dtype=torch.float64)
    y0, y1 = torch.empty_like(x), torch.empty_like(x)
    ops.groupnorm_stats(x, stats, rows, ns, c)
    ops.groupnorm_apply(x, y0, stats, gamma, beta, rows, ns, c, 1e-5, True)
    ws = ops.groupnorm_workspace(DEV)
    ops.groupnorm(x, y1, gamma, beta, rows, ns, c, 1e-5, True, ws)
    assert_close(y1, y0, rtol=1.0 / 128, atol=1e-2, what="one-launch vs pair")
    # strided input (a column slice of a wider matrix), dense output
    wide = bf(torch.randn(ns * rows, c + 64, device=DEV))
    xs = wide[:, 64:]
    y2, y3 = torch.empty_like(x), torch.empty_like(x)
    ops.groupnorm(xs, y2, gamma, beta, rows, ns, c, 1e-5, False, ws, ldx=c + 64)
    ops.groupnorm(xs.contiguous(), y3, gamma, beta, rows, ns, c, 1e-5, False, ws)
    assert torch.equal(y2, y3)


@pytest.mark.parametrize("rows,c,rpf", [(4096, 320, 1024), (777, 1280, 7), (128, 64, 128), (300, 640, 100)])
def test_layernorm(rows, c, rpf):
    x = rnd(rows, c, scale=2.0)
    gamma, beta = torch.randn(c, device=DEV), torch.randn(c, device=DEV)
    y = torch.empty_like(x)
    ops.layernorm(x, y, gamma, beta, rows, c)
    assert_close(y, F.layer_norm(x.float(), (c,), gamma, beta, 1e-5), what="layernorm")
    add = torch.randn((rows + rpf - 1) // rpf, c, device=DEV)
    ysum = torch.empty_like(x)
    ops.layernorm(x, y, gamma, beta, rows, c, add=add, ysum=ysum, rows_per_frame=rpf)
    z = x.float() + add.repeat_interleave(rpf, 0)[:rows]
    assert_close(ysum, z, what="layernorm ysum")
    assert_close(y, F.layer_norm(ysum.float(), (c,), gamma, beta, 1e-5), what="layernorm(add)")


def test_softmax_rows():
    rows, n = 300, 4096
    x = rnd(rows, n, scale=3.0)
    ref = torch.softmax(x.float() * 0.5, dim=-1)
    ops.softmax_rows(x, rows, n, 0.5)
    assert_close(x, ref, atol=1e-4, what="softmax rows")


# --------------------------------------------------------------------------------------------
# attention
# --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("nb,ntok,heads", [(2, 16, 4), (3, 64, 20), (2, 256, 10), (2, 1024, 5), (1, 4096, 5),
                                           (2, 200, 2), (1, 1000, 3), (2, 300, 2), (1, 600, 1), (3, 2048, 2)])
# "tcgen05" names the product kernel (v3d_attention_spatial, now wgmma); the id is kept so the test's history stays one
@pytest.mark.parametrize("impl", ["tcgen05", "mma"])
def test_attention_spatial(nb, ntok, heads, impl):
    c = heads * 64
    qkv = rnd(nb * ntok, 3 * c)
    out = torch.empty(nb * ntok, c, device=DEV, dtype=torch.bfloat16)
    fn = ops.attention_spatial if impl == "tcgen05" else ops.attention_spatial_mma
    fn(qkv, out, nb, ntok, heads, 64 ** -0.5)
    q, k, v = [t.reshape(nb, ntok, heads, 64).permute(0, 2, 1, 3).float() for t in qkv.split(c, dim=-1)]
    ref = F.scaled_dot_product_attention(q, k, v).permute(0, 2, 1, 3).reshape(nb * ntok, c)
    assert_close(out, ref, atol=3e-2, what="spatial attention")


@pytest.mark.parametrize("nb,T,S,heads", [(2, 4, 16, 4), (2, 18, 64, 20), (2, 14, 100, 5), (1, 25, 33, 10), (2, 32, 8, 1)])
def test_attention_temporal(nb, T, S, heads):
    c = heads * 64
    qkv = rnd(nb * T * S, 3 * c)
    out = torch.empty(nb * T * S, c, device=DEV, dtype=torch.bfloat16)
    ops.attention_temporal(qkv, out, nb, T, S, heads, 64 ** -0.5)
    # rows are (b t s); reference attends over t for every (b, s, head)
    q, k, v = [t.reshape(nb, T, S, heads, 64).permute(0, 2, 3, 1, 4).float() for t in qkv.split(c, dim=-1)]
    ref = F.scaled_dot_product_attention(q, k, v)  # [nb, S, heads, T, 64]
    ref = ref.permute(0, 3, 1, 2, 4).reshape(nb * T * S, c)
    assert_close(out, ref, atol=3e-2, what="temporal attention")


# --------------------------------------------------------------------------------------------
# data movement / small matrices / sampler arithmetic
# --------------------------------------------------------------------------------------------
def test_upsample_copy_im2col():
    n, h, w, c = 3, 8, 16, 64
    x = rnd(n, h, w, c)
    y = torch.empty(n, 2 * h, 2 * w, c, device=DEV, dtype=torch.bfloat16)
    ops.upsample_nearest2x(x, y, n, h, w, c)
    ref = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest").permute(0, 2, 3, 1)
    assert torch.equal(y.float(), ref)

    dst = torch.zeros(n * h * w, 192, device=DEV, dtype=torch.bfloat16)
    ops.copy_channels(x, c, dst[:, 128:], 192, n * h * w, c)
    assert torch.equal(dst[:, 128:], x.reshape(-1, c)) and dst[:, :128].abs().max() == 0

    for (cc, stride, pad) in [(8, 1, 1), (64, 2, 1), (4, 1, 1), (16, 2, 0)]:
        xi = rnd(n, h, w, cc)
        ho = (h + 2 * pad - 3) // stride + 1 if pad else (h + 1 - 3) // stride + 1
        wo = (w + 2 * pad - 3) // stride + 1 if pad else (w + 1 - 3) // stride + 1
        kpad = ((9 * cc + 63) // 64) * 64
        col = torch.empty(n * ho * wo, kpad, device=DEV, dtype=torch.bfloat16)
        ops.im2col3x3(xi, col, n, h, w, cc, stride, pad, ho, wo, kpad)
        xp = xi.float().permute(0, 3, 1, 2)
        if pad == 0:  # asymmetric (0,1,0,1) pad of the VAE encoder downsample
            xp = F.pad(xp, (0, 1, 0, 1))
        unf = F.unfold(xp, 3, padding=pad, stride=stride)  # [n, cc*9, L] with (c, ky, kx) ordering
        unf = unf.reshape(n, cc, 9, ho * wo).permute(0, 3, 2, 1).reshape(n * ho * wo, 9 * cc)
        assert torch.equal(col[:, :9 * cc].float(), unf), (cc, stride, pad)
        if kpad > 9 * cc:
            assert col[:, 9 * cc:].abs().max() == 0


def test_layout_conversions():
    n, c, h, w = 5, 8, 16, 24
    x = torch.randn(n, c, h, w, device=DEV)
    y = torch.empty(n, h, w, c, device=DEV, dtype=torch.bfloat16)
    ops.nchw_f32_to_nhwc_bf16(x, y, 0.5)
    assert torch.equal(y, bf(x.permute(0, 2, 3, 1) * 0.5))
    src = torch.randn(n * h * w, 16, device=DEV)
    out = torch.empty(n, 4, h, w, device=DEV)
    ops.nhwc_to_nchw_f32(src, out, n, 4, h * w, 16, 2.0)
    assert torch.equal(out, (src[:, :4] * 2.0).reshape(n, h, w, 4).permute(0, 3, 1, 2))
    srcb = bf(src)
    ops.nhwc_to_nchw_f32(srcb, out, n, 4, h * w, 16)
    assert torch.equal(out, srcb[:, :4].float().reshape(n, h, w, 4).permute(0, 3, 1, 2))


@pytest.mark.parametrize("m,k,n", [(36, 320, 1280), (36, 1280, 320), (2, 1024, 640), (8, 768, 1280), (50, 64, 24)])
def test_small_linear(m, k, n):
    x = torch.randn(m, k, device=DEV)
    w = rnd(n, k, scale=k ** -0.5)
    b = torch.randn(n, device=DEV)
    y = torch.empty(m, n, device=DEV)
    ops.small_linear(x, w, b, y, act_in=ops.ACT_SILU)
    ref = F.silu(x) @ w.float().t() + b
    tol0 = dict(rtol=2e-2, atol=2e-2) if k % 64 == 0 else dict(rtol=1e-4, atol=1e-4)
    assert_close(y, ref, what="small_linear silu-in", **tol0)
    ops.small_linear(x, w, None, y, act_out=ops.ACT_SILU, accumulate=True)
    # paths differ in input rounding: K % 64 == 0 runs on tensor cores with bf16(act_in(x)), else fp32 SIMT
    tol = dict(rtol=2e-2, atol=2e-2) if k % 64 == 0 else dict(rtol=1e-4, atol=1e-4)
    assert_close(y, ref + F.silu(x @ w.float().t()), what="small_linear accumulate", **tol)


@pytest.mark.parametrize("m,k,n,ld", [(36, 1280, 38400, 0), (36, 1024, 640, 2048), (2, 320, 1280, 0), (64, 64, 200, 0), (70, 128, 256, 0)])
def test_small_linear_tensor_core_path(m, k, n, ld):
    """M<=64 linears as W x X^T with transposed fp32 store, strided x/y, accumulate, N not a multiple of 128."""
    xw = torch.randn(m, ld or k, device=DEV)
    x = xw[:, :k]
    w = rnd(n, k, scale=k ** -0.5)
    b = torch.randn(n, device=DEV)
    yw = torch.zeros(m, n + 64, device=DEV)
    y = yw[:, 32:32 + n]
    ops.small_linear(x, w, b, y, act_in=ops.ACT_SILU)
    ref = bf(F.silu(x)).float() @ w.float().t() + b
    assert_close(y, ref, rtol=1e-3, atol=2e-3, what="small-M tensor-core")
    assert yw[:, :32].abs().max() == 0 and yw[:, 32 + n:].abs().max() == 0
    ops.small_linear(x, w, None, y, accumulate=True)
    assert_close(y, ref + bf(x).float() @ w.float().t(), rtol=1e-3, atol=4e-3, what="small-M accumulate")


def test_timestep_embedding():
    t = torch.tensor([0.0, 1.0, 17.0, -1.55, 1.637], device=DEV)
    for dim in (320, 1280, 64):
        out = torch.empty(t.numel(), dim, device=DEV)
        ops.timestep_embedding(t, out, dim)
        half = dim // 2
        freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=DEV) / half)
        args = t[:, None] * freqs[None]
        ref = torch.cat([torch.cos(args), torch.sin(args)], -1)
        assert_close(out, ref, rtol=0, atol=2e-5, what="timestep embedding")


def test_sampler_arithmetic_and_u8():
    T, per = 6, 4 * 16 * 16
    x = torch.randn(2 * T, per, device=DEV)
    sigma = torch.rand(2 * T, device=DEV) * 700 + 0.002
    y = torch.empty_like(x)
    cn = torch.empty(2 * T, device=DEV)
    ops.edm_scale_input(x, sigma, y, cn, 2 * T, per)
    assert_close(y, x / (sigma[:, None] ** 2 + 1) ** 0.5, rtol=1e-6, atol=1e-7, what="c_in")
    assert_close(cn, 0.25 * sigma.log(), rtol=1e-6, atol=1e-6, what="c_noise")
    net = torch.randn_like(x)
    den = torch.empty_like(x)
    ops.edm_denoise_combine(net, x, sigma, den, 2 * T, per)
    s2 = sigma[:, None] ** 2 + 1
    assert_close(den, net * (-sigma[:, None] / s2 ** 0.5) + x / s2, rtol=1e-5, atol=1e-6, what="denoise combine")
    scale = torch.linspace(1.0, 3.5, T, device=DEV)
    g = torch.empty(T, per, device=DEV)
    ops.cfg_combine(den, scale, g, 1, T, per)
    xu, xc = den.chunk(2)
    assert_close(g, xu + scale[:, None] * (xc - xu), rtol=1e-6, atol=1e-6, what="cfg")
    sh, sn = sigma[:T].contiguous(), (sigma[:T] * 0.7).contiguous()
    xs = x[:T].contiguous()
    out = torch.empty_like(xs)
    ops.euler_step(xs, g, sh, sn, out, T, per)
    d = (xs - g) / sh[:, None]
    assert_close(out, xs + (sn - sh)[:, None] * d, rtol=1e-5, atol=1e-5, what="euler")

    img = torch.randn(100, 16, device=DEV) * 0.8
    u8 = torch.empty(100, 3, device=DEV, dtype=torch.uint8)
    ops.decode_to_u8(img, 16, u8, 100)
    ref = (torch.clamp((img[:, :3] + 1.0) / 2.0, 0.0, 1.0) * 255).to(torch.uint8)
    assert (u8.int() - ref.int()).abs().max() <= 1  # fp rounding of the *255 product may differ by one ulp


def test_heun_step_kernel():
    """v3d_heun_step vs the formula of HeunEDMSampler.possible_correction_step (sampling.py:221-237)."""
    n, per = 6, 4 * 16 * 16
    x, den, den2 = (torch.randn(n, per, device=DEV) for _ in range(3))
    sh = torch.rand(n, device=DEV) * 5 + 1.0
    sn = sh * 0.5
    sn[-2:] = 0.0  # samples whose next sigma is 0 keep the Euler proposal
    xe = torch.empty_like(x)
    ops.euler_step(x, den, sh, sn, xe, n, per)
    out = torch.empty_like(x)
    ops.heun_step(x, den, xe, den2, sh, sn, out, n, per)
    d = (x - den) / sh[:, None]
    dt = (sn - sh)[:, None]
    d2 = (xe - den2) / sn.clamp_min(1e-30)[:, None]
    ref = torch.where(sn[:, None] > 0, x + (d + d2) / 2 * dt, x + dt * d)
    assert torch.allclose(out, ref, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("poly", [1, 2, 3])
def test_attention_poly_exp2_subprocess(poly):
    """FMA-pipe exp2 for 2 / 4 / 6 of a tile's 8 key chunks (V3D_ATTN_POLY, read once per process): the spatial
    attention tests (random and peaked rows, vs fp32 SDPA and the mma.sync twin; tail and planted-score cases vs fp64)
    re-run in a child with the switch on.  The polynomial's max relative error is 8e-5 (1.5e-4 at 2^-126), far inside
    those tests' bf16 tolerances."""
    import subprocess
    import sys
    from pathlib import Path

    here = Path(__file__).resolve().parent
    env = dict(os.environ, V3D_ATTN_POLY=str(poly))
    res = subprocess.run([sys.executable, "-m", "pytest", str(here / "test_kernels_gpu.py"),
                          str(here / "test_zz_attention_rescale_gpu.py"), str(here / "test_kernel_edges_fp64_gpu.py"),
                          "-x", "-q", "-m", "gpu", "-k", "attention_spatial"], env=env, capture_output=True, text=True,
                         timeout=600)
    assert res.returncode == 0, res.stdout[-3000:] + res.stderr[-2000:]


def test_concat_timestep_embedder_device():
    """Native ConcatTimestepEmbedderND (SURVEY 8(f)-1) vs the reference's vector conditioning (golden, fp32)."""
    from pathlib import Path

    from v3d_b200 import conditioning

    gold = torch.load(Path(__file__).resolve().parent / "golden" / "conditioning.pt")
    cond = conditioning.GeneralConditioner(conditioning.V3D_512_EMB_MODELS).to(DEV)
    c, uc = conditioning.assemble_v3d_conditioning(cond, gold["clip_emb"].to(DEV), gold["latent"].to(DEV), 6.0, 127.0,
                                                   0.02, 18)
    assert torch.allclose(c["vector"].cpu(), gold["c"]["vector"], atol=2e-5)
    assert torch.equal(c["crossattn"].cpu(), gold["c"]["crossattn"]) and torch.equal(uc["concat"].cpu(), gold["uc"]["concat"])

