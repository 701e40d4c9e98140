"""Residuals staged by TMA give the same bytes as residuals read by the epilogue.

The bf16-output GEMM loads R1 (and R2 where the tile leaves room for a second buffer) into its shared-memory staging
buffer by TMA during the main loop, and reads them back at the address the output goes to.  A residual whose base or
row pitch is not 16-byte aligned cannot be addressed by TMA, so the epilogue reads it from global memory instead.  Each
case runs the same GEMM on the same values twice: once with contiguous residuals (staged), once with copies of pitch
N + 2 elements or a base 4 bytes off alignment (read by the epilogue).  Both outputs start out NaN-filled and must be
byte-equal, and close to an fp32 ATen reference.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def ops():
    from v3d_b200 import ops as _ops

    return _ops


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).to(torch.bfloat16)


def unaligned(t, how):
    """The same values as the [rows, n] tensor t, at a row pitch (n + 2) or a base (+4 bytes) TMA cannot address."""
    rows, n = t.shape
    if how == "pitch":
        buf = torch.empty(rows, n + 2, device=DEV, dtype=t.dtype)
        view = buf[:, :n]
    else:
        buf = torch.empty(rows * n + 8, device=DEV, dtype=t.dtype)
        view = buf[2:2 + rows * n].view(rows, n)
    view.copy_(t)
    return view, n + 2 if how == "pitch" else n


def nan_out(rows, n):
    return torch.full((rows, n), float("nan"), device=DEV, dtype=torch.bfloat16)


def run_pair(ops, a, w, rows, n, kw, *, r1, r2=None, how="pitch", in_place=False):
    """Staged launch (contiguous residuals, optionally in place) and __ldg launch; returns both outputs."""
    if in_place:
        staged = r1.clone()
        ops.gemm(a, w, staged, r1=staged, r2=r2, **kw)
    else:
        staged = nan_out(rows, n)
        ops.gemm(a, w, staged, r1=r1, r2=r2, **kw)
    u1, ld1 = unaligned(r1, how)
    extra = {}
    if r2 is not None:
        u2, ld2 = unaligned(r2, how)
        extra = dict(r2=u2, ldr2=ld2)
    loaded = nan_out(rows, n)
    ops.gemm(a, w, loaded, r1=u1, ldr1=ld1, **extra, **kw)
    torch.cuda.synchronize()
    return staged, loaded


def check(staged, loaded, ref, what):
    assert not torch.isnan(staged).any(), f"{what}: staged output has unwritten (NaN) elements"
    assert not torch.isnan(loaded).any(), f"{what}: __ldg output has unwritten (NaN) elements"
    diff = (staged.view(torch.int16) != loaded.view(torch.int16))
    assert not diff.any(), f"{what}: {int(diff.sum())} of {diff.numel()} elements differ between staged and __ldg"
    err = (staged.float() - ref).abs()
    bad = err > 3e-2 + ref.abs() / 128
    assert not bad.any(), f"{what}: {int(bad.sum())} out of tolerance, max err {err.max().item():.4g}"


@pytest.mark.parametrize("block_n", [128, 160, 256])
@pytest.mark.parametrize("residuals", ["r1", "r1r2", "r1_fbias"])
def test_linear_batch1_tail(ops, block_n, residuals):
    M, K, N, rpf = 128 * 5 + 37, 128, 1280, 100
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    r1, r2 = rnd(M, N), rnd(M, N)
    kw = dict(K=K, N=N, rows_per_batch=M, bias=bias, block_n=block_n, s0=0.5, s1=0.75)
    core = a.float() @ w.float().t() + bias
    ref = 0.5 * core + 0.75 * r1.float()
    extra = {}
    if residuals == "r1r2":
        kw["s2"] = 0.25
        extra["r2"] = r2
        ref = ref + 0.25 * r2.float()
    if residuals == "r1_fbias":
        fbias = torch.randn((M + rpf - 1) // rpf, N, device=DEV)
        kw.update(fbias=fbias, rows_per_frame=rpf)
        ref = ref + 0.5 * fbias.repeat_interleave(rpf, 0)[:M]
    for how in ("pitch", "base"):
        staged, loaded = run_pair(ops, a, w, M, N, kw, r1=r1, how=how, **extra)
        check(staged, loaded, ref, f"linear BN={block_n} {residuals} {how}")


@pytest.mark.parametrize("rows", [200, 128 * 3])
def test_batched_linear_blend(ops, rows):
    batch, K, N = 3, 256, 320
    a, w = rnd(batch * rows, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    r1, r2 = rnd(batch * rows, N), rnd(batch * rows, N)
    kw = dict(K=K, N=N, rows_per_batch=rows, batch=batch, a_batch_stride=rows * K, bias=bias, s0=0.5, s1=0.75,
              s2=1.5)
    ref = 0.5 * (a.float() @ w.float().t() + bias) + 0.75 * r1.float() + 1.5 * r2.float()
    staged, loaded = run_pair(ops, a, w, batch * rows, N, kw, r1=r1, r2=r2)
    check(staged, loaded, ref, f"batched rows={rows}")


@pytest.mark.parametrize("block_n", [128, 160])
def test_linear_in_place(ops, block_n):
    M, K, N = 128 * 7 + 5, 320, 640
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    r1 = rnd(M, N)
    kw = dict(K=K, N=N, rows_per_batch=M, bias=bias, block_n=block_n)
    ref = a.float() @ w.float().t() + bias + r1.float()
    staged, loaded = run_pair(ops, a, w, M, N, kw, r1=r1, in_place=True)
    check(staged, loaded, ref, f"in place BN={block_n}")


def temporal_ref(x, w, batch, rows, hw, C, pad_x=None):
    """Conv3d (3,1,1) pad (1,0,0) on frame-major [batch][T*hw][C]: three row-shifted GEMMs."""
    xs = x.float().view(batch, rows, C) if pad_x is None else pad_x
    out = torch.zeros(batch, rows, C, device=DEV)
    wf = w.float().view(C, 3, C)
    for t in range(3):
        sh = (t - 1) * hw
        src = torch.zeros_like(xs)
        if sh >= 0:
            src[:, : rows - sh] = xs[:, sh:] if sh else xs
        else:
            src[:, -sh:] = xs[:, : rows + sh]
        out += src @ wf[:, t].t()
    return out.reshape(batch * rows, C)


@pytest.mark.parametrize("halo", [False, True])
def test_temporal_three_tap(ops, halo):
    batch, T, hw, C = 2, 6, 40, 320  # 240 rows per batch item: a tail tile
    rows = T * hw
    w = rnd(C, 3 * C, scale=(3 * C) ** -0.5)
    bias = torch.randn(C, device=DEV)
    r1 = rnd(batch * rows, C)
    if not halo:
        x = rnd(batch * rows, C)
        kw = dict(K=C, N=C, rows_per_batch=rows, batch=batch, a_batch_stride=rows * C, ntaps=3, tap_shift=hw,
                  bias=bias, s0=0.5, s1=1.0)
        core = temporal_ref(x, w, batch, rows, hw, C)
    else:
        # a halo'd operand: one frame of neighbours on each side; output row r reads A row hw + r (+ tap shifts)
        x = rnd(batch * (rows + 2 * hw), C)
        kw = dict(K=C, N=C, rows_per_batch=rows, batch=batch, a_batch_stride=(rows + 2 * hw) * C, ntaps=3,
                  tap_shift=hw, bias=bias, s0=0.5, s1=1.0, a_rows=rows + 2 * hw, a_row0=hw)
        xs = x.float().view(batch, rows + 2 * hw, C)
        wf = w.float().view(C, 3, C)
        core = sum(xs[:, t * hw: t * hw + rows] @ wf[:, t].t() for t in range(3)).reshape(batch * rows, C)
    ref = 0.5 * (core + bias) + r1.float()
    staged, loaded = run_pair(ops, x, w, batch * rows, C, kw, r1=r1)
    check(staged, loaded, ref, f"temporal halo={halo}")


@pytest.mark.parametrize("residuals", ["r1", "r1r2", "r1_fbias"])
def test_conv3x3_tail_image(ops, residuals):
    """8x8 images tile two to a 128-pixel box: with 5 images the last box holds one image past the end."""
    n, h, w_, c, co = 5, 8, 8, 64, 160
    x = rnd(n, h, w_, c)
    wt = torch.randn(co, c, 3, 3, device=DEV) * (9 * c) ** -0.5
    wp = wt.permute(0, 2, 3, 1).reshape(co, 9 * c).to(torch.bfloat16).contiguous()
    bias = torch.randn(co, device=DEV)
    rows = n * h * w_
    r1, r2 = rnd(rows, co), rnd(rows, co)
    kw = dict(K=c, N=co, rows_per_batch=rows, bias=bias, conv=(n, h, w_), s0=0.5, s1=1.0)
    core = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.to(torch.bfloat16).float(), bias, padding=1)
    core = core.permute(0, 2, 3, 1).reshape(rows, co)
    extra = {}
    if residuals == "r1_fbias":
        fbias = torch.randn(n, co, device=DEV)
        kw.update(fbias=fbias, rows_per_frame=h * w_)
        core = core + fbias.repeat_interleave(h * w_, 0)
    ref = 0.5 * core + r1.float()
    if residuals == "r1r2":
        kw["s2"] = -0.5
        extra["r2"] = r2
        ref = ref - 0.5 * r2.float()
    staged, loaded = run_pair(ops, x, wp, rows, co, kw, r1=r1, **extra)
    check(staged, loaded, ref, f"conv {residuals}")


@pytest.mark.parametrize("block_n", [128, 256])
def test_conv3x3_wide_in_place(ops, block_n):
    """32x32 images (8 rows of pixels per box), 256 output channels, the output is the residual."""
    n, h, w_, c, co = 3, 32, 32, 64, 256
    x = rnd(n, h, w_, c)
    wt = torch.randn(co, c, 3, 3, device=DEV) * (9 * c) ** -0.5
    wp = wt.permute(0, 2, 3, 1).reshape(co, 9 * c).to(torch.bfloat16).contiguous()
    bias = torch.randn(co, device=DEV)
    rows = n * h * w_
    r1 = rnd(rows, co)
    kw = dict(K=c, N=co, rows_per_batch=rows, bias=bias, conv=(n, h, w_), block_n=block_n)
    core = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.to(torch.bfloat16).float(), bias, padding=1)
    ref = core.permute(0, 2, 3, 1).reshape(rows, co) + r1.float()
    staged, loaded = run_pair(ops, x, wp, rows, co, kw, r1=r1, in_place=True)
    check(staged, loaded, ref, f"conv in place BN={block_n}")
