"""GEMM epilogue on tail rows with every per-row operand.

The epilogue's column loop reads bias, per-frame bias and residuals through pointers formed once per row.  For rows
past the end of the output (the tail of the last tile of a batch item or of the image set), it reads row 0 instead,
and relies on the stores never writing those rows: the TMA store clips them to the output's extent, and the fp32
stores check the row.  These cases put tail rows in every mode together with per-frame bias and residuals, in place
too.  They check the valid rows against fp32 ATen and that nothing past the output's end was written.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

DEV = "cuda"
SENTINEL = 7.0


@pytest.fixture(scope="module")
def ops():
    from v3d_b200 import ops as _ops

    torch.manual_seed(0)
    return _ops


def rnd(*shape, scale=1.0):
    return (torch.randn(*shape, device=DEV) * scale).to(torch.bfloat16)


def check(got, ref, what):
    err = (got.float() - ref).abs()
    bad = err > 3e-2 + ref.abs() / 128
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} out of tolerance, max err {err.max().item():.4g}"


@pytest.mark.parametrize("rows", [72, 200, 128 + 1])
def test_batched_linear_tail_rows_with_frame_bias_and_two_residuals(ops, rows):
    """Batch items whose rows end inside a tile; the per-frame bias changes inside a tile (40 rows per frame)."""
    batch, K, N, rpf = 3, 128, 320, 40
    a = rnd(batch * rows, K)
    w = rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    frames = (batch * rows + rpf - 1) // rpf
    fbias = torch.randn(frames, N, device=DEV)
    r1, r2 = rnd(batch * rows, N), rnd(batch * rows, N)
    buf = torch.full((batch * rows + 64, N), SENTINEL, device=DEV, dtype=torch.bfloat16)
    ops.gemm(a, w, buf, K=K, N=N, rows_per_batch=rows, batch=batch, a_batch_stride=rows * K, bias=bias,
             fbias=fbias, rows_per_frame=rpf, r1=r1, r2=r2, s0=0.5, s1=0.75, s2=0.25)
    core = a.float() @ w.float().t() + bias + fbias.repeat_interleave(rpf, 0)[: batch * rows]
    check(buf[: batch * rows], 0.5 * core + 0.75 * r1.float() + 0.25 * r2.float(), "batched tails")
    assert (buf[batch * rows:] == SENTINEL).all(), "rows past the output were written"


def test_linear_tail_rows_in_place_residual_and_fp32(ops):
    """In place (the output is the residual) with a tail, and the fp32 epilogue with a tail and per-frame bias."""
    M, K, N, rpf = 128 * 9 + 77, 64, 256, 100
    a, w = rnd(M, K), rnd(N, K, scale=K ** -0.5)
    bias = torch.randn(N, device=DEV)
    fbias = torch.randn((M + rpf - 1) // rpf, N, device=DEV)
    core = a.float() @ w.float().t() + bias + fbias.repeat_interleave(rpf, 0)[:M]
    buf = torch.full((M + 64, N), SENTINEL, device=DEV, dtype=torch.bfloat16)
    buf[:M] = rnd(M, N)
    r1 = buf[:M].float()
    ops.gemm(a, w, buf, K=K, N=N, rows_per_batch=M, bias=bias, fbias=fbias, rows_per_frame=rpf, r1=buf, s0=0.5,
             s1=1.0)
    check(buf[:M], 0.5 * core + r1, "in place")
    assert (buf[M:] == SENTINEL).all(), "rows past the output were written"
    o32 = torch.full((M + 64, N), SENTINEL, device=DEV)
    res = rnd(M, N)
    ops.gemm(a, w, o32, K=K, N=N, rows_per_batch=M, bias=bias, fbias=fbias, rows_per_frame=rpf, r1=res, s1=0.5)
    check(o32[:M], core + 0.5 * res.float(), "fp32")
    assert (o32[M:] == SENTINEL).all(), "rows past the output were written (fp32)"


def test_conv3x3_tail_image_with_image_bias_and_in_place_residual(ops):
    """8x8 images tile two to a 128-pixel box: with 5 images the last box holds one image past the end."""
    n, h, w, c, co = 5, 8, 8, 64, 160
    x = rnd(n, h, w, c)
    wt = torch.randn(co, c, 3, 3, device=DEV) * (9 * c) ** -0.5
    wp = wt.permute(0, 2, 3, 1).reshape(co, 9 * c).to(torch.bfloat16).contiguous()
    bias = torch.randn(co, device=DEV)
    fbias = torch.randn(n, co, device=DEV)
    rows = n * h * w
    buf = torch.full((rows + 128, co), SENTINEL, device=DEV, dtype=torch.bfloat16)
    buf[:rows] = rnd(rows, co)
    r1 = buf[:rows].float()
    ops.gemm(x, wp, buf, K=c, N=co, rows_per_batch=rows, bias=bias, fbias=fbias, rows_per_frame=h * w, r1=buf,
             s0=0.5, s1=1.0, conv=(n, h, w))
    ref = torch.nn.functional.conv2d(x.float().permute(0, 3, 1, 2), wt.to(torch.bfloat16).float(), bias, padding=1)
    ref = ref.permute(0, 2, 3, 1).reshape(rows, co) + fbias.repeat_interleave(h * w, 0)
    check(buf[:rows], 0.5 * ref + r1, "conv tail image")
    assert (buf[rows:] == SENTINEL).all(), "pixels past the last image were written"
