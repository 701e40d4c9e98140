"""Every compiled kernel variant held to one bf16 rounding of an fp64 reference, with inputs planted at the tile, tail,
chunk and frame boundaries where kernels go wrong.

Oracle.  Each reference below restates the contract of include/v3d_b200.h in plain fp64 torch, on the same
bf16-rounded inputs the kernel gets (it shares no code with tests/emu_ops.py, so a stand-in and a kernel cannot share a
mistake).  Next to every reference element it computes `mag`: the fp64 sum of the absolute values of every term that
feeds that element.  Every output element must then satisfy

    |got - ref| <= step * |ref| + c_family * mag

where step = 2^-8 for bf16 outputs (one correctly rounded bf16 step) and 2^-24 for fp32 outputs.  c_family is derived
from how the kernel computes, one line of reasoning each (u = 2^-24, the fp32 unit roundoff):

  gemm      (K_total + 8) * 2u.  wgmma adds K_total products into an fp32 accumulator, each add off by at most 2u of the
            running |sum| <= mag (2u allows an accumulator that truncates); the epilogue adds <= 8 more fp32 operations
            (bias, per-frame bias, s0, two residual FMAs), each within u of a partial result bounded by mag.
  geglu     2^-12 + 3 * gemm.  Phi comes from 0.5 (1 + tanh.approx(x P(x^2))): tanh.approx is within 2^-11 relative, so
            Phi within 2^-12 absolute, and the fitted P adds <= 2.5e-5 absolute to x Phi(x); with mag = Mv (Mg + 1) (Mv,
            Mg: magnitudes of the value and gate pre-activations) that is <= 2^-12 mag.  Accumulation errors pass
            through |gelu| <= |g| and |gelu'| <= 1.13: <= 3 * gemm * mag.
  silu      2^-12 + 2 * gemm (or + 2 * norm).  silu_f = x (0.5 tanh.approx(x / 2) + 0.5): <= 2^-12 |x| <= 2^-12 mag;
            upstream errors pass through |silu'| <= 1.1.
  attn      2^-8 + 2^-12.  P is rounded to bf16 (unit roundoff 2^-8) for the P V product while the normaliser sums
            the fp32 P: <= 2^-8 of sum(p |v|) / sum(p) = mag.  With few keys these roundings do not average out (the
            temporal kernel at T = 2..8 reaches 1.2x a 2^-9 bound).  ex2.approx (2^-22), the V3D_ATTN_POLY polynomial
            (1.5e-4 < 2^-12), the fp32 scores (64 exact bf16 products) and the online rescales (<= 64 multiplies) stay
            inside 2^-12.
  norm      2^-14.  Every fp32 partial sum in the norm kernels is a chain of <= 512 adds (per-thread rows, in-CTA trees,
            warp shuffles) before it is folded in fp64, so the (sum, sumsq) statistics are within 2^-15 relative to
            their magnitudes and var = E[x^2] - mu^2 within 3 * 2^-15 E[x^2]; mag carries the terms that error feeds
            (gamma rstd (|x| + |mu| + |x - mu| E[x^2] rstd^2) + |beta|), and the factor 2 covers the <= 4 fp32
            operations of the apply.
  softmax   2^-16.  mag = p (1 + |arg| + |max|) with arg = scale x - max: __expf = ex2.approx(arg log2 e) is within
            2^-22 + |arg| 2^-23 relative, the fp32 product scale x within u |scale x|, and the row sum is <= 64 fp32
            adds per chain (2^-18).
  mix       2^-20.  time_mix_conv is <= 13 fp32 FMAs per output (3 C taps + bias, C <= 4), each within u of a partial
            sum bounded by mag: 13 u < 2^-20.
  move      0.  Data movement (the K|V scatter) is bit for bit.

Where the error model predicts it (GEMM without GEGLU or SiLU, norms without SiLU), at least 99 % of the bf16 outputs
must also equal bf16(ref64) bit for bit: that catches a sub-ulp systematic shift (a truncating store, a C - 1 divisor)
that the bound alone lets through.  Every output lives inside a larger buffer filled with a sentinel; nothing outside
the output may change.

Inputs.  GEMM A rows at the first / last row of every 128-row tile, the last row of every batch item and the halo rows
are 16x larger; bias, per-frame bias and residual columns at every N-tile edge hold distinct large values: a row or
column taken from a neighbour becomes an O(1) error.  Attention runs two planted patterns: every real score near -8
nats (a masked key that leaks in with score 0 then dominates), and one dominant key per query (margin >= 9 nats) at
positions 0 / 63 / 64 / 127 / 128 / ntok-1 with V rows that encode their key index.  GroupNorm plants 30-sigma outlier
rows at rows 0, rows-1 and 2^k +- 1, a constant group, a group with variance ~ eps and groups with |mu| / sigma = 8 and
64 (how far the one-pass fp32 (sum x, sum x^2) holds).

Every case runs over `impl`: the kernel on CUDA (marked gpu), and, where one exists, the CPU stand-in of
tests/emu_ops.py on a reduced shape list (unmarked), which runs the builders, the oracle and
the index decoding without a GPU and pins the stand-ins at the same edges.

Each check prints one `EDGE <family> <case> ratio=<max |err| / bound> exact=<rate>` line (visible with -s or -rA).
"""
import math
import sys
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent))

import emu_ops  # noqa: E402
from v3d_b200 import ops  # noqa: E402

U = 2.0 ** -24
BF = torch.bfloat16
F64 = torch.float64
SENTINEL = -1232.0  # exact in bf16 and fp32


def c_gemm(ktot):
    return (ktot + 8) * 2 * U


def c_geglu(ktot):
    return 2.0 ** -12 + 3 * c_gemm(ktot)


def c_silu(upstream):
    return 2.0 ** -12 + 2 * upstream


C_ATTN = 2.0 ** -8 + 2.0 ** -12
C_NORM = 2.0 ** -14
C_SOFTMAX = 2.0 ** -16
C_MIX = 2.0 ** -20

GPU = pytest.mark.gpu


def _dev(impl):
    return "cpu" if impl == "standin" else "cuda"


def _sync(impl):
    if impl != "standin":
        torch.cuda.synchronize()


def _gen(seed):
    g = torch.Generator()
    g.manual_seed(seed)
    return g


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, dtype=F64)


def _bf(x, dev):
    """bf16-round on the host and move: the kernel and the fp64 reference see the same values."""
    return x.to(BF).to(dev)


def _unravel(flat, shape):
    idx = []
    for s in reversed(shape):
        idx.append(flat % s)
        flat //= s
    return tuple(reversed(idx))


def check(what, fam, got, ref, mag, c, *, f32=False, exact=False, where=None):
    """|got - ref| <= step |ref| + c mag for every element; with exact=True also >= 99 % equal to bf16(ref)."""
    got64 = got.detach().to("cpu", F64)
    ref = ref.to("cpu", F64)
    mag = mag.to("cpu", F64)
    step = U if f32 else 2.0 ** -8
    err = (got64 - ref).abs()
    bound = step * ref.abs() + c * mag
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    ratio = torch.where(torch.isfinite(got64), ratio, torch.full_like(err, math.inf))
    worst = int(ratio.reshape(-1).argmax())
    wr = float(ratio.reshape(-1)[worst])
    rate = float("nan")
    if not f32:
        rate = float((got.detach().to("cpu") == ref.to(BF)).double().mean())
    print(f"EDGE {fam} {what} ratio={wr:.3g} exact={rate:.5f}")
    if not wr <= 1.0:
        ix = _unravel(worst, tuple(ref.shape))
        loc = where(ix) if where else str(ix)
        nbad = int((ratio > 1).sum())
        raise AssertionError(
            f"{what}: {nbad}/{ratio.numel()} elements exceed |err| <= {step:.3g}|ref| + {c:.3g} mag; worst at {loc}: "
            f"got {float(got64[ix]):.7g} ref {float(ref[ix]):.7g} mag {float(mag[ix]):.4g} bound "
            f"{float(bound[ix]):.4g} (ratio {wr:.3g})")
    if exact:
        assert rate >= 0.99, f"{what}: only {rate:.4%} of the outputs equal bf16(ref64) (expected >= 99 %)"
    return wr


class Guarded:
    """rows x cols output (row stride ld) inside a sentinel-filled buffer with `pad` elements before and after."""

    def __init__(self, rows, cols, dtype, dev, ld=None, pad=64):
        self.rows, self.cols, self.ld, self.pad = rows, cols, ld or cols, pad
        self.buf = torch.full((2 * pad + rows * self.ld,), SENTINEL, dtype=dtype, device=dev)
        self.view = self.buf[pad:pad + rows * self.ld].view(rows, self.ld)[:, :cols]

    def assert_margins(self, what):
        probe = self.buf.clone()
        probe[self.pad:self.pad + self.rows * self.ld].view(self.rows, self.ld)[:, :self.cols] = SENTINEL
        bad = probe != SENTINEL
        if bad.any():
            i = int(bad.nonzero()[0])
            o = i - self.pad
            raise AssertionError(f"{what}: {int(bad.sum())} elements written outside the output; first at buffer "
                                 f"offset {o} (row {o // self.ld}, column {o % self.ld}; output is {self.rows} x "
                                 f"{self.cols}, ld {self.ld})")


# ------------------------------------------------------------------------------------------------------------------
# GEMM: all 45 (mode, BN, epilogue) instantiations of gemm_tc_kernel, forced through block_n
# ------------------------------------------------------------------------------------------------------------------
BNS = (16, 32, 64, 128, 160, 256)
GEMM_VARIANTS = ([("linear", bn, e) for bn in BNS for e in ("bf16", "bf16r2", "f32")] +
                 [("linear", bn, "geglu") for bn in (32, 64, 128, 160, 256)] +
                 [("linear", bn, "trans") for bn in (16, 32, 64, 128)] +
                 [("conv", bn, e) for bn in BNS for e in ("bf16", "bf16r2", "f32")])
assert len(GEMM_VARIANTS) == 45


def _impl_params(cases, standin_ok, ids):
    """kernel leg for every case (gpu), stand-in leg where standin_ok(case)"""
    out = []
    for case, cid in zip(cases, ids):
        out.append(pytest.param(*case, "kernel", marks=GPU, id=f"{cid}-kernel"))
        if standin_ok(case):
            out.append(pytest.param(*case, "standin", id=f"{cid}-standin"))
    return out


def _edge_cols(n, tile):
    return [c for c in range(n) if c % tile in (0, tile - 1)]


def _plant_cols(t, tile):
    """columns at every N-tile edge get distinct integer values (exact in bf16 and fp32)"""
    cols = _edge_cols(t.shape[-1], tile)
    for c in cols:
        t[..., c] = float((c * 7) % 61 - 30)
    return t


def _plant_rows(a, rows_per_item, row0=0):
    """a: [batch, a_rows, K]; the rows read by output rows at the first / last row of every 128-row tile and the last
    row of every item, and the halo rows outside [row0, row0 + rows_per_item), x16"""
    arows = a.shape[1]
    for r in range(arows):
        o = r - row0
        if o < 0 or o >= rows_per_item or o % 128 in (0, 127) or o == rows_per_item - 1:
            a[:, r] *= 16.0
    return a


def _linear_ref(A, B, rpb, taps, shift, row0):
    """A [batch, a_rows, K], B [batch or 1, N, taps K] -> (acc, mag) [batch, rpb, N]; out row r, tap t reads A row
    row0 + r + (t - taps // 2) shift, zero outside [0, a_rows)"""
    batch, arows, K = A.shape
    N = B.shape[1]
    acc = torch.zeros(batch, rpb, N, dtype=F64)
    mag = torch.zeros(batch, rpb, N, dtype=F64)
    for t in range(taps):
        src = row0 + torch.arange(rpb) + (t - taps // 2) * shift
        ok = (src >= 0) & (src < arows)
        At = torch.zeros(batch, rpb, K, dtype=F64)
        At[:, ok] = A[:, src[ok]]
        Bt = B[:, :, t * K:(t + 1) * K].transpose(1, 2)
        acc += At @ Bt
        mag += At.abs() @ Bt.abs()
    return acc, mag


def _conv_ref(X, Wt):
    """X [n, h, w, K], Wt [N, 9 K] (ky, kx, c) -> (acc, mag) [n h w, N]: 3x3, stride 1, zero padding 1"""
    n, h, w, K = X.shape
    N = Wt.shape[0]
    x = X.permute(0, 3, 1, 2)
    wt = Wt.reshape(N, 3, 3, K).permute(0, 3, 1, 2)
    acc = F.conv2d(x, wt, padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    mag = F.conv2d(x.abs(), wt.abs(), padding=1).permute(0, 2, 3, 1).reshape(-1, N)
    return acc, mag


def _epilogue_ref(acc, mag, *, bias=None, fbias=None, rpf=1, silu=False, s0=1.0, r1=None, s1=1.0, r2=None, s2=1.0):
    rows = acc.shape[0]
    if bias is not None:
        acc, mag = acc + bias, mag + bias.abs()
    if fbias is not None:
        fb = fbias[torch.arange(rows) // rpf]
        acc, mag = acc + fb, mag + fb.abs()
    if silu:
        acc = acc * torch.sigmoid(acc)                  # |silu(x)| <= |x| <= mag
    out, omag = s0 * acc, abs(s0) * mag
    for r, s in ((r1, s1), (r2, s2)):
        if r is not None:
            out, omag = out + s * r, omag + abs(s) * r.abs()
    return out, omag


def _gemm_where(rows_per_batch, out_tile):
    def where(ix):
        r, c = int(ix[0]), int(ix[1])
        b, rr = divmod(r, rows_per_batch)
        return f"(batch {b}, row {rr}, tile ({rr // 128}, {c // out_tile}), column {c})"
    return where


def _run_gemm(impl, *args, **kw):
    (ops.gemm if impl == "kernel" else emu_ops.gemm)(*args, **kw)
    _sync(impl)


@pytest.mark.parametrize("mode,bn,epi,impl", _impl_params(GEMM_VARIANTS, lambda c: c[2] != "trans",
                                                        [f"{m}-bn{b}-{e}" for m, b, e in GEMM_VARIANTS]))
def test_gemm_variant(mode, bn, epi, impl):
    """One launch per compiled (mode, BN, epilogue): a row tail, two N-tiles, every per-row operand the epilogue
    accepts (GEGLU: bias; TRANS: per-row bias, valid_cols < N, accumulate)."""
    dev = _dev(impl)
    g = _gen(1000 + bn + 7 * len(epi) + (500 if mode == "conv" else 0))
    K = 64 if mode == "conv" else 128
    what = f"gemm {mode} bn={bn} {epi}"
    if epi == "trans":
        # small-M mode: A = W [n_w, K] (row tail), B = X [N, K]; D fp32 [valid_cols][ldd], D[col][row] += acc + bias[row]
        n_w = 200
        N = 2 * bn if bn <= 64 else 256
        vc, ldd = N - 5, n_w + 24
        A = _plant_rows(_randn(g, 1, n_w, K), n_w)[0].to(BF).double()
        B = (_randn(g, N, K) * K ** -0.5).to(BF).double()
        bias = _randn(g, n_w).float().double()
        prior = _randn(g, vc, n_w).float().double()
        out = Guarded(vc, n_w, torch.float32, dev, ld=ldd, pad=(N - vc + 1) * ldd)
        out.view.copy_(prior)
        ops.gemm(A.to(BF).to(dev), B.to(BF).to(dev), out.view, K=K, N=N, rows_per_batch=n_w, ldd=ldd,
                 bias=bias.float().to(dev), transposed=True, valid_cols=vc, accumulate=True, block_n=bn)
        _sync(impl)
        acc = A @ B.t() + bias[:, None]
        mag = A.abs() @ B.abs().t() + bias.abs()[:, None]
        ref, rmag = (prior + acc.t()[:vc]), (prior.abs() + mag.t()[:vc])
        check(what, "gemm", out.view, ref, rmag, c_gemm(K), f32=True,
              where=lambda ix: f"(column {int(ix[0])}, row {int(ix[1])}, tile ({int(ix[1]) // 128}, "
                               f"{int(ix[0]) // bn}))")
        out.assert_margins(what)
        return

    if epi == "geglu":
        n_out = bn                                   # N = 2 bn: two N-tiles, bn / 2 output columns each
        N = 2 * n_out
        out_tile = bn // 2
    else:
        N = 2 * bn
        n_out = N
        out_tile = bn
    if mode == "conv":
        cn, ch, cw = 3, 4, 16                        # 64-pixel images, two per 128-pixel tile: the last tile is half
        rows = cn * ch * cw                          # empty (a tail image)
        rpb, batch = rows, 1
        X = _randn(g, cn, ch, cw, K)
        for y in range(ch):
            for x in range(cw):
                if y in (0, ch - 1) or x in (0, cw - 1) or (y * cw + x) % 128 in (0, 127):
                    X[:, y, x] *= 16.0
        X = X.to(BF).double()
        Wt = (_randn(g, N, 9 * K) * (9 * K) ** -0.5).to(BF).double()
        acc, mag = _conv_ref(X, Wt)
        a_dev, w_dev = _bf(X, dev), _bf(Wt, dev)
        gkw = dict(K=K, N=N, rows_per_batch=rows, conv=(cn, ch, cw))
    else:
        batch, rpb = 2, 200                          # 128 + 72: a row tail in both batch items
        rows = batch * rpb
        A = _plant_rows(_randn(g, batch, rpb, K), rpb).to(BF).double()
        Bm = (_randn(g, N, K) * K ** -0.5).to(BF).double()
        acc, mag = _linear_ref(A, Bm[None], rpb, 1, 0, 0)
        acc, mag = acc.reshape(rows, N), mag.reshape(rows, N)
        a_dev, w_dev = _bf(A, dev), _bf(Bm, dev)
        gkw = dict(K=K, N=N, rows_per_batch=rpb, batch=batch, a_batch_stride=rpb * K)

    if epi == "geglu":
        # proj rows: value rows [0, n_out), gate rows [n_out, 2 n_out); the kernel takes them packed per N-tile
        proj = (_randn(g, N, K) * K ** -0.5).to(BF).double()
        pb = _plant_cols(_randn(g, N).float().double(), n_out)
        perm = ops.geglu_perm(n_out, bn)
        y = A.reshape(rows, K) @ proj.t() + pb
        ym = A.reshape(rows, K).abs() @ proj.abs().t() + pb.abs()
        v, gt = y[:, :n_out], y[:, n_out:]
        mv, mg = ym[:, :n_out], ym[:, n_out:]
        ref = v * 0.5 * gt * (1.0 + torch.erf(gt / math.sqrt(2.0)))
        rmag = mv * (mg + 1.0)
        out = Guarded(rows, n_out, BF, dev, ld=n_out + 24)
        _run_gemm(impl, a_dev, _bf(proj[perm], dev), out.view, **gkw, ldd=n_out + 24,
                  bias=pb[perm].float().to(dev), act=ops.ACT_GEGLU, block_n=bn)
        check(what, "geglu", out.view, ref, rmag, c_geglu(K), where=_gemm_where(rpb, out_tile))
        out.assert_margins(what)
        return

    rpf = 50 if mode == "linear" else 40             # per-frame bias changes inside a tile
    frames = (rows + rpf - 1) // rpf
    bias = _plant_cols(_randn(g, N).float().double(), bn)
    fbias = _plant_cols(_randn(g, frames, N).float().double(), bn)
    r1 = _plant_cols(_randn(g, rows, n_out), bn).to(BF).double()
    r2 = _plant_cols(_randn(g, rows, n_out + 8), bn).to(BF).double() if epi != "bf16" else None
    s0, s1, s2 = 0.75, 0.5, 1.25
    ref, rmag = _epilogue_ref(acc, mag, bias=bias, fbias=fbias, rpf=rpf, s0=s0, r1=r1, s1=s1,
                              r2=None if r2 is None else r2[:, :n_out], s2=s2)
    f32 = epi == "f32"
    out = Guarded(rows, n_out, torch.float32 if f32 else BF, dev, ld=n_out + 24)
    kw = dict(gkw, ldd=n_out + 24, bias=bias.float().to(dev), fbias=fbias.float().to(dev), rows_per_frame=rpf,
              r1=_bf(r1, dev), s0=s0, s1=s1, block_n=bn)
    if r2 is not None:
        kw.update(r2=_bf(r2, dev), ldr2=n_out + 8, s2=s2)
    ktot = K * (9 if mode == "conv" else 1)
    _run_gemm(impl, a_dev, w_dev, out.view, **kw)
    check(what, "gemm", out.view, ref, rmag, c_gemm(ktot), f32=f32, exact=not f32, where=_gemm_where(rpb, out_tile))
    out.assert_margins(what)


def test_gemm_variant_ids_cover_every_instantiation():
    """The dispatcher's validity rules (gemm_tc.cu dispatch_epi): GEGLU needs (BN / 2) % 16 == 0 and linear mode,
    TRANS needs BN <= 128 and linear mode; BF16 / BF16R2 / F32 exist for every BN in both modes."""
    want = set()
    for conv in (False, True):
        for bn in BNS:
            for e in ("bf16", "bf16r2", "f32"):
                want.add(("conv" if conv else "linear", bn, e))
            if not conv and (bn // 2) % 16 == 0:
                want.add(("linear", bn, "geglu"))
            if not conv and bn <= 128:
                want.add(("linear", bn, "trans"))
    assert want == set(GEMM_VARIANTS)


OPERAND_MODES = ["batched_b", "temporal", "halo_first", "halo_last"]


@pytest.mark.parametrize("mode,impl", _impl_params([(m,) for m in OPERAND_MODES], lambda c: True, OPERAND_MODES))
def test_gemm_operand_modes(mode, impl):
    """Batched B (per-item weights), the 3-tap temporal shift, and a halo'd A operand with batch > 1 whose a_row0 sits
    at either end of the halo (a frame-sharded temporal conv at the first or the last rank)."""
    dev = _dev(impl)
    g = _gen({"batched_b": 11, "temporal": 12, "halo_first": 13, "halo_last": 14}[mode])
    K, N = 128, 96
    batch = 3 if mode == "batched_b" else 2
    taps, shift, row0 = 1, 0, 0
    if mode == "batched_b":
        rpb = 200
        arows = rpb
    else:
        taps, shift = 3, 24                          # 5 frames of 24 pixels: rows_per_batch 120 (a tail)
        rpb = 5 * shift
        arows = rpb if mode == "temporal" else rpb + 2 * shift
        row0 = {"temporal": 0, "halo_first": 0, "halo_last": arows - rpb}[mode]
    A = _plant_rows(_randn(g, batch, arows, K), rpb, row0).to(BF).double()
    nbb = batch if mode == "batched_b" else 1
    B = (_randn(g, nbb, N, taps * K) * (taps * K) ** -0.5).to(BF).double()
    bias = _plant_cols(_randn(g, N).float().double(), 32)
    r1 = _randn(g, batch * rpb, N).to(BF).double()
    acc, mag = _linear_ref(A, B, rpb, taps, shift, row0)
    ref, rmag = _epilogue_ref(acc.reshape(-1, N), mag.reshape(-1, N), bias=bias, r1=r1)
    out = Guarded(batch * rpb, N, BF, dev, ld=N + 8)
    kw = dict(K=K, N=N, rows_per_batch=rpb, batch=batch, a_batch_stride=arows * K, ldd=N + 8,
              bias=bias.float().to(dev), r1=_bf(r1, dev), ntaps=taps, tap_shift=shift, block_n=32)
    if mode == "batched_b":
        kw["b_batch_stride"] = N * K
    if mode.startswith("halo"):
        kw.update(a_rows=arows, a_row0=row0)
    _run_gemm(impl, _bf(A, dev), _bf(B, dev), out.view, **kw)
    check(f"gemm {mode}", "gemm", out.view, ref, rmag, c_gemm(taps * K), exact=True, where=_gemm_where(rpb, 32))
    out.assert_margins(f"gemm {mode}")


@pytest.mark.gpu
@pytest.mark.parametrize("bn", [32, 64, 128, 160, 256])
def test_gemm_kv_scatter(bn):
    """The fused K|V all-gather: output columns >= kv_col0 (a multiple of 32 inside the first N-tile) are stored again
    into two destination matrices, with one residual; the destinations equal the output bit for bit and nothing
    around them is written."""
    dev = "cuda"
    g = _gen(40 + bn)
    K, rows = 128, 328                               # 2 x 128 + 72 rows
    N = 2 * bn
    col0 = max(32, bn // 2 // 32 * 32)
    A = _plant_rows(_randn(g, 1, rows, K), rows).to(BF).double()
    Bm = (_randn(g, N, K) * K ** -0.5).to(BF).double()
    bias = _plant_cols(_randn(g, N).float().double(), bn)
    r1 = _plant_cols(_randn(g, rows, N), bn).to(BF).double()
    acc, mag = _linear_ref(A, Bm[None], rows, 1, 0, 0)
    ref, rmag = _epilogue_ref(acc[0], mag[0], bias=bias, r1=r1, s1=0.5)
    out = Guarded(rows, N, BF, dev, ld=N + 8)
    kv_ld = N - col0 + 8
    dsts = [Guarded(rows, N - col0, BF, dev, ld=kv_ld) for _ in range(2)]
    ops.gemm(_bf(A, dev), _bf(Bm, dev), out.view, K=K, N=N, rows_per_batch=rows, ldd=N + 8,
             bias=bias.float().to(dev), r1=_bf(r1, dev), s1=0.5, block_n=bn,
             kv=(col0, [d.view.data_ptr() for d in dsts], kv_ld))
    torch.cuda.synchronize()
    what = f"gemm kv scatter bn={bn}"
    check(what, "gemm", out.view, ref, rmag, c_gemm(K), exact=True, where=_gemm_where(rows, bn))
    out.assert_margins(what)
    for i, d in enumerate(dsts):
        same = d.view == out.view[:, col0:]
        assert same.all(), f"{what}: destination {i} differs from the output at {same.logical_not().nonzero()[0].tolist()}"
        print(f"EDGE move {what} dst{i} ratio=0 exact=1.00000")
        d.assert_margins(f"{what} destination {i}")


CONV_GRIDS = [(2, 72, 128), (1, 48, 64), (5, 2, 32)]


@pytest.mark.parametrize("n,h,w,impl", _impl_params(CONV_GRIDS, lambda c: True, [f"{n}x{h}x{w}" for n, h, w in CONV_GRIDS]))
def test_conv3x3_tile_grids(n, h, w, impl):
    """Non-power-of-two tile grids (72 rows of 128 pixels, 24 boxes of 64 x 2; the `%` / `/` branch of tile_origin)
    and a tail image (five 64-pixel images, two per tile), at the auto-picked N tile, with a residual."""
    dev = _dev(impl)
    g = _gen(60 + h)
    K, N = 64, 320
    X = _randn(g, n, h, w, K)
    X[:, 0] *= 16.0
    X[:, -1] *= 16.0
    X[:, :, 0] *= 16.0
    X[:, :, -1] *= 16.0
    X = X.to(BF).double()
    Wt = (_randn(g, N, 9 * K) * (9 * K) ** -0.5).to(BF).double()
    bias = _randn(g, N).float().double()
    rows = n * h * w
    r1 = _randn(g, rows, N).to(BF).double()
    acc, mag = _conv_ref(X, Wt)
    ref, rmag = _epilogue_ref(acc, mag, bias=bias, r1=r1)
    out = Guarded(rows, N, BF, dev)
    _run_gemm(impl, _bf(X, dev), _bf(Wt, dev), out.view, K=K, N=N, rows_per_batch=rows, conv=(n, h, w),
              bias=bias.float().to(dev), r1=_bf(r1, dev))
    hw = h * w

    def where(ix):
        r, c = int(ix[0]), int(ix[1])
        return f"(image {r // hw}, y {r % hw // w}, x {r % w}, column {c})"

    check(f"conv3x3 {n}x{h}x{w}", "gemm", out.view, ref, rmag, c_gemm(9 * K), exact=True, where=where)
    out.assert_margins(f"conv3x3 {n}x{h}x{w}")


@pytest.mark.parametrize("impl", [pytest.param("kernel", marks=GPU), "standin"])
def test_gemm_f32_silu(impl):
    """fp32 output with the fused SiLU, row tail and two N-tiles."""
    dev = _dev(impl)
    g = _gen(77)
    K, rows, N = 192, 200, 320
    A = _plant_rows(_randn(g, 1, rows, K), rows).to(BF).double()
    Bm = (_randn(g, N, K) * K ** -0.5).to(BF).double()
    bias = _plant_cols(_randn(g, N).float().double(), 160)
    acc, mag = _linear_ref(A, Bm[None], rows, 1, 0, 0)
    ref, rmag = _epilogue_ref(acc[0], mag[0], bias=bias, silu=True)
    out = Guarded(rows, N, torch.float32, dev)
    _run_gemm(impl, _bf(A, dev), _bf(Bm, dev), out.view, K=K, N=N, rows_per_batch=rows, bias=bias.float().to(dev),
              act=ops.ACT_SILU, block_n=160)
    check("gemm f32 silu", "silu", out.view, ref, rmag, c_silu(c_gemm(K)), f32=True, where=_gemm_where(rows, 160))
    out.assert_margins("gemm f32 silu")


# ------------------------------------------------------------------------------------------------------------------
# attention
# ------------------------------------------------------------------------------------------------------------------
SCALE = 0.125


def _attn_inputs(g, nseq, heads, L, pattern):
    """q, k, v [nseq, heads, L, 64] fp64 holding bf16 values.
    neg: every real score ~ -8 nats (q ~ +1, k ~ -1 in every dimension).
    dom: query i has one dominant key (score 10 nats, the rest within ~1) at positions[i % n]; v[j, :12] = bits of j."""
    if pattern == "neg":
        q = 1.0 + 0.25 * _randn(g, nseq, heads, L, 64)
        k = -(1.0 + 0.25 * _randn(g, nseq, heads, L, 64))
        v = _randn(g, nseq, heads, L, 64)
    else:
        q = 0.5 * _randn(g, nseq, heads, L, 64)
        k = 0.5 * _randn(g, nseq, heads, L, 64)
        q[..., 52:], k[..., 52:] = 0.0, 0.0
        pos = sorted({p for p in (0, 7, 8, 15, 16, 31, 63, 64, 127, 128, L - 1) if p < L})
        for m, p in enumerate(pos):                              # <= 11 positions: one coordinate each
            k[:, :, p, 52 + m] = 1.0
        i = torch.arange(L)
        q[:, :, i, 52 + i % len(pos)] = 10.0 / SCALE
        v = 0.5 * _randn(g, nseq, heads, L, 64)
        bits = torch.arange(L)[:, None].bitwise_right_shift(torch.arange(12)[None]).bitwise_and(1)
        v[..., :12] = (2.0 * bits - 1.0).to(F64)
    return q.to(BF).double(), k.to(BF).double(), v.to(BF).double()


def _attn_ref(q, k, v, dev):
    """softmax(q k^T scale) v and mag = sum p |v| / sum p, fp64 on `dev`, chunked over the leading dims"""
    o = torch.empty_like(q)
    m = torch.empty_like(q)
    for i in range(q.shape[0]):
        qi, ki, vi = q[i].to(dev), k[i].to(dev), v[i].to(dev)
        p = torch.softmax((qi @ ki.transpose(-1, -2)) * SCALE, dim=-1)
        o[i] = (p @ vi).cpu()
        m[i] = (p @ vi.abs()).cpu()
    return o, m


SPATIAL_NTOK = [1, 2, 63, 64, 65, 127, 128, 129, 257, 511, 512, 513, 4095, 4096]
SPATIAL_HEADS = [1, 5, 20]


def _spatial_params():
    out = []
    for ntok in SPATIAL_NTOK:
        for heads in SPATIAL_HEADS:
            for impl in ("tc", "mma"):
                out.append(pytest.param(ntok, heads, impl, marks=GPU, id=f"ntok{ntok}-h{heads}-{impl}"))
            if ntok in (1, 2, 63, 64, 65, 129) and heads in (1, 5):
                out.append(pytest.param(ntok, heads, "standin", id=f"ntok{ntok}-h{heads}-standin"))
    return out


@pytest.mark.parametrize("ntok,heads,impl", _spatial_params())
def test_attention_spatial_edges(ntok, heads, impl):
    """v3d_attention_spatial (wgmma, "tc") and its mma.sync twin (BM 64 below 512 tokens, 128 from 512) over two
    batch items: a tail must mask its own missing keys and never read the next item's."""
    dev = _dev(impl)
    nb, C = 2, heads * 64
    fn = {"tc": ops.attention_spatial, "mma": ops.attention_spatial_mma, "standin": emu_ops.attention_spatial}[impl]
    for pattern in ("neg", "dom"):
        g = _gen(ntok * 31 + heads + (7 if pattern == "dom" else 0))
        q, k, v = _attn_inputs(g, nb, heads, ntok, pattern)
        ref, mag = _attn_ref(q, k, v, dev)
        pack = [t.permute(0, 2, 1, 3).reshape(nb * ntok, C) for t in (q, k, v)]
        qkv = torch.cat(pack, dim=1).to(BF).to(dev)
        out = Guarded(nb * ntok, C, BF, dev)                    # the wrapper's row stride is out.shape[-1]
        fn(qkv, out.view, nb, ntok, heads, SCALE)
        _sync(impl)
        flat = lambda t: t.permute(0, 2, 1, 3).reshape(nb * ntok, C)  # noqa: E731
        what = f"attention spatial {impl} ntok={ntok} heads={heads} {pattern}"

        def where(ix):
            r, c = int(ix[0]), int(ix[1])
            return f"(batch {r // ntok}, query {r % ntok}, query tile {r % ntok // 128}, head {c // 64}, dim {c % 64})"

        check(what, "attn", out.view, flat(ref), flat(mag), C_ATTN, where=where)
        out.assert_margins(what)


def _temporal_params():
    out = []
    for T in range(1, 33):
        out.append(pytest.param(T, "kernel", marks=GPU, id=f"T{T}-kernel"))
        if T in (1, 2, 17, 32):
            out.append(pytest.param(T, "standin", id=f"T{T}-standin"))
    return out


@pytest.mark.parametrize("T,impl", _temporal_params())
def test_attention_temporal_edges(T, impl):
    """v3d_attention_temporal for every T it supports: keys >= T must be masked (the 32-row tiles are zero there)."""
    dev = _dev(impl)
    nb, S, heads = 2, 40, 5
    C = heads * 64
    fn = ops.attention_temporal if impl == "kernel" else emu_ops.attention_temporal
    for pattern in ("neg", "dom"):
        g = _gen(300 + T + (50 if pattern == "dom" else 0))
        q, k, v = _attn_inputs(g, nb * S, heads, T, pattern)     # sequences (b, s) of T frames
        ref, mag = (t[0] for t in _attn_ref(q[None], k[None], v[None], dev))
        # [b s, h, t, d] -> rows (b t s), columns (h d)
        lay = lambda t: t.reshape(nb, S, heads, T, 64).permute(0, 3, 1, 2, 4).reshape(nb * T * S, C)  # noqa: E731
        qkv = torch.cat([lay(q), lay(k), lay(v)], dim=1).to(BF).to(dev)
        out = Guarded(nb * T * S, C, BF, dev)                   # the wrapper's row stride is out.shape[-1]
        fn(qkv, out.view, nb, T, S, heads, SCALE)
        _sync(impl)
        what = f"attention temporal T={T} {pattern}"

        def where(ix):
            r, c = int(ix[0]), int(ix[1])
            return f"(batch {r // (T * S)}, frame {r // S % T}, pixel {r % S}, head {c // 64}, dim {c % 64})"

        check(what, "attn", out.view, lay(ref), lay(mag), C_ATTN, where=where)
        out.assert_margins(what)


@pytest.mark.parametrize("blocks,rank,impl", [
    pytest.param((5, 7, 6), 1, "kernel", marks=GPU, id="5-7-6-rank1-kernel"),
    pytest.param((3, 13), 0, "kernel", marks=GPU, id="3-13-rank0-kernel"),
    pytest.param((11, 10, 11), 2, "kernel", marks=GPU, id="11-10-11-rank2-kernel"),
    pytest.param((5, 7, 6), 1, "standin", id="5-7-6-rank1-standin"),
])
def test_attention_temporal_kv_edges(blocks, rank, impl):
    """The frame-sharded form: this rank's Tq query frames against all Tk key frames of a rank-major K|V buffer with
    uneven rank blocks, a gap between the ranks' regions and per-frame CFG-half strides (kv_bstride = block x S)."""
    dev = _dev(impl)
    nb, S, heads = 2, 24, 3
    C = heads * 64
    Tk = sum(blocks)
    f0 = sum(blocks[:rank])
    Tq = blocks[rank]
    kv_row, kv_bstride, base = [], [], 0
    for n in blocks:
        for lf in range(n):
            kv_row.append(base + lf * S)
            kv_bstride.append(n * S)
        base += nb * n * S + 8                                   # 8 unused rows between the ranks' regions
    fn = ops.attention_temporal_kv if impl == "kernel" else emu_ops.attention_temporal_kv
    for pattern in ("neg", "dom"):
        g = _gen(500 + Tk + rank + (9 if pattern == "dom" else 0))
        q, k, v = _attn_inputs(g, nb * S, heads, Tk, pattern)    # all Tk frames; queries are frames f0 .. f0 + Tq
        qs = q[:, :, f0:f0 + Tq]
        ref, mag = (t[0] for t in _attn_ref(qs[None], k[None], v[None], dev))
        lay = lambda t, n: t.reshape(nb, S, heads, n, 64).permute(0, 3, 1, 2, 4).reshape(nb * n * S, C)  # noqa: E731
        kvbuf = torch.zeros(base, 2 * C, dtype=F64)
        kk = k.reshape(nb, S, heads, Tk, 64).permute(0, 3, 1, 2, 4).reshape(nb, Tk, S, C)
        vv = v.reshape(nb, S, heads, Tk, 64).permute(0, 3, 1, 2, 4).reshape(nb, Tk, S, C)
        for f in range(Tk):
            for b in range(nb):
                r = kv_row[f] + b * kv_bstride[f]
                kvbuf[r:r + S, :C] = kk[b, f]
                kvbuf[r:r + S, C:] = vv[b, f]
        qbuf = torch.zeros(nb * Tq * S, C + 64, dtype=F64)
        qbuf[:, :C] = lay(qs, Tq)
        qd = qbuf.to(BF).to(dev)
        out = Guarded(nb * Tq * S, C, BF, dev, ld=C + 16)
        fn(qd[:, :C], kvbuf.to(BF).to(dev), out.view, nb, Tq, S, heads, kv_row, kv_bstride, SCALE)
        _sync(impl)
        what = f"attention temporal_kv blocks={blocks} rank={rank} {pattern}"

        def where(ix):
            r, c = int(ix[0]), int(ix[1])
            return f"(batch {r // (Tq * S)}, frame {f0 + r // S % Tq}, pixel {r % S}, head {c // 64}, dim {c % 64})"

        check(what, "attn", out.view, lay(ref, Tq), lay(mag, Tq), C_ATTN, where=where)
        out.assert_margins(what)


# ------------------------------------------------------------------------------------------------------------------
# norms
# ------------------------------------------------------------------------------------------------------------------
def _norm_ref(xg, eps):
    """xg [..., n]: the values behind one statistic -> (xhat, core magnitude)"""
    mu = xg.mean(-1, keepdim=True)
    var = ((xg - mu) ** 2).mean(-1, keepdim=True)
    e2 = (xg * xg).mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(var + eps)
    core = rstd * (xg.abs() + mu.abs() + (xg - mu).abs() * e2 * rstd ** 2)
    return (xg - mu) * rstd, core


def _gn_input(g, ns, rows, C, groups=32):
    """x [ns, rows, C]: group 0 constant, group 1 variance ~ eps, groups 2 / 3 with |mu| / sigma = 8 / 64, and 30-sigma
    outlier rows at 0, rows - 1 and 2^k +- 1 in the other groups (a different group per row)"""
    cpg = C // groups
    x = _randn(g, ns, rows, C)
    grp = lambda i: slice(i * cpg, (i + 1) * cpg)  # noqa: E731
    x[..., grp(0)] = 3.140625
    x[..., grp(1)] = 0.003 * _randn(g, ns, rows, cpg)
    x[..., grp(2)] = 8.0 + x[..., grp(2)]
    x[..., grp(3)] = -64.0 + x[..., grp(3)]
    special = {0, rows - 1} | {(1 << kk) + d for kk in range(1, 20) for d in (-1, 1) if (1 << kk) + d < rows}
    for i, r in enumerate(sorted(special)):
        gi = 4 + (5 * i) % (groups - 4)
        x[:, r, grp(gi)] = 30.0 * (1 if i % 2 else -1) + x[:, r, grp(gi)]
    return x.to(BF).double()


GN_CASES = [  # (variant, C, ns, frames, hw, silu): C = 320 launches the <256, 3> instances, C = 2560 the <512, 1> ones
    ("pair", 320, 2, 3, 300, False), ("pair", 2560, 2, 2, 64, True),
    ("fused", 320, 2, 3, 300, False), ("fused", 320, 3, 1, 1000, True), ("fused", 2560, 2, 2, 64, False),
    ("det_pair", 320, 2, 3, 300, False), ("det_pair", 2560, 2, 2, 64, True),
    ("det", 320, 2, 3, 300, True), ("det", 320, 3, 1, 1000, False), ("det", 2560, 2, 2, 64, False),
]


@pytest.mark.parametrize("variant,C,ns,frames,hw,silu,impl", _impl_params(
    GN_CASES, lambda c: True, [f"{v}-C{c}-ns{n}-{f}x{h}{'-silu' if s else ''}" for v, c, n, f, h, s in GN_CASES]))
def test_groupnorm_edges(variant, C, ns, frames, hw, silu, impl):
    """Statistics + apply pair, the single launch, and the deterministic partials / fold-apply pair and single launch."""
    dev = _dev(impl)
    g = _gen(700 + C + ns + hw)
    rows = frames * hw
    groups, eps = 32, 1e-5
    cpg = C // groups
    x = _gn_input(g, ns, rows, C)
    gamma = _randn(g, C).float().double()
    beta = _randn(g, C).float().double()
    xg = x.reshape(ns, rows, groups, cpg).permute(0, 2, 1, 3).reshape(ns, groups, rows * cpg)
    xhat, core = _norm_ref(xg, eps)
    back = lambda t: t.reshape(ns, groups, rows, cpg).permute(0, 2, 1, 3).reshape(ns * rows, C)  # noqa: E731
    y = back(xhat) * gamma + beta
    mag = back(core) * gamma.abs() + beta.abs()
    if silu:
        y = y * torch.sigmoid(y)
    o = ops if impl == "kernel" else emu_ops
    xd, gd, bd = _bf(x.reshape(ns * rows, C), dev), gamma.float().to(dev), beta.float().to(dev)
    out = Guarded(ns * rows, C, BF, dev)
    if variant == "pair":
        stats = torch.empty(ns, groups, 2, dtype=F64, device=dev)
        o.groupnorm_stats(xd, stats, rows, ns, C)
        o.groupnorm_apply(xd, out.view, stats, gd, bd, rows, ns, C, eps, silu)
    elif variant == "fused":
        o.groupnorm(xd, out.view, gd, bd, rows, ns, C, eps, silu, o.groupnorm_workspace(dev))
    elif variant == "det_pair":
        nblk = o.groupnorm_det_blocks(rows, hw)
        part = torch.empty(ns, nblk, groups, 2, dtype=torch.float32, device=dev)
        o.groupnorm_partials(xd, part, rows, hw, ns, C)
        o.groupnorm_fold_apply(xd, out.view, part, gd, bd, rows, ns, C, eps, silu, nblk)
    else:
        ws = o.groupnorm_det_workspace(dev, o.groupnorm_det_workspace_bytes(rows, hw, ns, groups))
        o.groupnorm_det(xd, out.view, gd, bd, rows, hw, ns, C, eps, silu, ws)
    _sync(impl)
    what = f"groupnorm {variant} C={C} ns={ns} rows={rows}{' silu' if silu else ''}"

    def where(ix):
        r, c = int(ix[0]), int(ix[1])
        return f"(sample {r // rows}, row {r % rows}, group {c // cpg}, channel {c})"

    fam = "norm+silu" if silu else "norm"
    check(what, fam, out.view, y, mag, c_silu(C_NORM) if silu else 2 * C_NORM, exact=not silu, where=where)
    out.assert_margins(what)
    if not silu:
        # the constant group normalises to beta: its mean is exact and its (maybe slightly negative) variance clamped
        const = out.view.reshape(ns, rows, C)[:, :, :cpg].double().cpu()
        assert (const - beta[:cpg]).abs().max() <= (2 * C_NORM * mag.reshape(ns, rows, C)[:, :, :cpg]).max() + \
            2.0 ** -8 * beta[:cpg].abs().max(), f"{what}: a constant group does not normalise to beta"


LN_C = [64, 200, 320, 512, 640, 768, 1024, 1152, 1280, 1536, 1792, 2048]


@pytest.mark.parametrize("C,impl", _impl_params([(c,) for c in LN_C], lambda c: True, [f"C{c}" for c in LN_C]))
def test_layernorm_edges(C, impl):
    """Every LayerNorm instance: layernorm40<8 / 16 / 32> (C = 320 / 640 / 1280) and the generic kernel at 1 .. 5 and 8
    vectors per lane, partly empty lanes included (C = 200, 1152, 1536, 1792); a row tail; then the fused per-frame
    add (3 rows per frame: the frame changes inside every CTA) with its bf16 sum."""
    dev = _dev(impl)
    g = _gen(900 + C)
    rows, rpf, eps = 8 * 37 + 5, 3, 1e-5
    x = 2.0 * _randn(g, rows, C)
    x[:, 0] -= 8.0                                               # the first and last channel of every row planted
    x[:, C - 1] += 8.0
    x[::7] += 3.0                                                # mean offsets on every 7th row
    x = x.to(BF).double()
    gamma = _randn(g, C).float().double()
    beta = _randn(g, C).float().double()
    add = _randn(g, (rows + rpf - 1) // rpf, C).float().double()
    o = ops if impl == "kernel" else emu_ops

    def where(ix):
        return f"(row {int(ix[0])}, CTA row {int(ix[0]) % 8}, channel {int(ix[1])}, lane {int(ix[1]) // 8 % 32})"

    for fused in (False, True):
        z = x
        if fused:
            # x + add in fp32 (the contract's fp32 add), rounded once to bf16: the residual stream is the LN input
            z = (x.float() + add.float().repeat_interleave(rpf, 0)[:rows]).to(BF).double()
        xhat, core = _norm_ref(z, eps)
        y = xhat * gamma + beta
        mag = core * gamma.abs() + beta.abs()
        out = Guarded(rows, C, BF, dev)
        what = f"layernorm C={C}{' +add' if fused else ''}"
        if fused:
            ysum = Guarded(rows, C, BF, dev)
            o.layernorm(_bf(x, dev), out.view, gamma.float().to(dev), beta.float().to(dev), rows, C, eps,
                        add=add.float().to(dev), ysum=ysum.view, rows_per_frame=rpf)
            _sync(impl)
            zz = x + add.float().double().repeat_interleave(rpf, 0)[:rows]
            check(what + " ysum", "norm", ysum.view, zz, zz.abs(), 2 * U, exact=True, where=where)
            ysum.assert_margins(what + " ysum")
        else:
            o.layernorm(_bf(x, dev), out.view, gamma.float().to(dev), beta.float().to(dev), rows, C, eps)
            _sync(impl)
        check(what, "norm", out.view, y, mag, 2 * C_NORM, exact=True, where=where)
        out.assert_margins(what)


def _softmax_input(g, rows, n):
    """random rows, plus: -1e30 padded columns, -inf padded columns, a row with one finite entry (first and last)"""
    x = 3.0 * _randn(g, rows, n)
    pad = max(1, n // 4)
    x[1, n - pad:] = -1e30
    x[2, n - pad:] = -math.inf
    x[3, :] = -math.inf
    x[3, n - 1] = 0.5
    x[4, :] = -1e30
    x[4, 0] = -2.0
    return x


def _softmax_ref(x, scale):
    s = x * scale
    m = s.max(-1, keepdim=True).values
    p = torch.softmax(s, dim=-1)
    arg = torch.where(torch.isfinite(s), s - m, torch.zeros_like(s))
    return p, p * (1.0 + arg.abs() + m.abs())


@pytest.mark.parametrize("n,impl", _impl_params([(n,) for n in (4, 320, 4096, 4100)], lambda c: True,
                                                [f"n{n}" for n in (4, 320, 4096, 4100)]))
def test_softmax_rows_f32_edges(n, impl):
    dev = _dev(impl)
    g = _gen(1100 + n)
    rows, scale = 9, 0.7
    x = _softmax_input(g, rows, n).float().double()
    p, mag = _softmax_ref(x, scale)
    out = Guarded(rows, n, BF, dev)
    (ops if impl == "kernel" else emu_ops).softmax_rows_f32(x.float().to(dev), out.view, rows, n, scale)
    _sync(impl)
    check(f"softmax_rows_f32 n={n}", "softmax", out.view, p, mag, C_SOFTMAX,
          where=lambda ix: f"(row {int(ix[0])}, column {int(ix[1])}, thread {int(ix[1]) // 4 % 256})")
    out.assert_margins(f"softmax_rows_f32 n={n}")


@pytest.mark.gpu
@pytest.mark.parametrize("n", [8, 320, 4096, 4104])
def test_softmax_rows_bf16_edges(n):
    g = _gen(1200 + n)
    rows, scale = 9, 0.7
    x = _softmax_input(g, rows, n).to(BF).double()
    p, mag = _softmax_ref(x, scale)
    buf = Guarded(rows, n, BF, "cuda")
    buf.view.copy_(x.to(BF))
    ops.softmax_rows(buf.view, rows, n, scale)
    torch.cuda.synchronize()
    check(f"softmax_rows n={n}", "softmax", buf.view, p, mag, C_SOFTMAX,
          where=lambda ix: f"(row {int(ix[0])}, column {int(ix[1])}, thread {int(ix[1]) // 8 % 256})")
    buf.assert_margins(f"softmax_rows n={n}")


# ------------------------------------------------------------------------------------------------------------------
# time_mix_conv
# ------------------------------------------------------------------------------------------------------------------
TMC = [(c, t) for c in (1, 2, 3, 4) for t in (1, 2, 18)]


@pytest.mark.parametrize("C,T,impl", _impl_params(TMC, lambda c: True, [f"C{c}-T{t}" for c, t in TMC]))
def test_time_mix_conv_edges(C, T, impl):
    """Conv3d (3, 1, 1) over frames, C <= 4: the first and last frame of every video x16, so a tap that reads across a
    video boundary or misses the zero padding is an O(1) error."""
    dev = _dev(impl)
    g = _gen(1300 + 10 * C + T)
    nb, HW, ldx = 2, 37, 8
    x = _randn(g, nb, T, HW, ldx)
    x[:, 0] *= 16.0
    x[:, T - 1] *= 16.0
    x = x.float().double()
    w = _randn(g, C, C, 3).float().double()
    bias = _randn(g, C).float().double()
    xs = x[..., :C]
    ref = bias.reshape(1, 1, C, 1).expand(nb, T, C, HW).clone()
    mag = bias.abs().reshape(1, 1, C, 1).expand(nb, T, C, HW).clone()
    for tap in range(3):
        src = torch.arange(T) + tap - 1
        ok = (src >= 0) & (src < T)
        xt = torch.zeros(nb, T, HW, C, dtype=F64)
        xt[:, ok] = xs[:, src[ok]]
        ref += torch.einsum("oi,btpi->btop", w[:, :, tap], xt)
        mag += torch.einsum("oi,btpi->btop", w[:, :, tap].abs(), xt.abs())
    out = Guarded(nb * T * C, HW, torch.float32, dev)
    (ops if impl == "kernel" else emu_ops).time_mix_conv(x.float().to(dev).reshape(-1, ldx), ldx, w.float().to(dev),
                                                         bias.float().to(dev), out.view, nb, T, HW, C)
    _sync(impl)
    check(f"time_mix_conv C={C} T={T}", "mix", out.view, ref.reshape(nb * T * C, HW), mag.reshape(nb * T * C, HW),
          C_MIX, f32=True, where=lambda ix: f"(video {int(ix[0]) // (T * C)}, frame {int(ix[0]) // C % T}, "
                                            f"channel {int(ix[0]) % C}, pixel {int(ix[1])})")
    out.assert_margins(f"time_mix_conv C={C} T={T}")
