"""PixelNeRF scene conditioning on the H100: the fused kernels (csrc/pixelnerf.cu) against the fp64 restatement of
oracle/ref_pixelnerf.py, and the module against the reference fixtures (oracle/make_golden_scene.py).

Bound of the kernel check.  The restatement (precision="kernel") rounds to bf16 at exactly the points the kernel
rounds: weights, the MLP input row (mean | std | positional encoding), both hidden activations of each MLP, and the
per-ray feature before the decoder.  Between those points the kernel computes in fp32 and the restatement in fp64.
An fp32 value within its own rounding error of a bf16 rounding boundary rounds the other way and moves one element by
one bf16 ulp (2^-8 relative); the positional encoding dominates, because sin(x f) is evaluated at arguments up to
~100 rad whose fp32 rounding (~6e-6 absolute) flips about 3e-3 of its roundings.  That floor is measured, not guessed:
the same restatement with fp32 arithmetic between the rounding points (precision="kernel32") sits at rel-L2 ~1e-3
from fp64 on these inputs.  The kernel's fp32 order differs from torch's, so its flips are different ones but as
many: it must stay within twice that floor (+1e-4), and no single element may be off by more than 1e-2 of the
output scale.
"""
from __future__ import annotations

import pytest
import torch

from oracle import ref_pixelnerf as R
from oracle.make_golden_scene import look_at_cams

pytestmark = pytest.mark.gpu

FLOOR_FACTOR, FLOOR_SLACK, MAX_ABS = 2.0, 1e-4, 1e-2


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30)), float((a - b).abs().max() / b.abs().max())


def _module(C, ns, std, pe, interp="bilinear", padding="border", disparity=False, seed=0, sampler=None):
    from v3d_b200.pixelnerf import PixelNeRF

    m = PixelNeRF(num_samples_per_ray=ns, feature_dim=C, interp=interp, padding=padding, disparity=disparity,
                  use_feats_std=std, use_pos_emb=pe, jitter_sampler=sampler)
    sd = R.state_dict(m.d_in, seed, scale=2.0)
    m.load_state_dict(sd)
    return m.cuda(), sd


def _run_case(*, B=1, T=2, S=2, C=3, H=20, W=20, rs=8, ns=16, std=True, pe=True, interp="bilinear",
              padding="border", disparity=False, cams=None, scams=None, img=None, seed=0):
    g = torch.Generator().manual_seed(seed)
    if cams is None:
        cams = torch.stack([look_at_cams(T, 0.2 + 0.9 * b) for b in range(B)])
    if scams is None:
        scams = torch.stack([look_at_cams(S, 1.0 + 0.6 * b, 2.3) for b in range(B)])
    if img is None:
        img = torch.rand(B, S, C, H, W, generator=g) * 2 - 1
    u = torch.rand(ns, B * T, rs * rs, 1, generator=g) if not disparity else torch.rand(ns, generator=g)
    m, sd = _module(C, ns, std, pe, interp, padding, disparity, seed, sampler=lambda shape, dev: u.to(dev))
    dev = torch.device("cuda")
    sc2w, sk = scams[..., :16].reshape(B, S, 4, 4), scams[..., 16:].reshape(B, S, 3, 3)
    rgb, fe = m(img.to(dev), sc2w.to(dev), sk.to(dev), cams[..., :16].reshape(B, T, 4, 4).to(dev),
                cams[..., 16:].reshape(B, T, 3, 3).to(dev), rs)
    torch.cuda.synchronize()
    jit = u.reshape(ns, -1) if not disparity else torch.linspace(0, 1 - 1.0 / ns, ns) + u * (1.0 / ns)
    kw = dict(use_std=std, use_pe=pe, interp=interp, padding=padding, disparity=disparity)
    r_rgb, r_fe, _ = R.pixelnerf(sd, img, sc2w, sk, cams, rs, jit, ns, precision="kernel", **kw)
    f_rgb, f_fe, _ = R.pixelnerf(sd, img, sc2w, sk, cams, rs, jit, ns, precision="kernel32", **kw)
    return (rgb, fe), ((r_rgb, f_rgb), (r_fe, f_fe)), m


def _check(got, ref, what):
    for name, a, (b, floor32) in zip(("rgb", "feats"), got, ref):
        assert torch.isfinite(a).all(), f"{what}: non-finite {name}"
        rl2, mx = _rel(a, b)
        bound = FLOOR_FACTOR * _rel(floor32, b)[0] + FLOOR_SLACK
        assert rl2 <= bound and mx <= MAX_ABS, f"{what}: {name} rel-L2 {rl2:.2e} (bound {bound:.2e}), max {mx:.2e}"


@pytest.mark.parametrize("ns", [2, 16, 127, 128, 129, 300])
def test_samples_per_ray(ns):
    got, ref, _ = _run_case(ns=ns, rs=6, seed=ns)
    _check(got, ref, f"ns={ns}")


@pytest.mark.parametrize("S", [1, 2, 4])
@pytest.mark.parametrize("C", [3, 64])
def test_sources_channels(S, C):
    got, ref, _ = _run_case(S=S, C=C, H=18, W=26, rs=7, ns=20, seed=10 * S + C)
    _check(got, ref, f"S={S} C={C}")


@pytest.mark.parametrize("std,pe", [(False, False), (True, False), (False, True)])
def test_std_posenc(std, pe):
    got, ref, _ = _run_case(std=std, pe=pe, C=16, seed=3)
    _check(got, ref, f"std={std} pe={pe}")


@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
@pytest.mark.parametrize("padding", ["border", "zeros"])
def test_interp_padding(interp, padding):
    # wide field of view: many samples project outside the source image
    scams = look_at_cams(2, 1.0, 2.3)
    scams[:, 16] *= 2.5
    scams[:, 20] *= 2.5
    got, ref, _ = _run_case(interp=interp, padding=padding, scams=scams[None], H=15, W=23, seed=7)
    _check(got, ref, f"{interp}/{padding}")


def test_disparity():
    got, ref, _ = _run_case(disparity=True, ns=33, seed=5)
    _check(got, ref, "disparity")


def test_render_size_tail_and_two_batches():
    got, ref, _ = _run_case(B=2, T=3, rs=17, ns=40, H=13, W=31, seed=11)
    _check(got, ref, "rs=17, B=2")
    # b = 2 has its own cameras: the two items must differ
    assert (got[1][0] - got[1][1]).abs().max() > 1e-3


def test_all_rays_miss_and_some_miss():
    far = look_at_cams(2, 0.0, 6.0)
    far[:, 3], far[:, 7], far[:, 11] = far[:, 3] + 40.0, far[:, 7], far[:, 11]  # looking past the box
    got, ref, _ = _run_case(cams=far[None], seed=12)
    _check(got, ref, "all miss")
    wide = look_at_cams(2, 0.5, 1.9)
    wide[:, 16] *= 0.3  # ~120 degree field of view: the border rays miss
    wide[:, 20] *= 0.3
    got, ref, _ = _run_case(cams=wide[None], rs=12, seed=13)
    _check(got, ref, "some miss")


def test_behind_source_camera():
    # a source camera inside the box: part of every ray lies behind it and projects through -z (not masked)
    inside = look_at_cams(2, 0.7, 0.4)
    got, ref, _ = _run_case(scams=inside[None], padding="zeros", seed=14)
    _check(got, ref, "behind / far outside")


@pytest.mark.parametrize("interp", ["bilinear", "nearest"])
def test_planted_texel(interp):
    # one lit texel per source and channel: a shifted coordinate, a dropped sample or a dropped source changes the
    # output far beyond the bound
    S, C, H, W = 3, 4, 11, 13
    img = torch.zeros(1, S, C, H, W)
    for s in range(S):
        for c in range(C):
            img[0, s, c, (3 + 2 * s + c) % H, (5 + 3 * s + 2 * c) % W] = 4.0 + s + c
    got, ref, _ = _run_case(S=S, C=C, H=H, W=W, img=img, interp=interp, rs=16, ns=48, seed=15)
    _check(got, ref, f"planted {interp}")


def test_deterministic_and_sentinels():
    from v3d_b200 import ops

    (rgb, fe), _, m = _run_case(B=2, T=2, rs=9, ns=37, seed=16)
    (rgb2, fe2), _, _ = _run_case(B=2, T=2, rs=9, ns=37, seed=16)
    assert torch.equal(rgb, rgb2) and torch.equal(fe, fe2)
    # the render writes every row of a caller-owned, NaN-filled feature buffer, with the bytes of a fresh one
    g = torch.Generator().manual_seed(17)
    cams = torch.stack([look_at_cams(2, 0.2 + 0.9 * b) for b in range(2)]).cuda()
    scams = torch.stack([look_at_cams(2, 1.0 + 0.6 * b, 2.3) for b in range(2)]).cuda()
    img = (torch.rand(2, 2, 3, 20, 20, generator=g) * 2 - 1).cuda()
    args = (img, scams[..., :16].reshape(2, 2, 4, 4), scams[..., 16:].reshape(2, 2, 3, 3),
            cams[..., :16].reshape(2, 2, 4, 4), cams[..., 16:].reshape(2, 2, 3, 3), 9)
    fresh = m.ray_features(*args)
    feat_nan = torch.full((2 * 2 * 81, 128), float("nan"), device="cuda")
    m.ray_features(*args, feat=feat_nan)
    torch.cuda.synchronize()
    assert torch.isfinite(feat_nan).all() and torch.equal(feat_nan, fresh)
    # the decoder writes every element of caller-owned buffers: refill them with a sentinel and decode again
    feat = torch.randn(2 * 2 * 81, 128, device="cuda")
    _, dec = m.packed(torch.device("cuda"))
    out1 = (torch.full((4, 3, 81), 12345.0, device="cuda"), torch.full((4, 128, 81), -777.0, device="cuda"))
    out2 = (torch.full((4, 3, 81), float("nan"), device="cuda"), torch.full((4, 128, 81), float("nan"), device="cuda"))
    ops.pixelnerf_decode(feat, 81, dec, *out1)
    ops.pixelnerf_decode(feat, 81, dec, *out2)
    torch.cuda.synchronize()
    assert torch.equal(out1[0], out2[0]) and torch.equal(out1[1], out2[1])


@pytest.mark.parametrize("tag", ["scene_s1", "scene_s3"])
def test_embedder_meets_reference_fixture(tag):
    # the real reference PixelNeRFEmbedder's fp32 output; bound on the whole output and on its pixel-varying part
    # (R.fixture_errors).  The same module fed zeroed or swapped sources must miss that bound.
    from pathlib import Path

    from v3d_b200.pixelnerf import PixelNeRFEmbedder

    fx = torch.load(Path(__file__).parent / "golden" / f"{tag}.pt", weights_only=False)
    cs = fx["case"]
    jit = fx["jitter"]
    emb = PixelNeRFEmbedder(
        {"target": "v3d_b200.sgm.modules.encoders.pixelnerf.ImageEncoder"},
        {"target": "v3d_b200.sgm.modules.encoders.pixelnerf.PixelNeRF",
         "params": dict(num_samples_per_ray=cs["ns"], feature_dim=cs["C"], use_feats_std=cs["use_feats_std"],
                        use_pos_emb=cs["use_pos_emb"])},
        render_size=cs["render_size"], num_video_frames=cs["T"]).cuda()
    emb.pixelnerf_encoder.load_state_dict(fx["state_dict"])
    emb.pixelnerf_encoder.jitter_sampler = lambda shape, dev: jit.to(dev)

    def run(inputs):
        return emb({k: (v.cuda() if isinstance(v, torch.Tensor) else v) for k, v in inputs.items()})

    rgb, fe = run(fx["inputs"])
    for name, a, b in (("rgb", rgb, fx["rgb"]), ("feats", fe, fx["feats"])):
        whole, varying = R.fixture_errors(a, b)
        cos = float(torch.nn.functional.cosine_similarity(a.double().cpu().flatten(), b.double().flatten(), dim=0))
        assert whole <= R.FIXTURE_REL_L2 and varying <= R.FIXTURE_REL_L2 and cos >= 0.999, \
            f"{tag} {name}: rel-L2 {whole:.2e}, pixel-varying {varying:.2e}, cosine {cos:.6f}"
    for what, inp in R.altered_sources(fx["inputs"]).items():
        rgb, fe = run(inp)
        for name, a, b in (("rgb", rgb, fx["rgb"]), ("feats", fe, fx["feats"])):
            assert R.fixture_errors(a, b)[1] > 3 * R.FIXTURE_REL_L2, f"{tag} {what} {name} passes the bound"


def test_shape_mismatches_raise_before_launch():
    from v3d_b200 import ops

    m, _ = _module(3, 16, True, True)
    cams = look_at_cams(3, 0.2)[None].repeat(2, 1, 1).cuda()
    scams = look_at_cams(1, 1.0, 2.3)[None].cuda()
    img = torch.rand(1, 1, 3, 12, 12, device="cuda")  # one source batch for two target batches
    with pytest.raises(ValueError):
        m(img, scams[..., :16].reshape(1, 1, 4, 4), scams[..., 16:].reshape(1, 1, 3, 3),
          cams[..., :16].reshape(2, 3, 4, 4), cams[..., 16:].reshape(2, 3, 3, 3), 4)
    agg, dec = m.packed(torch.device("cuda"))
    rays = torch.zeros(2 * 3 * 16, 8, device="cuda")
    limits = torch.zeros(2, dtype=torch.int32, device="cuda")
    jit = torch.rand(16, 96, device="cuda")
    w2c = torch.zeros(1, 1, 3, 4, device="cuda")
    k = torch.ones(1, 1, 4, device="cuda")
    feat = torch.empty(96, 128, device="cuda")
    with pytest.raises(RuntimeError, match="source batches"):
        ops.pixelnerf_render(rays, limits, jit, img, w2c, k, 48, 16, m.flags, 2.0, 1e-4, agg, m.d_in, feat)
    with pytest.raises(RuntimeError, match="jitter"):
        ops.pixelnerf_render(rays, limits, jit[:8], img.repeat(2, 1, 1, 1, 1), w2c.repeat(2, 1, 1, 1),
                             k.repeat(2, 1, 1), 48, 16, m.flags, 2.0, 1e-4, agg, m.d_in, feat)
    with pytest.raises(RuntimeError, match="packed MLP"):
        ops.pixelnerf_render(rays, limits, jit, img.repeat(2, 1, 1, 1, 1), w2c.repeat(2, 1, 1, 1),
                             k.repeat(2, 1, 1), 48, 16, m.flags, 2.0, 1e-4, dec, m.d_in, feat)
    with pytest.raises(RuntimeError, match="rgb"):
        ops.pixelnerf_decode(feat, 16, dec, torch.empty(6, 3, 15, device="cuda"), torch.empty(6, 128, 16, device="cuda"))
