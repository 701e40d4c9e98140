"""The ancestral / DPM++ / LMS step kernels and their drop-in samplers on the GPU.

  * kernels against an fp64 restatement of their formulas (rel-L2 <= 1e-6: fp32 rounding) and bit for bit against
    their torch stand-ins (tests/emu_ops.py, same operation order), at the V3D_512 state size and at an odd
    per-sample size, with sigma_next = 0 rows and `out` aliasing `x`;
  * the four drop-ins with the bf16 VideoUNet (unet_small weights) and the fixtures' seeded noise against the real
    reference's outputs (tests/golden/edm_small_{euler_ancestral,dpmpp2s,dpmpp2m,lms}.pt);
  * no device->host synchronisation inside a sampler call.
"""
import json
import sys
from pathlib import Path

import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, str(Path(__file__).resolve().parent))
DEV = "cuda"
GOLD = Path(__file__).resolve().parent / "golden"
MANIFEST = json.loads((GOLD / "MANIFEST.json").read_text())          # the unet_small weights
SAMPLERS = json.loads((GOLD / "SAMPLERS.json").read_text())          # the fixtures of oracle/make_golden_samplers.py
SHAPES = [(18, 4, 64, 64), (5, 3, 7, 11)]        # V3D_512's [T, 4, 64, 64] and an odd per_sample (231)
BASE = "v3d_b200.sgm.modules.diffusionmodules."


def _rand(shape, seed, scale=1.0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randn(*shape, device=DEV, generator=g) * scale


def _f32(v: float) -> float:
    return float(torch.tensor(v, dtype=torch.float32))


def _rel(a, b):
    return ((a.double() - b.double()).norm() / b.double().norm().clamp_min(1e-300)).item()


def _run_both(name, make_args, alias: bool):
    """Kernel and stand-in on identical inputs; `make_args(out)` builds the argument list around the output buffer
    (alias: out is x itself).  Returns (kernel result, stand-in result, the kernel's arguments)."""
    import emu_ops
    from v3d_b200 import ops

    results = []
    for impl in (ops, emu_ops):
        args = make_args(None if alias else "fresh")
        getattr(impl, name)(*args)
        results.append(args)
    torch.cuda.synchronize()
    return results


def _nps(shape):
    return shape[0], shape[1] * shape[2] * shape[3]


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("sigma_next", [0.0, 2.5])
@pytest.mark.parametrize("alias", [False, True])
def test_ancestral_euler_step_kernel(shape, sigma_next, alias):
    n, per = _nps(shape)
    sigma, s_noise = _f32(14.6), _f32(0.95)
    sigma_down, sigma_up = (_f32(1.2), _f32(2.2)) if sigma_next > 0 else (0.0, 0.0)
    x0, den, noise = _rand(shape, 1, sigma), _rand(shape, 2), _rand(shape, 3)

    def make(out):
        x = x0.clone()
        return [x, den, noise, x if out is None else torch.empty_like(x), sigma, sigma_down, sigma_up, sigma_next,
                s_noise, n, per]

    k, s = _run_both("ancestral_euler_step", make, alias)
    x, d, z = x0.double(), den.double(), noise.double()
    want = x + (sigma_down - sigma) * ((x - d) / sigma)
    if sigma_next > 0:
        want = want + z * s_noise * sigma_up
    assert _rel(k[3], want) <= 1e-6
    assert torch.equal(k[3], s[3])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("alias", [False, True])
def test_dpmpp2s_stage_kernel(shape, alias):
    n, per = _nps(shape)
    m1, m2 = _f32(0.43), _f32(-0.57)
    x0, den = _rand(shape, 4, 20.0), _rand(shape, 5)

    def make(out):
        x = x0.clone()
        return [x, den, x if out is None else torch.empty_like(x), m1, m2, n, per]

    k, s = _run_both("dpmpp2s_stage", make, alias)
    assert _rel(k[2], m1 * x0.double() - m2 * den.double()) <= 1e-6
    assert torch.equal(k[2], s[2])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("last", [False, True])
@pytest.mark.parametrize("alias", [False, True])
def test_dpmpp2s_step_kernel(shape, last, alias):
    """last: sigma_down = sigma_next = 0 (the combine falls back to the Euler step and drops the noise)."""
    n, per = _nps(shape)
    sigma, s_noise, m3, m4 = _f32(3.1), _f32(1.0), _f32(0.19), _f32(-0.81)
    sigma_down, sigma_up, sigma_next = (0.0, 0.0, 0.0) if last else (_f32(0.6), _f32(0.9), _f32(1.1))
    x0, den, den2, noise = _rand(shape, 6, 4.0), _rand(shape, 7), _rand(shape, 8), _rand(shape, 9)

    def make(out):
        x = x0.clone()
        return [x, den, den2, noise, x if out is None else torch.empty_like(x), sigma, sigma_down, sigma_up,
                sigma_next, s_noise, m3, m4, n, per]

    k, s = _run_both("dpmpp2s_step", make, alias)
    x, d, d2, z = x0.double(), den.double(), den2.double(), noise.double()
    want = x + (sigma_down - sigma) * ((x - d) / sigma) if last else m3 * x - m4 * d2
    if sigma_next > 0:
        want = want + z * s_noise * sigma_up
    assert _rel(k[4], want) <= 1e-6
    assert torch.equal(k[4], s[4])


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("second_order", [False, True])
@pytest.mark.parametrize("alias", [False, True])
def test_dpmpp2m_step_kernel(shape, second_order, alias):
    n, per = _nps(shape)
    m1, m2, m3, m4 = _f32(0.21), _f32(-0.79), _f32(2.19), _f32(1.19)
    x0, den, old = _rand(shape, 10, 8.0), _rand(shape, 11), _rand(shape, 12)

    def make(out):
        x = x0.clone()
        return [x, den, old.clone(), x if out is None else torch.empty_like(x), m1, m2, m3, m4, second_order, n, per]

    k, s = _run_both("dpmpp2m_step", make, alias)
    x, d, o = x0.double(), den.double(), old.double()
    want = m1 * x - m2 * ((m3 * d - m4 * o) if second_order else d)
    assert _rel(k[3], want) <= 1e-6
    assert torch.equal(k[3], s[3])
    assert torch.equal(k[2], den) and torch.equal(s[2], den)      # the history now holds this step's estimate


@pytest.mark.parametrize("shape", SHAPES)
@pytest.mark.parametrize("order,ring_slots,step", [(1, 4, 0), (3, 4, 2), (4, 4, 9), (8, 8, 11)])
@pytest.mark.parametrize("alias", [False, True])
def test_lms_step_kernel(shape, order, ring_slots, step, alias):
    n, per = _nps(shape)
    sigma = _f32(1.7)
    coeffs = [_f32(v) for v in (1.3, -0.61, 0.37, -0.22, 0.11, -0.05, 0.03, -0.01)[:order]]
    slots = [(step - j) % ring_slots for j in range(order)]
    x0, den, ring0 = _rand(shape, 13, 2.0), _rand(shape, 14), _rand((ring_slots,) + shape, 15)

    def make(out):
        x = x0.clone()
        return [x, den, ring0.clone(), x if out is None else torch.empty_like(x), sigma, coeffs, slots, n, per]

    k, s = _run_both("lms_step", make, alias)
    x, d = x0.double(), den.double()
    slope = (x - d) / sigma
    want = coeffs[0] * slope
    for c, j in zip(coeffs[1:], slots[1:]):
        want = want + c * ring0[j].double()
    assert _rel(k[3], x + want) <= 1e-6
    assert torch.equal(k[3], s[3]) and torch.equal(k[2], s[2])
    assert _rel(k[2][slots[0]], slope) <= 1e-6
    untouched = [j for j in range(ring_slots) if j != slots[0]]
    assert torch.equal(k[2][untouched], ring0[untouched])


def test_lms_step_rejects_order_above_eight():
    from v3d_b200 import ops

    x = torch.zeros(1, 4, 2, 2, device=DEV)
    ring = torch.zeros(9, 1, 4, 2, 2, device=DEV)
    with pytest.raises(RuntimeError, match="order"):
        ops.lms_step(x, x, ring, x, 1.0, [0.1] * 9, list(range(9)), 1, 16)


# ---------------------------------------------------------------------------------------------------------------------
# the drop-ins with the real bf16 VideoUNet against the reference fixtures
# ---------------------------------------------------------------------------------------------------------------------
TAGS = ["edm_small_euler_ancestral", "edm_small_dpmpp2s", "edm_small_dpmpp2m", "edm_small_lms"]
_net = {}


def _unet_small():
    if "net" not in _net:
        from oracle import synth
        from test_samplers_cpu import UNET_KW
        from v3d_b200.unet import VideoUNet

        mu = MANIFEST["unet_small"]
        net = VideoUNet(**dict(UNET_KW, model_channels=mu["model_channels"]))
        net.load_state_dict(synth.synth_state_dict(net.param_shapes(), seed=mu["weight_seed"]), strict=True)
        _net["net"] = net.to(DEV).eval()
    return _net["net"]


@pytest.mark.parametrize("tag", TAGS)
def test_dropin_samplers_match_reference(tag):
    from oracle import make_golden_samplers as mgs
    from oracle import synth
    from test_samplers_cpu import HOST_PATH_BOUND
    from v3d_b200 import sampling

    m = SAMPLERS[tag]
    gold = torch.load(GOLD / f"{tag}.pt")
    T, hw = m["T"], m["latent_hw"]
    x, c, uc = synth.synth_inputs(T, hw)
    to = lambda d: {k: v.to(DEV) for k, v in d.items()}  # noqa: E731
    params = {k: m[k] for k in ("eta", "s_noise", "order") if m.get(k) is not None}
    sampler = getattr(sampling, m["sampler"])(
        num_steps=m["num_steps"],
        discretization_config={"target": BASE + "discretizer.EDMDiscretization", "params": {"sigma_max": m["sigma_max"]}},
        guider_config={"target": BASE + "guiders.LinearPredictionGuider",
                       "params": {"max_scale": m["max_scale"], "min_scale": m["min_scale"], "num_frames": T}},
        **params)
    if m.get("noise_seed") is not None:
        sampler.noise_sampler = mgs.seeded_noise(m["noise_seed"])     # CPU generator, moved to the device
    den = sampling.Denoiser({"target": BASE + "denoiser_scaling.VScalingWithEDMcNoise"})
    model = sampling.OpenAIWrapper(_unet_small())
    extra = {"image_only_indicator": torch.zeros(2, T, device=DEV), "num_video_frames": T}
    evals = [0]

    def denoiser(i, s, cc):
        evals[0] += 1
        return den(model, i, s, cc, **extra)

    out = sampler(denoiser, x.to(DEV), cond=to(c), uc=to(uc))
    torch.cuda.synchronize()
    r = _rel(out.cpu(), gold["out"])
    print(tag, "rel-l2", r)
    assert evals[0] == m["network_evals"]
    assert r <= HOST_PATH_BOUND[tag], f"{tag}: rel-L2 {r:.4f} > {HOST_PATH_BOUND[tag]}"


@pytest.mark.parametrize("name", ["EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
                                  "LinearMultistepSampler"])
def test_sampler_call_has_no_host_sync(name):
    """After a warm-up call (which uploads the guider's scale once), a whole sampler call - schedule upload, denoiser
    kernels, noise draws, history, step kernels - issues no device->host synchronisation."""
    from v3d_b200 import sampling

    T, hw = 4, 8
    sampler = getattr(sampling, name)(
        num_steps=5, discretization_config={"target": BASE + "discretizer.EDMDiscretization",
                                            "params": {"sigma_max": 80.0}},
        guider_config={"target": BASE + "guiders.LinearPredictionGuider", "params": {"max_scale": 2.5, "num_frames": T}})
    den = sampling.Denoiser({"target": BASE + "denoiser_scaling.VScalingWithEDMcNoise"})
    stub = lambda xx, t, cond: 0.9 * xx  # noqa: E731
    c = {"crossattn": torch.randn(T, 1, 8, device=DEV), "vector": torch.randn(T, 8, device=DEV)}
    uc = {k: torch.zeros_like(v) for k, v in c.items()}
    sampler(lambda i, s, cc: den(stub, i, s, cc), torch.randn(T, 4, hw, hw, device=DEV), cond=c, uc=uc)
    torch.cuda.synchronize()
    x = torch.randn(T, 4, hw, hw, device=DEV)
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = sampler(lambda i, s, cc: den(stub, i, s, cc), x, cond=c, uc=uc)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
