"""Generate tests/golden/edm_small_{euler_ancestral,dpmpp2s,dpmpp2m,lms}.pt from the REAL reference samplers and pin
oracle/ref_samplers.py against them.

TEST INFRASTRUCTURE; runs only where the reference checkout is importable (oracle/reference_shim.py):
    python oracle/make_golden_samplers.py

The network is the reference VideoUNet with the `unet_small` weights (oracle/synth.py, seed and width from
MANIFEST.json), T = 4, latent 32 x 32, LinearPredictionGuider 1.5 -> 3.5, sigma_max 700, run on CPU fp32.  The
ancestral samplers' `noise_sampler` is replaced by draws from a seeded CPU generator (`noise_seed`), so the tests
regenerate the same noise.  Only these four fixtures and their index tests/golden/SAMPLERS.json (sampler, steps, eta,
s_noise, order, noise seed, network evaluations, pin error, output std) are written; MANIFEST.json and the fixtures of
make_golden.py are only read.
"""
from __future__ import annotations

import json
import sys
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import ref_samplers, ref_sampling, ref_unet, reference_shim, synth  # noqa: E402

OUT = ROOT / "tests" / "golden"
PIN_TOL = 2e-4
T, HW, MIN_SCALE, MAX_SCALE, SIGMA_MAX = 4, 32, 1.5, 3.5, 700.0

# tag -> (reference class, steps, constructor kwargs, noise seed or None)
CASES = {
    "edm_small_euler_ancestral": ("EulerAncestralSampler", 3, {"eta": 1.0, "s_noise": 1.0}, 101),
    "edm_small_dpmpp2s": ("DPMPP2SAncestralSampler", 3, {"eta": 1.0, "s_noise": 1.0}, 102),
    "edm_small_dpmpp2m": ("DPMPP2MSampler", 3, {}, None),
    "edm_small_lms": ("LinearMultistepSampler", 5, {"order": 4}, None),
}


def seeded_noise(seed: int):
    """The noise source of the fixtures: standard normal draws from one CPU generator, in call order."""
    g = torch.Generator().manual_seed(seed)
    return lambda x: torch.randn(x.shape, generator=g, dtype=torch.float32).to(x.device)


def _pin(name: str, ref: torch.Tensor, ora: torch.Tensor) -> float:
    scale = ref.abs().max().clamp_min(1e-6)
    err = ((ref - ora).abs().max() / scale).item()
    print(f"  pin {name}: max|ref-oracle|/max|ref| = {err:.3e}")
    if not err <= PIN_TOL:
        raise SystemExit(f"oracle does not reproduce the reference on {name}: {err}")
    return err


def main() -> None:
    ns = reference_shim.load()
    torch.set_num_threads(8)
    mu = json.loads((OUT / "MANIFEST.json").read_text())["unet_small"]
    index = {}
    kw = dict(reference_shim.V3D_UNET_KW, model_channels=mu["model_channels"])
    net = ns.video_model.VideoUNet(**kw).eval()
    spec = ref_unet.UNetSpec(model_channels=mu["model_channels"])
    sd = synth.synth_state_dict(ref_unet.unet_param_shapes(spec), seed=mu["weight_seed"])
    net.load_state_dict(sd)
    wrapped = ns.wrappers.OpenAIWrapper(net)
    den = ns.denoiser.Denoiser({"target": "sgm.modules.diffusionmodules.denoiser_scaling.VScalingWithEDMcNoise"})
    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    x, c, uc = synth.synth_inputs(T, HW)
    scale = ref_sampling.guider_scale(MIN_SCALE, MAX_SCALE, T)

    def oracle_net(i, s, cc):
        return ref_sampling.denoiser(lambda xx, tt, cond, **k: ref_unet.openai_wrapper(sd, spec, xx, tt, cond, **k),
                                     i, s, cc, **extra)

    for tag, (cls, steps, params, seed) in CASES.items():
        sampler = getattr(ns.sampling, cls)(
            num_steps=steps,
            discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.EDMDiscretization",
                                   "params": {"sigma_max": SIGMA_MAX}},
            guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                           "params": {"max_scale": MAX_SCALE, "min_scale": MIN_SCALE, "num_frames": T}},
            device="cpu", **params)
        evals = [0]

        def ref_net(i, s, cc):
            evals[0] += 1
            return den(wrapped, i, s, cc, **extra)

        common = (x.clone(), c, uc, steps, scale, T)
        with torch.no_grad():
            if seed is not None:
                sampler.noise_sampler = seeded_noise(seed)
                ref = sampler(ref_net, x.clone(), cond=c, uc=uc)
                fn = {"EulerAncestralSampler": ref_samplers.euler_ancestral_sample,
                      "DPMPP2SAncestralSampler": ref_samplers.dpmpp2s_ancestral_sample}[cls]
                ora = fn(oracle_net, *common, noise_fn=seeded_noise(seed), **params)
            elif cls == "DPMPP2MSampler":
                ref = sampler(ref_net, x.clone(), cond=c, uc=uc)
                ora = ref_samplers.dpmpp2m_sample(oracle_net, *common)
            else:
                ref = sampler(ref_net, x.clone(), cond=c, uc=uc)
                ora = ref_samplers.lms_sample(oracle_net, *common, order=params["order"])
        err = _pin(tag, ref, ora)
        torch.save({"out": ref}, OUT / f"{tag}.pt")
        index[tag] = dict(sorted(dict(kind="edm_sample_variant", sampler=cls, guider="linear", T=T, latent_hw=HW,
                             num_steps=steps, min_scale=MIN_SCALE, max_scale=MAX_SCALE, sigma_max=SIGMA_MAX,
                             eta=params.get("eta"), s_noise=params.get("s_noise"), order=params.get("order"),
                             noise_seed=seed, network_evals=evals[0], pin_err=err, out_std=ref.std().item()).items()))
    (OUT / "SAMPLERS.json").write_text(json.dumps(index, indent=1, sort_keys=True) + "\n")
    print("wrote", sorted(CASES))


if __name__ == "__main__":
    main()
