"""Generate tests/golden/{unet_small_t40,unet_full_t48_16,edm_small_t40}.pt: the REAL reference VideoUNet and Euler-EDM
sampler on videos of more than 32 view-frames, and pin the oracle (oracle/ref_unet.py, oracle/ref_sampling.py) against
them.

TEST INFRASTRUCTURE; runs only where the reference checkout is importable (oracle/reference_shim.py):
    python tools/make_golden_longt.py                  # all three fixtures
    python tools/make_golden_longt.py unet_small_t40

Inputs come from `synth.synth_inputs` and weights from `synth.synth_state_dict`, like the fixtures of
oracle/make_golden.py, so the tests regenerate them from the seeds in tests/golden/LONGT.json (MANIFEST.json is left as
it is).  T = 40 is a multiple of neither 16 nor 32: the temporal attention's last 16-query tile is half empty and its
last 8 keys are masked.  The UNet fixtures hold the reference's fp32 output and six block outputs for the samples
{0 (uc half), T (c half)}, every 8th channel, fp16; the EDM fixture holds the sample after 3 Euler steps under
LinearPredictionGuider(num_frames=40).  Only the reference's outputs are stored.
"""
from __future__ import annotations

import json
import sys
import time
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import synth  # noqa: E402

OUT = ROOT / "tests" / "golden"
PIN_TOL = 2e-4
MAX_FIXTURE_BYTES = 1 << 20
TAPS = ["input_blocks.1.0", "input_blocks.1.1", "input_blocks.3.0", "middle_block.1", "output_blocks.2.1",
        "output_blocks.11.1"]

# tag -> (model_channels, T, latent, weight seed, sigma)
UNET_CASES = {
    "unet_small_t40": (64, 40, 16, 5, 40.0),
    "unet_full_t48_16": (320, 48, 16, 3, 3.0),
}
# tag -> (UNet fixture whose network it samples with, Euler steps, min / max guidance scale)
EDM_CASES = {"edm_small_t40": ("unet_small_t40", 3, 1.5, 3.5)}


def unet_inputs(T: int, hw: int, sigma: float):
    """One CFG-batched network input, uc half first: (xin [2T,8,h,w], timesteps [2T], context [2T,1,ctx], y [2T,768])."""
    x, c, uc = synth.synth_inputs(T, hw)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    ctx = torch.cat([uc["crossattn"], c["crossattn"]])
    y = torch.cat([uc["vector"], c["vector"]])
    ts = torch.full((2 * T,), 0.25 * torch.log(torch.tensor(sigma)).item())
    return xin, ts, ctx, y


def _pin(name: str, ref: torch.Tensor, ora: torch.Tensor) -> float:
    err = ((ref - ora).abs().max() / ref.abs().max().clamp_min(1e-6)).item()
    print(f"  pin {name}: max|ref-oracle|/max|ref| = {err:.3e}", flush=True)
    if not err <= PIN_TOL:
        raise SystemExit(f"oracle does not reproduce the reference on {name}: {err}")
    return err


def _save(tag: str, blob: dict) -> int:
    torch.save(blob, OUT / f"{tag}.pt")
    size = (OUT / f"{tag}.pt").stat().st_size
    if size > MAX_FIXTURE_BYTES:
        raise SystemExit(f"{tag}: {size} bytes, over {MAX_FIXTURE_BYTES}")
    return size


def _reference_net(ns, mc: int, wseed: int):
    from oracle import ref_unet, reference_shim

    net = ns.video_model.VideoUNet(**dict(reference_shim.V3D_UNET_KW, model_channels=mc)).eval()
    spec = ref_unet.UNetSpec(model_channels=mc)
    sd = synth.synth_state_dict(ref_unet.unet_param_shapes(spec), seed=wseed)
    net.load_state_dict(sd)
    return net, sd, spec


def _unet_case(ns, tag: str, manifest: dict) -> None:
    from oracle import ref_unet

    mc, T, hw, wseed, sigma = UNET_CASES[tag]
    net, sd, spec = _reference_net(ns, mc, wseed)
    xin, ts, ctx, y = unet_inputs(T, hw, sigma)
    ind = torch.zeros(2, T)
    mods = dict(net.named_modules())
    taps_ref = {}
    hooks = [mods[w].register_forward_hook(lambda m, i, o, w=w: taps_ref.__setitem__(w, o.detach().clone()))
             for w in TAPS]
    with torch.no_grad():
        t0 = time.time()
        ref = net(xin, ts, ctx, y, None, T, ind)
        t_ref = time.time() - t0
        taps_or = {}
        ora = ref_unet.unet_forward(sd, spec, xin, ts, ctx, y, T, ind, taps=taps_or)
    for h in hooks:
        h.remove()
    err = _pin(tag, ref, ora)
    for w in TAPS:
        _pin(f"{tag}:{w}", taps_ref[w], taps_or[w])
    blob = {"out": ref.contiguous(), "timesteps": ts}
    for w in TAPS:
        blob["tap:" + w] = taps_ref[w][[0, T]][:, ::8].half().contiguous()
    size = _save(tag, blob)
    manifest[tag] = dict(kind="unet_forward", model_channels=mc, T=T, latent_hw=hw, weight_seed=wseed, input_seed=23,
                         sigma=sigma, pin_err=err, ref_cpu_seconds=round(t_ref, 2), out_std=ref.std().item(),
                         tap_stride=1)
    print(f"  {tag}: {size} bytes, reference {t_ref:.1f} s", flush=True)


def _edm_case(ns, tag: str, manifest: dict) -> None:
    from oracle import ref_sampling, ref_unet

    unet_tag, steps, smin, smax = EDM_CASES[tag]
    mc, T, hw, wseed, _ = UNET_CASES[unet_tag]
    net, sd, spec = _reference_net(ns, mc, wseed)
    x, c, uc = synth.synth_inputs(T, hw)
    sampler = ns.sampling.EulerEDMSampler(
        num_steps=steps,
        discretization_config={"target": "sgm.modules.diffusionmodules.discretizer.EDMDiscretization",
                               "params": {"sigma_max": 700.0}},
        guider_config={"target": "sgm.modules.diffusionmodules.guiders.LinearPredictionGuider",
                       "params": {"max_scale": smax, "min_scale": smin, "num_frames": T}},
        device="cpu")
    den = ns.denoiser.Denoiser({"target": "sgm.modules.diffusionmodules.denoiser_scaling.VScalingWithEDMcNoise"})
    wrapped = ns.wrappers.OpenAIWrapper(net)
    extra = {"image_only_indicator": torch.zeros(2, T), "num_video_frames": T}
    with torch.no_grad():
        ref = sampler(lambda i, s, cc: den(wrapped, i, s, cc, **extra), x.clone(), cond=c, uc=uc)
        ora = ref_sampling.euler_edm_sample(
            lambda i, s, cc: ref_sampling.denoiser(
                lambda xx, tt, cond, **kw: ref_unet.openai_wrapper(sd, spec, xx, tt, cond, **kw), i, s, cc, **extra),
            x.clone(), c, uc, steps, ref_sampling.guider_scale(smin, smax, T), T)
    err = _pin(tag, ref, ora)
    size = _save(tag, {"out": ref.contiguous()})
    manifest[tag] = dict(kind="edm_sample", unet=unet_tag, T=T, latent_hw=hw, num_steps=steps, min_scale=smin,
                         max_scale=smax, sigma_max=700.0, pin_err=err, out_std=ref.std().item())
    print(f"  {tag}: {size} bytes", flush=True)


def main(argv) -> None:
    from oracle import reference_shim

    ns = reference_shim.load()
    torch.set_num_threads(8)
    mpath = OUT / "LONGT.json"
    manifest = json.loads(mpath.read_text()) if mpath.exists() else {}
    for tag in UNET_CASES:
        if not argv or tag in argv:
            _unet_case(ns, tag, manifest)
    for tag in EDM_CASES:
        if not argv or tag in argv:
            _edm_case(ns, tag, manifest)
    mpath.write_text(json.dumps(manifest, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main(sys.argv[1:])
