#!/usr/bin/env python
"""Wall time of one V3D_512 image per sampler and step count.

    python tools/sampler_timing.py [--steps 10 15 25] [--samplers ...] [--repeats 2]

Builds the V3D_512 engine once (T = 18 views, 512 x 512, latent 4 x 64 x 64, CFG 3.5; the per-name seeded weights of
the parity fixtures) and, for each sampler and step count, times `DiffusionEngine.sample_views` (sampler loop with
CFG + first-stage decode) with CUDA events after one warm-up call.  One JSON line per case: sampler, steps, network
evaluations, ms per image, view-frames/s, plus the GPU name, power limit and SM clock read in the same run.  Needs a
CUDA device; there is no CPU fallback.
"""
from __future__ import annotations

import argparse
import json
import subprocess
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))

SAMPLERS = ["EulerEDMSampler", "EulerAncestralSampler", "DPMPP2SAncestralSampler", "DPMPP2MSampler",
            "LinearMultistepSampler"]


def gpu_info(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        line = subprocess.run(["nvidia-smi", f"--id={index}", f"--query-gpu={q}", "--format=csv,noheader,nounits"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, sm, sm_max = [f.strip() for f in line.split(",")]
        return {"gpu": name, "power_limit_w": float(power), "sm_clock_mhz": float(sm), "sm_clock_max_mhz": float(sm_max)}
    except Exception as e:  # noqa: BLE001 - report what could not be read instead of failing the measurement
        import torch

        return {"gpu": torch.cuda.get_device_name(index), "power_limit_w": None, "sm_clock_mhz": None,
                "nvidia_smi_error": str(e)}


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--steps", type=int, nargs="+", default=[10, 15, 25])
    ap.add_argument("--samplers", nargs="+", default=SAMPLERS, choices=SAMPLERS)
    ap.add_argument("--repeats", type=int, default=2, help="timed calls per case (the mean is reported)")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("sampler_timing.py needs a CUDA device")
    from bench import load_synth_
    from v3d_b200 import engine
    from v3d_b200.sampling import get_obj_from_str

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    T, L = 18, 64
    cfg = engine.v3d_512_config(num_frames=T)
    with torch.device("meta"):
        eng = engine.DiffusionEngine(**cfg)
    manifest = json.loads((ROOT / "tests" / "golden" / "MANIFEST.json").read_text())
    load_synth_(eng.model.diffusion_model, dev, manifest["unet_v3d512"]["weight_seed"])
    load_synth_(eng.first_stage_model.decoder, dev, manifest["decoder_v3d512"]["weight_seed"])
    eng.eval()
    g = torch.Generator().manual_seed(23)
    x0 = torch.randn(T, 4, L, L, generator=g).to(dev)
    c = {"crossattn": torch.randn(1, 1, 1024, generator=g).repeat(T, 1, 1).to(dev),
         "concat": torch.randn(1, 4, L, L, generator=g).repeat(T, 1, 1, 1).to(dev),
         "vector": torch.randn(T, 768, generator=g).to(dev)}
    uc = {"crossattn": torch.zeros_like(c["crossattn"]), "concat": torch.zeros_like(c["concat"]),
          "vector": c["vector"].clone()}
    base = cfg["sampler_config"]["params"]
    for name in args.samplers:
        for steps in args.steps:
            eng.sampler = get_obj_from_str("v3d_b200.sampling." + name)(**dict(base, num_steps=steps))
            evals = [0]
            denoise = eng.denoiser.forward

            def counting(*a, **k):
                evals[0] += 1
                return denoise(*a, **k)

            eng.denoiser.forward = counting
            try:
                eng.sample_views(x0.clone(), c, uc, num_frames=T, decoding_t=T)            # warm-up
                evals[0] = 0
                torch.cuda.synchronize()
                start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                start.record()
                for _ in range(args.repeats):
                    out = eng.sample_views(x0.clone(), c, uc, num_frames=T, decoding_t=T)
                end.record()
                torch.cuda.synchronize()
            finally:
                del eng.denoiser.forward
            assert torch.isfinite(out).all(), (name, steps)
            ms = start.elapsed_time(end) / args.repeats
            print(json.dumps({"sampler": name, "steps": steps, "network_evals": evals[0] // args.repeats,
                              "ms_per_image": round(ms, 1), "view_frames_per_s": round(T / (ms / 1e3), 3),
                              "frames": T, "resolution": 8 * L, **gpu_info(0)}), flush=True)


if __name__ == "__main__":
    main()
