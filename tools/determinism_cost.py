#!/usr/bin/env python
"""Cost of the deterministic mode (V3D_DETERMINISTIC=1): one V3D_512 image, and the GroupNorm family alone.

    python tools/determinism_cost.py [--repeats 3]

Image: the V3D_512 engine (T = 18 views, 512 x 512, 25 Euler-EDM steps with CFG, decode included; per-name seeded
weights as in tools/sampler_timing.py) times `DiffusionEngine.sample_views` with CUDA events, the default and the
deterministic mode alternated in one process after one warm-up call each (each mode has its own captured graphs).
Norms: the GroupNorm shapes of tools/microbench.py, each timed the way the modules launch it in either mode (one
launch for the 2-D norms, the two-kernel form for the 3-D norms; the same rule in both modes).  One JSON line per
measurement, with the GPU name, power limit and SM clock read in the same run.  Needs a CUDA device.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
from pathlib import Path

ROOT = Path(__file__).resolve().parent.parent
sys.path.insert(0, str(ROOT))
sys.path.insert(0, str(ROOT / "tools"))

NORM_SHAPES = [("gn2d L0 320", 36, 4096, 4096, 320), ("gn3d L0 320", 2, 18 * 4096, 4096, 320),
               ("gn2d L0 640", 36, 4096, 4096, 640), ("gn2d L1 640", 36, 1024, 1024, 640),
               ("gn3d L1 640", 2, 18 * 1024, 1024, 640), ("gn2d L2 1280", 36, 256, 256, 1280),
               ("gn2d L3 1280", 36, 64, 64, 1280), ("gn3d L3 1280", 2, 18 * 64, 64, 1280),
               ("gn2d dec512 128", 18, 262144, 262144, 128), ("gn3d dec512 128", 1, 18 * 262144, 262144, 128)]


def _events_ms(torch, fn, iters: int) -> float:
    fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(iters):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / iters


def norms(torch, info: dict) -> None:
    from v3d_b200 import ops

    dev = torch.device("cuda", 0)
    for name, ns, rows, hw, c in NORM_SHAPES:
        x = (torch.randn(ns * rows, c, device=dev) + 0.3).to(torch.bfloat16)
        y = torch.empty_like(x)
        g, b = torch.ones(c, device=dev), torch.zeros(c, device=dev)
        one_launch = 8 <= ns <= 256 and x.numel() * 2 <= 300e6          # the modules' selection (KernelModule._gn)
        st = torch.zeros(ns, 32, 2, device=dev, dtype=torch.float64)
        ws = ops.groupnorm_workspace(dev)
        nblk = ops.groupnorm_det_blocks(rows, hw)
        part = torch.empty(ns, nblk, 32, 2, device=dev)
        dws = ops.groupnorm_det_workspace(dev, ops.groupnorm_det_workspace_bytes(rows, hw, ns))
        if one_launch:
            default = lambda: ops.groupnorm(x, y, g, b, rows, ns, c, 1e-5, True, ws)
            det = lambda: ops.groupnorm_det(x, y, g, b, rows, hw, ns, c, 1e-5, True, dws)
        else:
            def default():
                ops.groupnorm_stats(x, st, rows, ns, c)
                ops.groupnorm_apply(x, y, st, g, b, rows, ns, c, 1e-5, True)

            def det():
                ops.groupnorm_partials(x, part, rows, hw, ns, c)
                ops.groupnorm_fold_apply(x, y, part, g, b, rows, ns, c, 1e-5, True, nblk)
        ms = {"default": [], "deterministic": []}
        for _ in range(3):                                              # alternated
            ms["default"].append(_events_ms(torch, default, 20))
            ms["deterministic"].append(_events_ms(torch, det, 20))
        d, e = min(ms["default"]), min(ms["deterministic"])
        print(json.dumps({"kind": "norm", "shape": name, "form": "one launch" if one_launch else "pair",
                          "default_ms": round(d, 4), "deterministic_ms": round(e, 4),
                          "overhead_pct": round(100 * (e / d - 1), 1), **info}), flush=True)


def image(torch, repeats: int, info: dict) -> None:
    from bench import load_synth_
    from v3d_b200 import engine

    dev = torch.device("cuda", 0)
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

    def run_mode(det: bool):
        if det:
            os.environ["V3D_DETERMINISTIC"] = "1"
        else:
            os.environ.pop("V3D_DETERMINISTIC", None)
        return _events_ms(torch, lambda: eng.sample_views(x0.clone(), c, uc, num_frames=T, decoding_t=T), 1)

    run_mode(False)                                                     # warm-up (eager pass, then graph capture)
    run_mode(True)
    ms = {"default": [], "deterministic": []}
    for _ in range(repeats):
        ms["default"].append(run_mode(False))
        ms["deterministic"].append(run_mode(True))
    os.environ.pop("V3D_DETERMINISTIC", None)
    d, e = sum(ms["default"]) / repeats, sum(ms["deterministic"]) / repeats
    print(json.dumps({"kind": "image", "frames": T, "resolution": 8 * L, "steps": 25,
                      "default_ms": [round(v, 1) for v in ms["default"]],
                      "deterministic_ms": [round(v, 1) for v in ms["deterministic"]],
                      "overhead_pct": round(100 * (e / d - 1), 2), **info}), flush=True)


def main() -> None:
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    ap.add_argument("--repeats", type=int, default=3, help="timed images per mode (alternated)")
    ap.add_argument("--skip-image", action="store_true")
    args = ap.parse_args()

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("determinism_cost.py needs a CUDA device")
    from sampler_timing import gpu_info

    torch.cuda.set_device(0)
    norms(torch, gpu_info(0))
    if not args.skip_image:
        image(torch, args.repeats, gpu_info(0))
    print(json.dumps({"kind": "clock_after", **gpu_info(0)}), flush=True)


if __name__ == "__main__":
    main()
