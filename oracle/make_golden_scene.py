"""Generate tests/golden/scene_*.pt from the REAL reference PixelNeRFEmbedder / PixelNeRF / ExtraConditioner
(sgm/modules/encoders/modules.py:1075-1187, pixelnerf.py) on seeded weights, and pin the oracle
(oracle/ref_pixelnerf.py) against them.

TEST INFRASTRUCTURE; runs only where the reference checkout is importable (oracle/reference_shim.py):
    python -m oracle.make_golden_scene

modules.py imports open_clip and kornia at module level (neither is used by these classes); they are stubbed here as
empty modules, in this script only.  Each case runs the real PixelNeRFEmbedder in one of its two input forms (the
first frame as the one source, or S source images with their own cameras).  The uniforms of RaySampler come from a
seeded tensor that replaces `torch.rand_like` for the call, so the fixture holds exactly the jitter the module must be
given.  The weights are nn.Linear's default init scaled by WEIGHT_SCALE: at scale 1 the outputs are almost entirely
bias, and zeroed source images would move them by less than a bf16 forward does.  The scene_s1 fixture also holds
(c, uc) of the real ExtraConditioner around that embedder.  The script refuses to write unless the oracle agrees with
the reference to 2e-4 of the output scale.
"""
from __future__ import annotations

import importlib
import math
import sys
import types
from pathlib import Path

import torch

ROOT = Path(__file__).resolve().parent.parent
if str(ROOT) not in sys.path:
    sys.path.insert(0, str(ROOT))

from oracle import ref_pixelnerf, reference_shim  # noqa: E402

OUT = ROOT / "tests" / "golden"
PIN_TOL = 2e-4
WEIGHT_SCALE = 3.0
MAX_FIXTURE_BYTES = 1 << 20

# tag -> (form, B, T, S, C, H, W, render, ns, std, pos_emb, seed)
CASES = {
    "scene_s1": ("frames", 1, 4, 1, 3, 24, 24, 8, 16, True, True, 41),
    "scene_s3": ("sources", 2, 3, 3, 3, 20, 28, 8, 24, True, True, 42),
}


def look_at_cams(n: int, phase: float, radius: float = 2.6) -> torch.Tensor:
    """[n, 25] rows of cameras on a circle around the box, looking at the origin (OpenGL axes: -z forward), with a
    small skew so the skew term of RayGenerator is exercised."""
    rows = []
    for i in range(n):
        a = phase + 2 * math.pi * i / max(n, 1) * 0.35
        pos = torch.tensor([radius * math.sin(a), 0.35 + 0.1 * i, radius * math.cos(a)])
        z = pos / pos.norm()
        x = torch.linalg.cross(torch.tensor([0.0, 1.0, 0.0]), z)
        x = x / x.norm()
        y = torch.linalg.cross(z, x)
        c2w = torch.eye(4)
        c2w[:3, 0], c2w[:3, 1], c2w[:3, 2], c2w[:3, 3] = x, y, z, pos
        K = torch.tensor([[1.3 + 0.02 * i, 0.015, 0.5], [0.0, 1.25, 0.47], [0.0, 0.0, 1.0]])
        rows.append(torch.cat([c2w.reshape(16), K.reshape(9)]))
    return torch.stack(rows)


def make_inputs(form, B, T, S, C, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    cams = torch.stack([look_at_cams(T, 0.3 + 0.5 * b) for b in range(B)])
    if form == "frames":
        return {"frames": torch.rand(B, T, C, H, W, generator=g) * 2 - 1, "cameras": cams}
    return {"cameras": cams, "source_index": torch.arange(S),
            "source_images": torch.rand(B, S, C, H, W, generator=g) * 2 - 1,
            "source_cameras": torch.stack([look_at_cams(S, 1.1 + 0.7 * b, 2.4) for b in range(B)])}


def _patched_rand_like(jitter):
    rand_like = torch.rand_like

    def f(t, *a, **k):
        return jitter.clone() if t.shape == jitter.shape else rand_like(t, *a, **k)
    return rand_like, f


def main() -> None:
    reference_shim.install()
    for name in ("kornia", "open_clip"):  # imported by modules.py, unused by the classes below
        sys.modules.setdefault(name, types.ModuleType(name))
    mods = importlib.import_module("sgm.modules.encoders.modules")
    for tag, (form, B, T, S, C, H, W, rs, ns, std, pe, seed) in CASES.items():
        inputs = make_inputs(form, B, T, S, C, H, W, seed)
        emb_cfg = {"target": "sgm.modules.encoders.modules.PixelNeRFEmbedder",
                   "params": {"image_encoder_config": {"target": "sgm.modules.encoders.pixelnerf.ImageEncoder"},
                              "pixelnerf_encoder_config": {
                                  "target": "sgm.modules.encoders.pixelnerf.PixelNeRF",
                                  "params": dict(num_samples_per_ray=ns, feature_dim=C, use_feats_std=std,
                                                 use_pos_emb=pe)},
                              "render_size": rs, "num_video_frames": T}}
        cond = mods.ExtraConditioner([
            {"input_key": "cond_frames", "target": "sgm.modules.encoders.modules.IdentityEncoder"},
            dict(emb_cfg, input_key="pixelnerf_input"),
            {"input_key": "clip", "target": "sgm.modules.encoders.modules.IdentityEncoder"},
        ])
        model = cond.embedders[1]
        sd = ref_pixelnerf.state_dict(model.pixelnerf_encoder.feature_aggregator[0].in_features, seed,
                                      scale=WEIGHT_SCALE)
        model.pixelnerf_encoder.load_state_dict(sd)
        jitter = torch.rand(ns, B * T, rs * rs, 1, generator=torch.Generator().manual_seed(seed + 100))
        g = torch.Generator().manual_seed(seed + 200)
        batch = {"frames": torch.zeros(B * T, 3, 8, 8), "num_video_frames": T,
                 "cond_frames": torch.randn(B, 4, rs, rs, generator=g), "clip": torch.randn(B, 1, 1024, generator=g),
                 "pixelnerf_input": inputs}
        rand_like, patched = _patched_rand_like(jitter)
        torch.rand_like = patched
        try:
            with torch.no_grad():
                rgb, fe = model(inputs)
                c, uc = cond.get_unconditional_conditioning(
                    batch, force_uc_zero_embeddings=["cond_frames", "pixelnerf_input", "clip"])
        finally:
            torch.rand_like = rand_like
        o_rgb, o_fe = ref_pixelnerf.embedder(sd, inputs, rs, jitter.reshape(ns, -1), ns, use_std=std, use_pe=pe)
        err = max(float((o_rgb - rgb).abs().max() / rgb.abs().max()), float((o_fe - fe).abs().max() / fe.abs().max()))
        if err > PIN_TOL:
            raise SystemExit(f"{tag}: oracle disagrees with the reference PixelNeRFEmbedder ({err:.3e} > {PIN_TOL})")
        fix = {"case": dict(form=form, B=B, T=T, S=S, C=C, H=H, W=W, render_size=rs, ns=ns, use_feats_std=std,
                            use_pos_emb=pe, seed=seed, weight_scale=WEIGHT_SCALE),
               "inputs": inputs, "jitter": jitter, "state_dict": sd,
               "reference_state_dict_shapes": {k: tuple(v.shape) for k, v in
                                               model.pixelnerf_encoder.state_dict().items()},
               "rgb": rgb, "feats": fe, "oracle_pin": err}
        if tag == "scene_s1":  # the conditioner around the embedder: keys, order, repeats, uc zeros
            fix["conditioner"] = {"batch": {k: v for k, v in batch.items() if k != "pixelnerf_input"},
                                  "c": c, "uc": uc, "c_keys": list(c.keys()), "uc_keys": list(uc.keys())}
        path = OUT / f"{tag}.pt"
        torch.save(fix, path)
        size = path.stat().st_size
        if size > MAX_FIXTURE_BYTES:
            path.unlink()
            raise SystemExit(f"{tag}: fixture is {size} bytes (> {MAX_FIXTURE_BYTES})")
        print(f"{tag}: oracle vs reference {err:.2e}, {size} bytes")


if __name__ == "__main__":
    main()
