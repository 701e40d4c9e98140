"""Generate tests/golden/unet_*_perframe.pt from the REAL reference VideoUNet on per-frame conditioning, and pin the
oracle (oracle/ref_unet.py) against them.

TEST INFRASTRUCTURE; runs only where the reference checkout is importable (oracle/reference_shim.py):
    python -m oracle.make_golden_perframe

The inputs come from `synth.synth_inputs_perframe`: every frame and both CFG halves have their own crossattn, concat
and vector, and every sample its own timestep.  A schedule that reads another frame's bias row, another sample's
time embedding or the wrong frame's temporal context therefore changes the output of that frame, which the
frame-invariant fixtures of make_golden.py cannot show.  Each fixture holds the full fp32 output and every block's
output (conv_in, res, attn, down, up) for all 2T samples, in fp16, every 4th channel and every `tap_stride`-th pixel
(rows and columns from 0, so the border pixel (0, 0) of every image is kept).  The strides keep each file under
1 MB like the other fixtures; the taps at full resolution are checked in fp64 on the GPU by
tests/test_unet_blocks_fp64_gpu.py, which needs no fixture.
Only these fixtures and their index tests/golden/PERFRAME.json are written; MANIFEST.json is left as it is.
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

from oracle import ref_unet, reference_shim, synth  # noqa: E402

OUT = ROOT / "tests" / "golden"
PIN_TOL, TAP_PIN_TOL = 2e-4, 2e-3
INPUT_SEED = 29
TAP_KINDS = ("conv_in", "res", "attn", "down", "up")

MAX_FIXTURE_BYTES = 1 << 20

# tag -> (model_channels, T, latent, weight seed, tap pixel stride)
CASES = {
    "unet_small_t18_perframe": (64, 18, 16, 2, 4),
    "unet_full_t5_perframe": (320, 5, 32, 3, 8),
}


def perframe_inputs(T: int, hw: int):
    """The network input of one CFG-batched evaluation: (xin [2T,8,h,w], timesteps [2T], context [2T,1,1024],
    y [2T,768]), uc half first."""
    x, c, uc, ts = synth.synth_inputs_perframe(T, hw, seed=INPUT_SEED)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    return xin, ts, torch.cat([uc["crossattn"], c["crossattn"]]), torch.cat([uc["vector"], c["vector"]])


def tap_names(spec: ref_unet.UNetSpec):
    return [name for name, kind, _ in spec.blocks if kind in TAP_KINDS]


def _pin(name: str, ref: torch.Tensor, ora: torch.Tensor, tol: float) -> float:
    err = ((ref - ora).abs().max() / ref.abs().max().clamp_min(1e-6)).item()
    if not err <= tol:
        raise SystemExit(f"oracle does not reproduce the reference on {name}: {err}")
    return err


def main() -> None:
    ns = reference_shim.load()
    torch.set_num_threads(8)
    index = {}
    for tag, (mc, T, hw, wseed, stride) in CASES.items():
        net = ns.video_model.VideoUNet(**dict(reference_shim.V3D_UNET_KW, model_channels=mc)).eval()
        spec = ref_unet.UNetSpec(model_channels=mc)
        sd = synth.synth_state_dict(ref_unet.unet_param_shapes(spec), seed=wseed)
        net.load_state_dict(sd)
        xin, ts, ctx, y = perframe_inputs(T, hw)
        ind = torch.zeros(2, T)
        mods = dict(net.named_modules())
        taps_ref = {}
        hooks = [mods[w].register_forward_hook(lambda m, i, o, w=w: taps_ref.__setitem__(w, o.detach().clone()))
                 for w in tap_names(spec)]
        with torch.no_grad():
            t0 = time.time()
            ref = net(xin, ts, ctx, y, None, T, ind)
            t_ref = time.time() - t0
            taps_or = {}
            ora = ref_unet.unet_forward(sd, spec, xin, ts, ctx, y, T, ind, taps=taps_or)
        for h in hooks:
            h.remove()
        err = _pin(tag, ref, ora, PIN_TOL)
        tap_err = max(_pin(f"{tag}:{w}", taps_ref[w], taps_or[w], TAP_PIN_TOL) for w in taps_ref)
        print(f"  pin {tag}: output {err:.3e}, worst tap {tap_err:.3e} ({len(taps_ref)} taps), reference {t_ref:.1f} s")
        blob = {"out": ref.contiguous(), "timesteps": ts, "tap_stride": stride}
        for w, v in taps_ref.items():
            blob["tap:" + w] = v[:, ::4, ::stride, ::stride].half().contiguous()
        torch.save(blob, OUT / f"{tag}.pt")
        size = (OUT / f"{tag}.pt").stat().st_size
        if size > MAX_FIXTURE_BYTES:
            raise SystemExit(f"{tag}: {size} bytes, over {MAX_FIXTURE_BYTES}: raise its tap stride")
        index[tag] = dict(kind="unet_forward_perframe", model_channels=mc, T=T, latent_hw=hw, weight_seed=wseed,
                          input_seed=INPUT_SEED, tap_channel_stride=4, tap_stride=stride, pin_err=err,
                          tap_pin_err=tap_err, ref_cpu_seconds=round(t_ref, 2), out_std=ref.std().item())
    (OUT / "PERFRAME.json").write_text(json.dumps(index, indent=1, sort_keys=True) + "\n")
    print("wrote", sorted(CASES))


if __name__ == "__main__":
    main()
