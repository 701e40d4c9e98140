"""Generate tests/golden/unet_*_ctx*.pt: the REAL reference VideoUNet over cross-attention contexts of more than one
token, and pin the oracle (oracle/ref_unet.py) against them.

TEST INFRASTRUCTURE; runs only where the reference checkout is importable (oracle/reference_shim.py):
    python tools/make_golden_ctx.py            # all three fixtures
    python tools/make_golden_ctx.py unet_small_ctx3

x, concat and vector come from `synth.synth_inputs` like the single-token fixtures of oracle/make_golden.py; the
c half's context is drawn per frame and per token (`ctx_inputs`, seed CTX_SEED) and the uc half's is zero, as the
sampler receives it, so a schedule that attends to another frame's keys, to the wrong frame 0 in the temporal attn2,
or to the other half's context changes the output.  Each fixture holds the reference's fp32 output and, like the single-token fixtures, six
block outputs for the samples {0 (uc half), T (c half)}, every 8th channel, fp16.  The tests regenerate the inputs
with `ctx_inputs`; their index is tests/golden/CTX.json (MANIFEST.json is left as it is).
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
CTX_SEED = 37
MAX_FIXTURE_BYTES = 1 << 20
TAPS = ["input_blocks.1.0", "input_blocks.1.1", "input_blocks.3.0", "middle_block.1", "output_blocks.2.1",
        "output_blocks.11.1"]

# tag -> (model_channels, T, latent, context tokens, weight seed, sigma)
CASES = {
    "unet_small_ctx3": (64, 4, 32, 3, 1, 3.0),
    "unet_small_t18_ctx77": (64, 18, 16, 77, 2, 40.0),
    "unet_full_t18_16_ctx4": (320, 18, 16, 4, 3, 3.0),
}


def ctx_inputs(T: int, hw: int, M: int, sigma: float, ctx_dim: int = 1024):
    """One CFG-batched network input with an M-token context: (xin [2T,8,h,w], timesteps [2T], context [2T,M,ctx],
    y [2T,768]), uc half first.  Every frame and token of the c half's context has its own N(0, 1) draw; the uc half's
    context is zero (the unconditional embedding V3D_512.py:255-258 forces)."""
    x, c, uc = synth.synth_inputs(T, hw)
    xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
    g = torch.Generator().manual_seed(CTX_SEED)
    ctx = torch.cat([torch.zeros(T, M, ctx_dim), torch.randn(T, M, ctx_dim, generator=g)])
    y = torch.cat([uc["vector"], c["vector"]])
    ts = torch.full((2 * T,), 0.25 * torch.log(torch.tensor(sigma)).item())
    return xin, ts, ctx, y


def _pin(name: str, ref: torch.Tensor, ora: torch.Tensor) -> float:
    err = ((ref - ora).abs().max() / ref.abs().max().clamp_min(1e-6)).item()
    print(f"  pin {name}: max|ref-oracle|/max|ref| = {err:.3e}")
    if not err <= PIN_TOL:
        raise SystemExit(f"oracle does not reproduce the reference on {name}: {err}")
    return err


def main(argv) -> None:
    from oracle import ref_unet, reference_shim

    ns = reference_shim.load()
    torch.set_num_threads(8)
    mpath = OUT / "CTX.json"
    manifest = json.loads(mpath.read_text()) if mpath.exists() else {}
    for tag, (mc, T, hw, M, wseed, sigma) in CASES.items():
        if argv and tag not in argv:
            continue
        net = ns.video_model.VideoUNet(**dict(reference_shim.V3D_UNET_KW, model_channels=mc)).eval()
        spec = ref_unet.UNetSpec(model_channels=mc)
        sd = synth.synth_state_dict(ref_unet.unet_param_shapes(spec), seed=wseed)
        net.load_state_dict(sd)
        xin, ts, ctx, y = ctx_inputs(T, hw, M, sigma)
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
        torch.save(blob, OUT / f"{tag}.pt")
        size = (OUT / f"{tag}.pt").stat().st_size
        if size > MAX_FIXTURE_BYTES:
            raise SystemExit(f"{tag}: {size} bytes, over {MAX_FIXTURE_BYTES}")
        manifest[tag] = dict(kind="unet_forward_ctx", model_channels=mc, T=T, latent_hw=hw, context_tokens=M,
                             weight_seed=wseed, input_seed=23, ctx_seed=CTX_SEED, sigma=sigma, pin_err=err,
                             ref_cpu_seconds=round(t_ref, 2), out_std=ref.std().item(), tap_stride=1)
        print(f"  {tag}: {size} bytes, reference {t_ref:.1f} s")
    mpath.write_text(json.dumps(manifest, indent=1, sort_keys=True) + "\n")


if __name__ == "__main__":
    main(sys.argv[1:])
