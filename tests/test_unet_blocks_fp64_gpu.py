"""Every UNet block on its own input, against the oracle in fp64, frame by frame.

The parity tests judge a whole forward with one rel-L2 of at most 3e-2, of which the bf16 path alone spends about
1.6e-2.  Behind that margin a schedule mistake confined to one frame of a CFG batch of 36 (a wrong bias row, time
embedding, position id or temporal context) and a precision regression inside one block (an intermediate stored in
bf16 instead of fp32) both pass.  This file takes the forward apart instead:

  * One forward of the drop-in VideoUNet with every block tapped.  A tap is the block's bf16 output widened to fp32,
    so it equals the next block's input bit for bit.
  * For every block, its input is rebuilt from the taps (the previous tap, or the previous tap concatenated with the
    saved skip tap), the oracle's block (oracle/ref_unet.py) runs on it in fp64 with the same weights, with the
    embeddings and context computed in fp64 from the same timesteps / y / context, and the result is compared with
    the block's tap.  The error the earlier blocks accumulated is thereby removed: each block answers for itself.
  * For every part p of a partition the error must satisfy

        ||err_p|| <= c_kind * ||upd_p|| + ||rnd_p||

    upd = ref - x_in when the block keeps its shape (the residual path would otherwise hide a wrong update), ref
    otherwise.  rnd = bf16(ref) - ref is the rounding of the exact output to the bf16 the block stores (0 for `out`,
    whose `out.2` conv stores fp32).  It stands where a worst-case 2^-8 ||ref|| could: on the stand-in leg below that
    term alone covers every block with room to spare (ratios 0.25-0.5 at c = 0), so a block whose own error doubled
    would still pass; the realised rounding leaves c_kind to bound what the block adds.
  * Budget: the whole block satisfies the bound (ratio <= 1).  Locality: every part's ratio is at most
    LOCALITY_FACTOR = 2 x the whole block's ratio + LOCALITY_FLOOR = 0.1 (the floor absorbs the statistical spread of
    small parts).  Partitions: each of the 2T samples, each frame position t, each 32-channel group, each 64-channel
    head (attention blocks), and the one-pixel border ring vs the interior (h, w >= 8).  A mistake confined to one
    frame is a small share of the whole but all of its part.

c_kind.  The stand-in leg (`standin`, no GPU) runs the same code with tests/emu_ops.py in place of the kernels: they
compute in fp64 and round to bf16 wherever the kernels store bf16 (weights included), so they make the rounding
errors the schedule implies and nothing else.  Its measured c = (||err|| - ||rnd||)+ / ||upd||, largest over the
blocks of a kind on both geometries at width 64 (STANDIN_C), times STANDIN_MARGIN = 1.25 is C_KIND.  The margin is
small on purpose: one more bf16 rounding of a block's main intermediate multiplies its c by about sqrt(2).  On one
H100 80GB HBM3 (700 W) the kernels' c matched the stand-ins' within 3 % for every kind (attention included: the
kernels' bf16 rounding of the softmax probabilities did not show at this scale); largest budget ratios over the
three GPU legs: conv_in 0.93, res 0.93, res_skip 0.89, attn 0.85, down 0.92, up 0.94, out 0.89; largest part ratio
1.39 (`out`, one sample, whole 0.89).  The fp64 oracle pass at the benchmark shape took 6.3 s and peaked at 23.7 GiB.

Legs: `standin` (CPU, unmarked) at width 64 on the two per-frame geometries; `gpu` on the inputs and weights of both
per-frame fixtures and at the benchmark shape itself (width 320, T = 18, CFG batch 36, latent 64^2, synthetic
weights, per-frame inputs), where the oracle's SDPA runs a few (sample, head) pairs per call
(ref_unet.SDPA_CHUNK_BYTES).  Each block prints
    BLOCK <name> kind=<k> ratio=<whole> worst=<partition>:<index>:<ratio> c=<measured c>

The last part of the file is end to end and per sample: the oracle on the CPU against the real reference's per-frame
fixtures (tests/golden/unet_*_perframe.pt, oracle/make_golden_perframe.py), and on the GPU the forward against them,
every one of the 2T samples on its own.
"""
import json
import sys
import time
from pathlib import Path

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, str(Path(__file__).resolve().parent))

from framewise import LOCALITY_FACTOR, LOCALITY_FLOOR, assert_per_sample, groups, judge, ring_interior  # noqa: E402

GOLD = Path(__file__).resolve().parent / "golden"
PERFRAME = json.loads((GOLD / "PERFRAME.json").read_text())

UNET_KW = dict(adm_in_channels=768, num_classes="sequential", use_checkpoint=True, in_channels=8, out_channels=4,
               model_channels=320, attention_resolutions=[4, 2, 1], num_res_blocks=2, channel_mult=[1, 2, 4, 4],
               num_head_channels=64, use_linear_in_transformer=True, transformer_depth=1, context_dim=1024,
               spatial_transformer_attn_type="softmax-xformers", extra_ff_mix_layer=True, use_spatial_context=True,
               merge_strategy="learned_with_images", video_kernel_size=[3, 1, 1])

TAP_KINDS = ("conv_in", "res", "attn", "down", "up")
STANDIN_MARGIN = 1.25
# largest c the stand-in leg measured per kind (both geometries at width 64), times STANDIN_MARGIN
STANDIN_C = {"conv_in": 7.07e-4, "res": 7.16e-3, "res_skip": 1.85e-3, "attn": 4.26e-3, "down": 7.28e-4,
             "up": 7.07e-4, "out": 2.24e-3}
C_KIND = {k: STANDIN_MARGIN * v for k, v in STANDIN_C.items()}

# leg -> (model_channels, T, latent, weight seed); the fixture legs take their inputs from make_golden_perframe
GPU_LEGS = {"unet_small_t18_perframe": None, "unet_full_t5_perframe": None, "bench_v3d512": (320, 18, 64, 3)}
STANDIN_LEGS = {"w64_t18_16": (64, 18, 16, 2), "w64_t5_32": (64, 5, 32, 2)}


def _leg(tag):
    if tag in PERFRAME:
        m = PERFRAME[tag]
        return m["model_channels"], m["T"], m["latent_hw"], m["weight_seed"]
    return GPU_LEGS.get(tag) or STANDIN_LEGS[tag]


def _build(mc: int, wseed: int, dev):
    from oracle import synth
    from v3d_b200.unet import VideoUNet

    net = VideoUNet(**dict(UNET_KW, model_channels=mc))
    sd = synth.synth_state_dict(net.param_shapes(), seed=wseed)
    net.load_state_dict(sd, strict=True)
    return net.to(dev).eval(), sd


def run_tapped(net, spec, xin, ts, ctx, y, T, dev):
    """One forward with every conv_in / res / attn / down / up block tapped -> (output, {name: tap})."""
    B, _, H, W = xin.shape
    net.debug_taps = dict.fromkeys(n for n, k, _ in spec.blocks if k in TAP_KINDS)
    try:
        with torch.no_grad():
            if dev.type == "cuda":
                out = net(xin.to(dev), ts.to(dev), ctx.to(dev), y.to(dev), None, T, torch.zeros(B // T, T, device=dev))
            else:       # the host schedule itself, with the CPU stand-ins installed by the caller
                out = net._run(net._pack(dev), xin.float().contiguous(), ts.float().contiguous(),
                               ctx.reshape(B, -1).float().contiguous(), y.float().contiguous(), B, T, B // T, H, W, dev)
        taps = dict(net.debug_taps)
    finally:
        net.debug_taps = None
    missing = [n for n, v in taps.items() if v is None]
    assert not missing, f"blocks not tapped: {missing}"
    return out, taps


def _kind(kind, prm):
    return "res_skip" if kind == "res" and prm["cin"] != prm["cout"] else kind


def unet_parts(kind, T):
    """The UNet's partitions of a block output [B, C, H, W]: each of the 2T samples, each frame position t, each
    32-channel group, each 64-channel head (attention blocks), the border ring vs the interior (h, w >= 8)."""
    def parts(sq):
        B, C, H, W = sq.shape
        bc = sq.sum((2, 3))
        sample = bc.sum(1)
        p = {"sample": sample, "frame": sample.reshape(B // T, T).sum(0), "chan32": groups(bc.sum(0), min(32, C))}
        if kind == "attn":
            p["head"] = groups(bc.sum(0), 64)
        if H >= 8 and W >= 8:
            p["ring|interior"] = ring_interior(sq.sum((0, 1)))
        return p
    return parts


@torch.no_grad()
def check_blocks(sd, spec, xin, ts, ctx, y, T, out, taps, dev, c_kind=None):
    """Rebuild every block's input from the taps, run the oracle's block on it in fp64, judge the tap."""
    from oracle import ref_unet

    c_kind = C_KIND if c_kind is None else c_kind
    f64 = torch.float64
    sd = {k: v.to(dev, f64) for k, v in sd.items()}
    B = xin.shape[0]
    ind = torch.zeros(B // T, T, device=dev)
    emb = ref_unet.unet_embedding(sd, spec, ts.to(dev), y.to(dev, f64))
    ctx = ctx.to(dev, f64)
    cur = xin.to(dev).to(torch.bfloat16).to(f64)          # conv_in reads the latent converted to bf16 NHWC
    hs, rows = [], []
    for name, kind, prm in spec.blocks:
        if kind == "push":
            hs.append(cur)
            continue
        if kind == "pop_cat":
            cur = torch.cat([cur, hs.pop()], 1)
            continue
        if kind == "conv_in":
            ref = F.conv2d(cur, sd[name + ".weight"], sd[name + ".bias"], padding=1)
        elif kind == "res":
            ref = ref_unet.video_res_block(sd, name, cur, emb, T, ind)
        elif kind == "attn":
            ref = ref_unet.spatial_video_transformer(sd, name, cur, ctx, T, ind, spec.num_head_channels)
        elif kind == "down":
            ref = F.conv2d(cur, sd[name + ".op.weight"], sd[name + ".op.bias"], stride=2, padding=1)
        elif kind == "up":
            ref = F.conv2d(F.interpolate(cur, scale_factor=2, mode="nearest"), sd[name + ".conv.weight"],
                           sd[name + ".conv.bias"], padding=1)
        else:
            ref = F.conv2d(F.silu(ref_unet.group_norm32(cur, sd, "out.0", 1e-5)), sd["out.2.weight"],
                           sd["out.2.bias"], padding=1)
        got = (out if kind == "out" else taps[name]).to(dev, f64)
        k = _kind(kind, prm)
        rows.append(judge(name, k, cur, ref, got, c_kind[k], unet_parts(k, T), bf16_out=kind != "out"))
        cur = got
        if kind == "conv_in":
            hs.append(cur)
    return rows


def _inputs(tag, T, hw):
    from oracle import make_golden_perframe

    return make_golden_perframe.perframe_inputs(T, hw)


def _assert_rows(tag, rows):
    assert len(rows) == 46, len(rows)
    bad = [(r["name"], round(r["ratio"], 3)) for r in rows if not (r["finite"] and r["ratio"] <= 1.0)]
    assert not bad, f"{tag}: blocks over their error budget: {bad}"
    loc = [(r["name"], round(r["ratio"], 3), r["local_bad"][:6]) for r in rows if r["local_bad"]]
    assert not loc, f"{tag}: error concentrated in a part (> {LOCALITY_FACTOR} x whole + {LOCALITY_FLOOR}): {loc}"


def _summary(tag, rows):
    kinds = sorted({r["kind"] for r in rows})
    for k in kinds:
        rs = [r for r in rows if r["kind"] == k]
        b = max(rs, key=lambda r: r["ratio"])
        w = max(rs, key=lambda r: r["worst"][2])
        print(f"KIND {tag} {k}: budget {b['ratio']:.3f} ({b['name']}), worst part {w['worst'][2]:.3f} "
              f"({w['name']} {w['worst'][0]}:{w['worst'][1]}), max c {max(r['c'] for r in rs):.3e}")


# ---------------------------------------------------------------------------------------------------------------
# stand-in leg: the same code on the CPU with the kernels' torch stand-ins (no GPU)
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("leg", list(STANDIN_LEGS))
def test_unet_blocks_fp64_standin(leg):
    import emu_ops
    from oracle import ref_unet

    mc, T, hw, wseed = _leg(leg)
    dev = torch.device("cpu")
    net, sd = _build(mc, wseed, dev)
    spec = ref_unet.UNetSpec(model_channels=mc)
    xin, ts, ctx, y = _inputs(leg, T, hw)
    with emu_ops.patched():
        out, taps = run_tapped(net, spec, xin, ts, ctx, y, T, dev)
    rows = check_blocks(sd, spec, xin, ts, ctx, y, T, out, taps, dev)
    _summary(leg, rows)
    _assert_rows(leg, rows)


def test_block_check_flags_a_wrong_frame():
    """The judge itself: one frame of one block's tap replaced by its neighbour's is outside the bound, and a
    bf16 rounding of the exact output is inside it."""
    g = torch.Generator().manual_seed(3)
    T, B, C, H = 6, 12, 64, 8
    x_in = torch.randn(B, C, H, H, generator=g, dtype=torch.float64)
    ref = x_in + 0.3 * torch.randn(B, C, H, H, generator=g, dtype=torch.float64)
    good = ref.to(torch.bfloat16).double()
    r = judge("synthetic", "res", x_in, ref, good, 1e-3, unet_parts("res", T))
    assert r["ratio"] <= 1.0 and not r["local_bad"], r
    bad = good.clone()
    bad[T - 1] = good[T - 2]                              # the last frame of the first video reads its neighbour
    r = judge("synthetic", "res", x_in, ref, bad, 1e-3, unet_parts("res", T))
    assert r["ratio"] > 1.0 and r["worst"][0] in ("sample", "frame") and r["worst"][1] == T - 1, r
    assert ("sample", T - 1) in [p[:2] for p in r["local_bad"]], r


# ---------------------------------------------------------------------------------------------------------------
# GPU leg
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("leg", list(GPU_LEGS))
def test_unet_blocks_fp64_gpu(leg):
    from oracle import ref_unet, synth

    mc, T, hw, wseed = _leg(leg)
    dev = torch.device("cuda")
    net, sd = _build(mc, wseed, dev)
    spec = ref_unet.UNetSpec(model_channels=mc)
    if leg in PERFRAME:
        xin, ts, ctx, y = _inputs(leg, T, hw)
    else:
        x, c, uc, ts = synth.synth_inputs_perframe(T, hw, seed=29)
        xin = torch.cat([torch.cat([x, x]), torch.cat([uc["concat"], c["concat"]])], 1)
        ctx, y = torch.cat([uc["crossattn"], c["crossattn"]]), torch.cat([uc["vector"], c["vector"]])
    out, taps = run_tapped(net, spec, xin, ts, ctx, y, T, dev)
    del net
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    rows = check_blocks(sd, spec, xin, ts, ctx, y, T, out, taps, dev)
    torch.cuda.synchronize()
    print(f"MEM {leg}: fp64 oracle pass {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.2f}"
          f" GiB allocated ({base / 2**30:.2f} GiB of it output and taps) on {torch.cuda.get_device_name()}")
    _summary(leg, rows)
    _assert_rows(leg, rows)


# ---------------------------------------------------------------------------------------------------------------
# end to end, per sample, against the real reference's per-frame fixtures
# ---------------------------------------------------------------------------------------------------------------
def _close(a, b, tol):
    return ((a - b).abs().max() / b.abs().max()).item() <= tol


@pytest.mark.parametrize("tag", list(PERFRAME))
def test_oracle_unet_vs_reference_perframe_golden(tag):
    """The oracle on per-frame conditioning against the real reference: output within 2e-4 of its largest value,
    every block's tap (fp16 in the fixture) within 2e-3 - the rule of tests/test_oracle_cpu.py."""
    from oracle import ref_unet, synth

    m = PERFRAME[tag]
    gold = torch.load(GOLD / f"{tag}.pt")
    spec = ref_unet.UNetSpec(model_channels=m["model_channels"])
    sd = synth.synth_state_dict(ref_unet.unet_param_shapes(spec), seed=m["weight_seed"])
    T, s = m["T"], m["tap_stride"]
    xin, ts, ctx, y = _inputs(tag, T, m["latent_hw"])
    assert torch.equal(ts, gold["timesteps"])
    taps = {}
    with torch.no_grad():
        out = ref_unet.unet_forward(sd, spec, xin, ts, ctx, y, T, torch.zeros(2, T), taps=taps)
    assert _close(out, gold["out"], 2e-4)
    names = [k[4:] for k in gold if k.startswith("tap:")]
    assert len(names) == 45
    for n in names:
        assert _close(taps[n][:, ::4, ::s, ::s], gold["tap:" + n].float(), 2e-3), n


@pytest.mark.gpu
@pytest.mark.parametrize("tag", list(PERFRAME))
def test_unet_perframe_golden_per_sample(tag):
    """VideoUNet on per-frame conditioning against the real reference: each of the 2T samples within rel-L2 3e-2 and
    cosine 0.999 of the reference on its own.  Every block's tap (as the fixture keeps it: every 4th channel, every
    tap_stride-th pixel) is held to rel-L2 2e-2 over all samples and reported per sample.

    Per sample, that tap bound does not hold reliably.  On one H100 80GB HBM3 the worst sample of
    unet_small_t18_perframe's output_blocks.1.0 tap (sample 20) measured 1.82e-2 and 2.07e-2 in two runs of this code:
    the default GroupNorm statistics are summed with fp64 atomics, so bf16 roundings land differently from run to
    run, and one sample's accumulated error moves with them.  That is the bf16 error accumulated over the blocks
    before the tap, not a schedule error: the same forward passes the block-isolated fp64 check above, where each
    block's own error stays inside its budget.  On the frame-invariant fixtures the deepest tap of the unconditional
    sample is at 2.1-2.2e-2 already with the stand-ins of the kernels (tests/test_host_schedule_cpu.py)."""
    from framewise import per_sample
    from oracle import ref_unet

    m = PERFRAME[tag]
    gold = torch.load(GOLD / f"{tag}.pt")
    T, s = m["T"], m["tap_stride"]
    dev = torch.device("cuda")
    net, _ = _build(m["model_channels"], m["weight_seed"], dev)
    xin, ts, ctx, y = _inputs(tag, T, m["latent_hw"])
    out, taps = run_tapped(net, ref_unet.UNetSpec(model_channels=m["model_channels"]), xin, ts, ctx, y, T, dev)
    torch.cuda.synchronize()
    worst = assert_per_sample(f"{tag} output", out, gold["out"], 3e-2, 0.999)
    whole = {n: float((v[:, ::4, ::s, ::s].cpu() - gold["tap:" + n].float()).norm() / gold["tap:" + n].float().norm())
             for n, v in taps.items()}
    assert max(whole.values()) <= 2e-2, whole
    worst_tap = max((max(r for _, r, _ in per_sample(v[:, ::4, ::s, ::s], gold["tap:" + n])), n) for n, v in taps.items())
    print(tag, "worst sample rel-L2 / cosine", worst, "worst tap", max(whole.values()), "worst tap sample", worst_tap)
