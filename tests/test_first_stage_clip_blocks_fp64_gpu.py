"""Every block of the first-stage decoder and encoder and every half-layer of the CLIP image tower, against the oracle
in fp64 on its own input.

The parity tests judge each of these networks on its final output only (rel-L2 <= 3e-2, cosine >= 0.999; per frame
for the decoder), and bf16 alone spends about half of that.  A mistake confined to one block - a merge weight applied to
the wrong branch, a temporal conv that does not restart at a video boundary, a pad on the wrong side, a key masked as
padding - fits in the other half.  This file takes the three forwards apart the way tests/test_unet_blocks_fp64_gpu.py
takes the UNet apart:

  * One forward with every block tapped (`debug_taps`).  A tap is the block's bf16 output widened to fp32, so it
    equals the next block's input bit for bit: NCHW for the decoder and encoder, the residual stream [B, n, width] for
    CLIP (`pre` after ln_pre, `L{i}.attn` / `L{i}.mlp` after the two halves of layer i).
  * Every block's input is rebuilt from the previous tap (the first block reads what the kernels read: bf16(z),
    bf16(x), the bf16 patch columns of the module's own preprocess), the oracle's block (oracle/ref_decoder.py,
    ref_encoder.py, ref_clip.py) runs on it in fp64 with the same weights, and the tap is judged by
    framewise.judge: ||err_p|| <= c_kind ||upd_p|| + ||rnd_p|| for the whole block (ratio <= 1) and every part's ratio
    at most 2 x the whole + 0.1.  The final outputs (decoder image, encoder moments, CLIP z) are fp32: rnd = 0.
  * Partitions.  Decoder: each sample, each frame position t, each video, each 32-channel group, border ring vs
    interior (h, w >= 8) and, for the mid attention, each 128-token tile of the h*w raster.  Encoder: each image, each
    32-channel group, ring vs interior (the downsample's pad sits on the last row and column).  CLIP: each image, the
    class token, each 64-token block (the last one ragged: token 256 alone at ViT-H/14), the last token, each
    32-channel group and, for the attention half, each head (width 80).

c_kind.  The stand-in leg (`standin`, no GPU) runs the same code with tests/emu_ops.py in place of the kernels (fp64
arithmetic, bf16 wherever the kernels store bf16), on the geometries of decoder_small (one video, T = 3, latent 16^2),
decoder_small_2videos (two videos of T = 2, latent 8^2), encoder_small (64^2) and clip_small, all at width 64 (CLIP:
320).  Its measured c = (||err|| - ||rnd||)+ / ||upd||, largest over the blocks of a kind, times STANDIN_MARGIN = 1.25 is
C_KIND.  On one H100 80GB HBM3 (700 W limit, running under its software power cap) the kernels' c matched the
stand-ins' within 3 % for every kind at the stand-in shapes, the decoder's mid attention included (bf16 probabilities
over 256 to 4096 keys: c 1.9e-4 to 4.6e-4, the block's budget taken almost entirely by the bf16 rounding of its
output).  The one kind above its stand-in value is the CLIP head at ViT-H/14 width (c 2.48e-3 against 2.07e-3 measured
at clip_small's width 320, inside C_KIND = 2.59e-3): a 1280-long contraction instead of a 320-long one.  Largest budget
ratios over the GPU legs: decoder conv_in 0.93, vres 0.93, vres_skip 0.89, attn 1.00, up 0.93, out 0.82; encoder
conv_in 0.93, res 0.89, res_skip 0.89, down 0.93, attn 0.97, out 0.81; CLIP embed 0.90, attn_half 0.93, mlp_half 0.93,
head 0.96.  Largest part ratio 1.24 (CLIP head, one 32-channel group, whole 0.96).  At the V3D decode shape the fp64
oracle pass took 5 s and peaked at 58.9 GiB, 20.2 GiB of it the output and taps: it fits beside them on an 80 GB card.

Legs: `standin` as above; `gpu` on the weights and inputs of decoder_small, decoder_small_2videos and decoder_full, at
the V3D decode shape itself (T = 18, latent 64^2, width 128, weight seed 6, the z of decoder_v3d512), on encoder_small,
encoder_full and one 512^2 image at width 128, and on clip_small and clip_vit_h14; there the oracle runs on the GPU and
each leg prints a MEM line.  Each tap is released as soon as its block is judged, so at the V3D decode shape the
fp32 taps (about 21 GB, from the shapes) are mostly gone when the 512^2 blocks' oracle runs.

The planted-fault tests at the end show the gap this closes: each fault keeps the whole output inside the parity bound
of tests/test_parity_gpu.py against the oracle, and fails here at the block and part where it was planted.
"""
import contextlib
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
MANIFEST = json.loads((GOLD / "MANIFEST.json").read_text())
BF = torch.bfloat16
F64 = torch.float64

DEC_KW = dict(attn_type="vanilla", double_z=True, z_channels=4, resolution=256, in_channels=3, out_ch=3, ch=64,
              ch_mult=[1, 2, 4, 4], num_res_blocks=2, attn_resolutions=[], dropout=0.0, video_kernel_size=[3, 1, 1])
ENC_KW = dict(attn_type="vanilla", double_z=True, z_channels=4, in_channels=3, out_ch=3, ch=64, ch_mult=[1, 2, 4, 4],
              num_res_blocks=2, attn_resolutions=[], dropout=0.0)

STANDIN_MARGIN = 1.25
# largest c the stand-in leg measured per kind, times STANDIN_MARGIN
STANDIN_C = {
    "decoder": {"conv_in": 6.95e-4, "vres": 6.82e-3, "vres_skip": 1.71e-3, "attn": 4.52e-4, "up": 7.01e-4,
                "out": 2.43e-3},
    "encoder": {"conv_in": 7.05e-4, "res": 2.37e-3, "res_skip": 1.66e-3, "down": 7.43e-4, "attn": 8.73e-4,
                "out": 2.64e-3},
    "clip": {"embed": 1.62e-3, "attn_half": 1.94e-3, "mlp_half": 1.43e-3, "head": 2.07e-3},
}
C_KIND = {net: {k: STANDIN_MARGIN * v for k, v in kinds.items()} for net, kinds in STANDIN_C.items()}

# leg -> (network, fixture / shape).  A fixture leg takes weights and inputs from tests/golden/MANIFEST.json.
STANDIN_LEGS = {"decoder_small": "decoder", "decoder_small_2videos": "decoder", "encoder_small": "encoder",
                "clip_small": "clip"}
GPU_LEGS = {"decoder_small": "decoder", "decoder_small_2videos": "decoder", "decoder_full": "decoder",
            "decoder_v3d512": "decoder", "encoder_small": "encoder", "encoder_full": "encoder",
            "encoder_512": "encoder", "clip_small": "clip", "clip_vit_h14": "clip"}
ENCODER_512 = dict(B=1, ch=128, image_hw=512, weight_seed=8, x_seed=78)


# ---------------------------------------------------------------------------------------------------------------
# networks, inputs and tapped forwards
# ---------------------------------------------------------------------------------------------------------------
def _decoder(tag, dev):
    """-> (module, state dict, module input z / 0.18215, T)"""
    from oracle import synth
    from v3d_b200.decoder import VideoDecoder

    m = MANIFEST[tag]
    dec = VideoDecoder(**dict(DEC_KW, ch=m["ch"]))
    sd = synth.synth_state_dict(dec.param_shapes(), seed=m["weight_seed"])
    dec.load_state_dict(sd, strict=True)
    if tag == "decoder_v3d512":
        g = torch.Generator().manual_seed(m["z_seed"])
        z = torch.randn(m["B"], 4, m["latent_hw"], m["latent_hw"], generator=g)
    else:
        z = torch.load(GOLD / f"{tag}.pt")["z"]
    return dec.to(dev).eval(), sd, z / 0.18215, m["T"]


def _encoder(tag, dev):
    """-> (module, state dict, image)"""
    from oracle import ref_encoder, synth
    from v3d_b200.encoder import Encoder

    m = ENCODER_512 if tag == "encoder_512" else MANIFEST[tag]
    enc = Encoder(**dict(ENC_KW, ch=m["ch"], resolution=m["image_hw"]))
    sd = synth.synth_state_dict(ref_encoder.encoder_param_shapes(ref_encoder.EncoderSpec(ch=m["ch"])),
                                seed=m["weight_seed"])
    enc.load_state_dict(sd, strict=True)
    if tag == "encoder_512":
        g = torch.Generator().manual_seed(m["x_seed"])
        x = torch.rand(m["B"], 3, m["image_hw"], m["image_hw"], generator=g) * 2.0 - 1.0
    else:
        x = torch.load(GOLD / f"{tag}.pt")["x"]
    return enc.to(dev).eval(), sd, x


def _clip(tag, dev):
    """-> (module, visual state dict, spec, image in [-1, 1])"""
    from oracle import ref_clip, synth
    from v3d_b200.clip import FrozenOpenCLIPImageEmbedder

    m = MANIFEST[tag]
    spec = ref_clip.ClipSpec(**m["spec"])
    emb = FrozenOpenCLIPImageEmbedder(freeze=True, vision_cfg=m["spec"])
    sd = synth.synth_state_dict(ref_clip.clip_visual_param_shapes(spec), seed=m["weight_seed"])
    missing, unexpected = emb.load_state_dict({"model.visual." + k: v for k, v in sd.items()}, strict=False)
    assert not unexpected and all(".visual." not in k for k in missing)
    g = torch.Generator().manual_seed(m["x_seed"])
    x = torch.rand(m["B"], 3, m["image_hw"], m["image_hw"], generator=g) * 2.0 - 1.0
    return emb.to(dev).eval(), sd, spec, x


def _tap_names(net, module):
    if net == "clip":
        return ["pre"] + [f"L{i}.{h}" for i in range(module.model.visual.layers) for h in ("attn", "mlp")]
    return ["conv_in"] + [n.rsplit(":", 1)[-1] for n, _, _ in module._blocks()]


def run_tapped(net, module, x, T=None):
    """One forward with every block tapped -> (fp32 output, {name: tap})."""
    module.debug_taps = dict.fromkeys(_tap_names(net, module))
    try:
        with torch.no_grad():
            if net == "decoder":
                out = module(x, timesteps=T)
            elif net == "encoder":
                out = module(x)
            else:
                out = module.encode_with_vision_transformer(x)
        taps = dict(module.debug_taps)
    finally:
        module.debug_taps = None
    missing = [n for n, v in taps.items() if v is None]
    assert not missing, f"blocks not tapped: {missing}"
    return out, taps


# ---------------------------------------------------------------------------------------------------------------
# partitions
# ---------------------------------------------------------------------------------------------------------------
def decoder_parts(kind, T):
    def parts(sq):                                                            # [B, C, H, W]
        B, C, H, W = sq.shape
        bc = sq.sum((2, 3))
        sample = bc.sum(1)
        per_video = sample.reshape(B // T, T)
        p = {"sample": sample, "frame": per_video.sum(0), "video": per_video.sum(1), "chan32": groups(bc.sum(0), 32)}
        if H >= 8 and W >= 8 or kind == "attn":
            hw = sq.sum((0, 1))
            if H >= 8 and W >= 8:
                p["ring|interior"] = ring_interior(hw)
            if kind == "attn":
                p["tile128"] = groups(hw.reshape(-1), 128)
        return p
    return parts


def encoder_parts(kind):
    def parts(sq):                                                            # [B, C, H, W]
        bc = sq.sum((2, 3))
        p = {"image": bc.sum(1), "chan32": groups(bc.sum(0), 32)}
        if sq.shape[2] >= 8 and sq.shape[3] >= 8:
            p["ring|interior"] = ring_interior(sq.sum((0, 1)))
        return p
    return parts


def clip_parts(kind, head_width):
    def parts(sq):
        if sq.dim() == 2:                                                     # head: [B, embed_dim]
            return {"image": sq.sum(1), "chan32": groups(sq.sum(0), 32)}
        tok, ch = sq.sum((0, 2)), sq.sum((0, 1))                              # [B, n, width]
        p = {"image": sq.sum((1, 2)), "cls": tok[:1], "tok64": groups(tok, 64), "last": tok[-1:],
             "chan32": groups(ch, 32)}
        if kind == "attn_half":
            p["head"] = groups(ch, head_width)
        return p
    return parts


# ---------------------------------------------------------------------------------------------------------------
# block-by-block checks
# ---------------------------------------------------------------------------------------------------------------
def _judge_tap(rows, taps, name, kind, cur, ref, c_kind, parts, dev):
    got = taps.pop(name).to(dev, F64)                                         # released once judged
    rows.append(judge(name, kind, cur, ref, got, c_kind[kind], parts))
    return got


@torch.no_grad()
def check_decoder(dec, sd, z, T, out, taps, dev, c_kind=None):
    from oracle import ref_decoder

    c_kind = C_KIND["decoder"] if c_kind is None else c_kind
    sd = {k: v.to(dev, F64) for k, v in sd.items()}
    taps, rows = dict(taps), []
    cur = z.to(dev).to(BF).to(F64)                                            # conv_in reads bf16 NHWC
    ref = F.conv2d(cur, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    cur = _judge_tap(rows, taps, "conv_in", "conv_in", cur, ref, c_kind, decoder_parts("conv_in", T), dev)
    for name, ci, co in dec._blocks():
        if name.startswith("@attn:"):
            name, kind = name[6:], "attn"
            ref = ref_decoder.attn_block(sd, name, cur)
        elif name.startswith("@up:"):
            name, kind = name[4:], "up"
            ref = ref_decoder.upsample(sd, name, cur)
        else:
            kind = "vres" if ci == co else "vres_skip"
            ref = ref_decoder.video_res_block(sd, name, cur, T)
        cur = _judge_tap(rows, taps, name, kind, cur, ref, c_kind, decoder_parts(kind, T), dev)
        del ref
    ref = ref_decoder.decoder_tail(sd, cur, T)
    rows.append(judge("out", "out", cur, ref, out.to(dev, F64), c_kind["out"], decoder_parts("out", T),
                      bf16_out=False))
    return rows


@torch.no_grad()
def check_encoder(enc, sd, x, out, taps, dev, c_kind=None):
    from oracle import ref_decoder, ref_encoder

    c_kind = C_KIND["encoder"] if c_kind is None else c_kind
    sd = {k: v.to(dev, F64) for k, v in sd.items()}
    taps, rows = dict(taps), []
    cur = x.to(dev).to(BF).to(F64)                                            # conv_in reads bf16 NHWC
    ref = F.conv2d(cur, sd["conv_in.weight"], sd["conv_in.bias"], padding=1)
    cur = _judge_tap(rows, taps, "conv_in", "conv_in", cur, ref, c_kind, encoder_parts("conv_in"), dev)
    for name, ci, co in enc._blocks():
        if name.startswith("@attn:"):
            name, kind = name[6:], "attn"
            ref = ref_decoder.attn_block(sd, name, cur)
        elif name.startswith("@down:"):
            name, kind = name[6:], "down"
            ref = ref_encoder.downsample(sd, name, cur)
        else:
            kind = "res" if ci == co else "res_skip"
            ref = ref_decoder.resnet_block(sd, name, cur)
        cur = _judge_tap(rows, taps, name, kind, cur, ref, c_kind, encoder_parts(kind), dev)
        del ref
    ref = ref_encoder.encoder_tail(sd, cur)
    rows.append(judge("out", "out", cur, ref, out.to(dev, F64), c_kind["out"], encoder_parts("out"), bf16_out=False))
    return rows


@torch.no_grad()
def check_clip(sd, spec, img, out, taps, dev, c_kind=None):
    from oracle import ref_clip

    c_kind = C_KIND["clip"] if c_kind is None else c_kind
    sd = {k: v.to(dev, F64) for k, v in sd.items()}
    taps, rows = dict(taps), []
    hd = spec.width // spec.heads
    img = img.to(dev).to(BF).to(F64)                                          # conv1 reads these as bf16 columns
    ref = ref_clip.clip_embed(sd, spec, img)
    cur = _judge_tap(rows, taps, "pre", "embed", img, ref, c_kind, clip_parts("embed", hd), dev)
    for i in range(spec.layers):
        ref = ref_clip.clip_attn_half(sd, spec, i, cur)
        cur = _judge_tap(rows, taps, f"L{i}.attn", "attn_half", cur, ref, c_kind, clip_parts("attn_half", hd), dev)
        ref = ref_clip.clip_mlp_half(sd, spec, i, cur)
        cur = _judge_tap(rows, taps, f"L{i}.mlp", "mlp_half", cur, ref, c_kind, clip_parts("mlp_half", hd), dev)
    ref = ref_clip.clip_head(sd, spec, cur)
    rows.append(judge("head", "head", cur, ref, out.to(dev, F64), c_kind["head"], clip_parts("head", hd),
                      bf16_out=False))
    return rows


def run_leg(tag, net, dev):
    """Tapped forward + block checks of one leg -> rows.  On the GPU the oracle pass prints a MEM line."""
    if net == "decoder":
        module, sd, z, T = _decoder(tag, dev)
        out, taps = run_tapped(net, module, z.to(dev), T)
        check = lambda: check_decoder(module, sd, z, T, out, taps, dev)           # noqa: E731
    elif net == "encoder":
        module, sd, x = _encoder(tag, dev)
        out, taps = run_tapped(net, module, x.to(dev))
        check = lambda: check_encoder(module, sd, x, out, taps, dev)              # noqa: E731
    else:
        module, sd, spec, x = _clip(tag, dev)
        out, taps = run_tapped(net, module, x.to(dev))
        img = module.preprocess(x.to(dev))                                        # the module's own preprocessing
        check = lambda: check_clip(sd, spec, img, out, taps, dev)                 # noqa: E731
    if dev.type != "cuda":
        return check()
    module.to("meta")                                                             # its packed weights go too
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    rows = check()
    torch.cuda.synchronize()
    print(f"MEM {tag}: fp64 oracle pass {time.time() - t0:.1f} s, peak {torch.cuda.max_memory_allocated() / 2**30:.2f}"
          f" GiB allocated ({base / 2**30:.2f} GiB of it output and taps) on {torch.cuda.get_device_name()}")
    return rows


def assert_rows(tag, rows):
    bad = [(r["name"], round(r["ratio"], 3)) for r in rows if not (r["finite"] and r["ratio"] <= 1.0)]
    assert not bad, f"{tag}: blocks over their error budget: {bad}"
    loc = [(r["name"], round(r["ratio"], 3), r["local_bad"][:6]) for r in rows if r["local_bad"]]
    assert not loc, f"{tag}: error concentrated in a part (> {LOCALITY_FACTOR} x whole + {LOCALITY_FLOOR}): {loc}"


def summary(tag, rows):
    for k in sorted({r["kind"] for r in rows}):
        rs = [r for r in rows if r["kind"] == k]
        b = max(rs, key=lambda r: r["ratio"])
        w = max(rs, key=lambda r: r["worst"][2])
        print(f"KIND {tag} {k}: budget {b['ratio']:.3f} ({b['name']}), worst part {w['worst'][2]:.3f} "
              f"({w['name']} {w['worst'][0]}:{w['worst'][1]}), max c {max(r['c'] for r in rs):.3e}")


# ---------------------------------------------------------------------------------------------------------------
# stand-in leg (CPU) and GPU leg
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("leg", list(STANDIN_LEGS))
def test_first_stage_clip_blocks_fp64_standin(leg):
    import emu_ops

    with emu_ops.patched():
        rows = run_leg(leg, STANDIN_LEGS[leg], torch.device("cpu"))
    summary(leg, rows)
    assert_rows(leg, rows)


@pytest.mark.gpu
@pytest.mark.parametrize("leg", list(GPU_LEGS))
def test_first_stage_clip_blocks_fp64_gpu(leg):
    rows = run_leg(leg, GPU_LEGS[leg], torch.device("cuda"))
    summary(leg, rows)
    assert_rows(leg, rows)


# ---------------------------------------------------------------------------------------------------------------
# the judge on the new partitions
# ---------------------------------------------------------------------------------------------------------------
def test_block_check_flags_a_wrong_token_row():
    """One CLIP token row replaced by its neighbour's (the last, ragged one: token 256) is flagged in that token's
    partitions, and a bf16 rounding of the exact output passes."""
    g = torch.Generator().manual_seed(5)
    x_in = torch.randn(2, 257, 320, generator=g, dtype=F64)
    ref = x_in + 0.3 * torch.randn(2, 257, 320, generator=g, dtype=F64)
    good = ref.to(BF).double()
    r = judge("synthetic", "attn_half", x_in, ref, good, 1e-3, clip_parts("attn_half", 80))
    assert r["ratio"] <= 1.0 and not r["local_bad"], r
    bad = good.clone()
    bad[1, 256] = good[1, 255]
    r = judge("synthetic", "attn_half", x_in, ref, bad, 1e-3, clip_parts("attn_half", 80))
    assert r["worst"][0] in ("last", "tok64") and r["worst"][1] == (0 if r["worst"][0] == "last" else 4), r
    assert ("tok64", 4) in [p[:2] for p in r["local_bad"]] and ("last", 0) in [p[:2] for p in r["local_bad"]], r


def test_block_check_flags_a_wrong_attention_tile():
    """One 128-token tile of the decoder attention's h*w raster replaced by its neighbour's is flagged there."""
    g = torch.Generator().manual_seed(6)
    x_in = torch.randn(4, 64, 32, 32, generator=g, dtype=F64)
    ref = x_in + 0.3 * torch.randn(4, 64, 32, 32, generator=g, dtype=F64)
    good = ref.to(BF).double()
    r = judge("synthetic", "attn", x_in, ref, good, 1e-3, decoder_parts("attn", 2))
    assert r["ratio"] <= 1.0 and not r["local_bad"], r
    bad = good.clone()
    bad[:, :, 20:24] = good[:, :, 16:20]                                      # tokens 640..767 read tokens 512..639
    r = judge("synthetic", "attn", x_in, ref, bad, 1e-3, decoder_parts("attn", 2))
    assert r["ratio"] > 1.0 and r["worst"][:2] == ("tile128", 5), r
    assert [p[:2] for p in r["local_bad"] if p[0] == "tile128"] == [("tile128", 5)], r


# ---------------------------------------------------------------------------------------------------------------
# planted schedule faults (stand-in leg): inside the parity bound, flagged at their block
# ---------------------------------------------------------------------------------------------------------------
def _rel_cos(got, ref):
    a, b = got.double().flatten(), ref.double().flatten()
    return float((a - b).norm() / b.norm()), float(a @ b / (a.norm() * b.norm()))


def _assert_flagged_only(rows, block):
    flagged = [r["name"] for r in rows if r["ratio"] > 1.0 or r["local_bad"]]
    assert flagged == [block], flagged
    return next(r for r in rows if r["name"] == block)


@contextlib.contextmanager
def _instance_override(module, attr, fn):
    object.__setattr__(module, attr, fn)
    try:
        yield
    finally:
        object.__delattr__(module, attr)


def test_planted_decoder_alpha_swap_is_flagged():
    """up.1.block.0 merges with 1 - alpha in place of alpha (alpha = sigmoid(mix_factor) = 0.47 here, so the swap moves
    the output little): per frame inside rel-L2 3e-2 / cosine 0.999 of the oracle, over budget at that block."""
    import emu_ops
    from oracle import ref_decoder

    dev = torch.device("cpu")
    dec, sd, z, T = _decoder("decoder_small", dev)
    with emu_ops.patched():
        P = dec.packed()
        P["up.1.block.0.alpha"] = 1.0 - P["up.1.block.0.alpha"]
        out, taps = run_tapped("decoder", dec, z, T)
    dec._invalidate()
    rows = check_decoder(dec, sd, z, T, out, taps, dev)
    ref = ref_decoder.decoder_forward({k: v.double() for k, v in sd.items()}, ref_decoder.DecoderSpec(ch=64),
                                      z.double(), T)
    r, cs = _rel_cos(out, ref)
    print(f"FAULT decoder alpha swap in up.1.block.0: whole output rel-L2 {r:.4f} cosine {cs:.6f}")
    assert r <= 3e-2 and cs >= 0.999
    assert_per_sample("decoder with the alpha swap", out, ref, 3e-2, 0.999)
    assert _assert_flagged_only(rows, "up.1.block.0")["ratio"] > 1.0


def test_planted_encoder_batch_pooled_groupnorm_is_flagged():
    """down.0.block.0's first GroupNorm takes its statistics over both images of the batch instead of each image's
    own (nsamples = 1 over B x h*w rows): inside rel-L2 3e-2 of the oracle's moments, over budget at that block."""
    import emu_ops
    from oracle import ref_encoder

    dev = torch.device("cpu")
    enc, sd, x = _encoder("encoder_small", dev)
    gn = enc._gn

    def pooled(P, key, x_, rows_per_sample, nsamples, c, eps, silu, **kw):
        if key == "down.0.block.0.norm1":
            rows_per_sample, nsamples = rows_per_sample * nsamples, 1
        return gn(P, key, x_, rows_per_sample, nsamples, c, eps, silu, **kw)

    with emu_ops.patched(), _instance_override(enc, "_gn", pooled):
        out, taps = run_tapped("encoder", enc, x)
    rows = check_encoder(enc, sd, x, out, taps, dev)
    ref = ref_encoder.encoder_forward({k: v.double() for k, v in sd.items()}, ref_encoder.EncoderSpec(ch=64),
                                      x.double())
    r, cs = _rel_cos(out, ref)
    print(f"FAULT encoder batch-pooled GroupNorm in down.0.block.0: whole output rel-L2 {r:.4f} cosine {cs:.6f}")
    assert r <= 3e-2 and cs >= 0.999
    assert _assert_flagged_only(rows, "down.0.block.0")["ratio"] > 1.0


def test_planted_clip_last_key_masked_is_flagged():
    """Layer 1 masks the last key (token n - 1) of head 2 as if it were padding: the pooled embedding stays inside
    rel-L2 3e-2 / cosine 0.999 of the oracle, the attention half of layer 1 is over budget."""
    import emu_ops
    from oracle import ref_clip
    from v3d_b200 import ops

    dev = torch.device("cpu")
    emb, sd, spec, x = _clip("clip_small", dev)
    n = (spec.image_size // spec.patch) ** 2 + 1
    calls = [0]
    with emu_ops.patched():
        softmax = ops.softmax_rows_f32

        def masked(s, p, rows, nk, scale=1.0):
            if calls[0] == 1:                                                 # one softmax per layer
                s.view(-1, spec.heads, n, nk)[:, 2, :, n - 1] = -1e30
            calls[0] += 1
            return softmax(s, p, rows, nk, scale)

        ops.softmax_rows_f32 = masked
        out, taps = run_tapped("clip", emb, x)
        img = emb.preprocess(x)
    assert calls[0] == spec.layers
    rows = check_clip(sd, spec, img, out, taps, dev)
    sd64 = {k: v.double() for k, v in sd.items()}
    ref = ref_clip.clip_visual_forward(sd64, spec, ref_clip.preprocess(x.double(), spec.image_size))
    r, cs = _rel_cos(out, ref)
    print(f"FAULT CLIP last key masked in layer 1, head 2: pooled embedding rel-L2 {r:.4f} cosine {cs:.6f}")
    assert r <= 3e-2 and cs >= 0.999
    assert _assert_flagged_only(rows, "L1.attn")["ratio"] > 1.0
