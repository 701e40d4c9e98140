"""fp32 CPU restatement of VideoUNet.forward over a reference-keyed state_dict (TEST INFRASTRUCTURE).

Follows sgm/modules/diffusionmodules/video_model.py:442-493 and the blocks it dispatches to; every
function names the lines it restates.  Tensors keep the reference's NCHW / "(b t) ..." conventions.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

SD = Dict[str, torch.Tensor]
SDPA_CHUNK_BYTES = 1 << 30      # largest score tensor one attention call materialises


@dataclass
class UNetSpec:
    """Constructor arguments that shape the network (scripts/pub/configs/V3D_512.yaml:29-57)."""
    in_channels: int = 8
    out_channels: int = 4
    model_channels: int = 320
    num_res_blocks: int = 2
    attention_resolutions: Sequence[int] = (4, 2, 1)
    channel_mult: Sequence[int] = (1, 2, 4, 4)
    num_head_channels: int = 64
    context_dim: int = 1024
    adm_in_channels: int = 768
    transformer_depth: int = 1
    # derived: list of (name, kind, params)
    blocks: List[Tuple[str, str, dict]] = field(default_factory=list)

    def __post_init__(self):
        self.blocks = _layout(self)


def _layout(s: UNetSpec) -> List[Tuple[str, str, dict]]:
    """Block list in execution order, mirroring the constructor loops of video_model.py:186-440.
    kinds: conv_in, res, attn, down, up, out."""
    out: List[Tuple[str, str, dict]] = [("input_blocks.0.0", "conv_in", {})]
    ch = s.model_channels
    ds = 1
    skip_ch = [ch]
    idx = 1
    for level, mult in enumerate(s.channel_mult):
        for _ in range(s.num_res_blocks):
            out.append((f"input_blocks.{idx}.0", "res", {"cin": ch, "cout": mult * s.model_channels, "stage": "in"}))
            ch = mult * s.model_channels
            if ds in s.attention_resolutions:
                out.append((f"input_blocks.{idx}.1", "attn", {"ch": ch, "stage": "in"}))
            out.append((f"input_blocks.{idx}", "push", {}))
            skip_ch.append(ch)
            idx += 1
        if level != len(s.channel_mult) - 1:
            out.append((f"input_blocks.{idx}.0", "down", {"ch": ch}))
            out.append((f"input_blocks.{idx}", "push", {}))
            skip_ch.append(ch)
            ds *= 2
            idx += 1
    out.append(("middle_block.0", "res", {"cin": ch, "cout": ch, "stage": "mid"}))
    out.append(("middle_block.1", "attn", {"ch": ch, "stage": "mid"}))
    out.append(("middle_block.2", "res", {"cin": ch, "cout": ch, "stage": "mid"}))
    idx = 0
    for level, mult in list(enumerate(s.channel_mult))[::-1]:
        for i in range(s.num_res_blocks + 1):
            ich = skip_ch.pop()
            out.append((f"output_blocks.{idx}", "pop_cat", {}))
            out.append((f"output_blocks.{idx}.0", "res", {"cin": ch + ich, "cout": mult * s.model_channels, "stage": "out"}))
            ch = mult * s.model_channels
            j = 1
            if ds in s.attention_resolutions:
                out.append((f"output_blocks.{idx}.1", "attn", {"ch": ch, "stage": "out"}))
                j = 2
            if level and i == s.num_res_blocks:
                out.append((f"output_blocks.{idx}.{j}", "up", {"ch": ch}))
                ds //= 2
            idx += 1
    out.append(("out", "out", {}))
    return out


# ------------------------------------------------------------------------------------------------
# primitives
# ------------------------------------------------------------------------------------------------
def timestep_embedding(t: torch.Tensor, dim: int, max_period: float = 10000.0) -> torch.Tensor:
    """diffusionmodules/util.py:207-231 (repeat_only=False): cos | sin halves, fp32."""
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32) / half).to(t.device)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    return emb


def group_norm32(x: torch.Tensor, sd: SD, p: str, eps: float) -> torch.Tensor:
    """GroupNorm32(32, C) eps 1e-5 in fp32 (util.py:259-276) / Normalize eps 1e-6 (attention.py:130-133).
    At least fp32: an fp64 input (the block-isolated checks) is normalised in fp64, on the input's device."""
    dt = torch.promote_types(x.dtype, torch.float32)
    return F.group_norm(x.to(dt), 32, sd[p + ".weight"].to(dt), sd[p + ".bias"].to(dt), eps).type(x.dtype)


def lin(x: torch.Tensor, sd: SD, p: str) -> torch.Tensor:
    return F.linear(x, sd[p + ".weight"], sd.get(p + ".bias"))


def layer_norm(x: torch.Tensor, sd: SD, p: str) -> torch.Tensor:
    return F.layer_norm(x, (x.shape[-1],), sd[p + ".weight"], sd[p + ".bias"], 1e-5)


def alpha_blend(sd: SD, p: str, x_spatial, x_temporal, indicator: torch.Tensor, pattern: str):
    """AlphaBlender, merge_strategy learned_with_images (util.py:341-369):
    alpha = where(indicator, 1, sigmoid(mix_factor)); alpha*x_spatial + (1-alpha)*x_temporal."""
    mix = torch.sigmoid(sd[p + ".mix_factor"])[..., None]
    alpha = torch.where(indicator.bool().to(mix.device), torch.ones(1, 1, dtype=mix.dtype, device=mix.device), mix)
    b, t = alpha.shape
    if pattern == "b t -> b 1 t 1 1":
        alpha = alpha.reshape(b, 1, t, 1, 1)
    elif pattern == "b t -> (b t) 1 1":
        alpha = alpha.reshape(b * t, 1, 1)
    else:
        raise ValueError(pattern)
    return alpha * x_spatial + (1.0 - alpha) * x_temporal


def res_block(sd: SD, p: str, x: torch.Tensor, emb: Optional[torch.Tensor], dims: int, exchange_temb: bool):
    """ResBlock._forward without up/down or scale-shift (openaimodel.py:338-364).
    dims=3: Conv3d k=(3,1,1) pad (1,0,0) and GroupNorm over (C/32, T, H, W) (openaimodel.py:262-271)."""
    conv = F.conv2d if dims == 2 else F.conv3d
    pad = 1 if dims == 2 else (1, 0, 0)
    h = F.silu(group_norm32(x, sd, p + ".in_layers.0", 1e-5))
    h = conv(h, sd[p + ".in_layers.2.weight"], sd[p + ".in_layers.2.bias"], padding=pad)
    if emb is not None:
        emb_out = F.linear(F.silu(emb), sd[p + ".emb_layers.1.weight"], sd[p + ".emb_layers.1.bias"])
        while emb_out.dim() < h.dim():
            emb_out = emb_out[..., None]
        if exchange_temb:  # "b t c ... -> b c t ..."
            emb_out = emb_out.transpose(1, 2)
        h = h + emb_out
    h = F.silu(group_norm32(h, sd, p + ".out_layers.0", 1e-5))
    h = conv(h, sd[p + ".out_layers.3.weight"], sd[p + ".out_layers.3.bias"], padding=pad)
    if p + ".skip_connection.weight" in sd:
        x = conv(x, sd[p + ".skip_connection.weight"], sd[p + ".skip_connection.bias"])
    return x + h


def video_res_block(sd: SD, p: str, x, emb, T: int, indicator):
    """VideoResBlock.forward (video_model.py:62-81)."""
    x = res_block(sd, p, x, emb, dims=2, exchange_temb=False)
    bt, c, h, w = x.shape
    b = bt // T
    x5 = x.reshape(b, T, c, h, w).permute(0, 2, 1, 3, 4)  # "(b t) c h w -> b c t h w"
    xt = res_block(sd, p + ".time_stack", x5, emb.reshape(b, T, -1), dims=3, exchange_temb=True)
    out = alpha_blend(sd, p + ".time_mixer", x5, xt, indicator, "b t -> b 1 t 1 1")
    return out.permute(0, 2, 1, 3, 4).reshape(bt, c, h, w)


def attention(sd: SD, p: str, x: torch.Tensor, context: Optional[torch.Tensor], heads: int) -> torch.Tensor:
    """CrossAttention.forward (attention.py:286-349): q,k,v Linear(no bias), SDPA scale d^-0.5, to_out."""
    ctx = x if context is None else context
    q = F.linear(x, sd[p + ".to_q.weight"])
    k = F.linear(ctx, sd[p + ".to_k.weight"])
    v = F.linear(ctx, sd[p + ".to_v.weight"])
    b, n, c = q.shape
    d = c // heads

    def split(t):
        return t.reshape(b, -1, heads, d).permute(0, 2, 1, 3)

    q, k, v = split(q), split(k), split(v)
    # the score matrices of every (sample, head) at once, unless they pass SDPA_CHUNK_BYTES (an fp64 SDPA over
    # 36 samples x 5 heads x 4096^2 scores is 24 GB): then a few (sample, head) pairs per call
    step = max(1, SDPA_CHUNK_BYTES // (q.shape[2] * k.shape[2] * q.element_size()))
    if step >= b * heads:
        o = F.scaled_dot_product_attention(q, k, v)
    else:
        q, k, v = (t.reshape(b * heads, 1, -1, d) for t in (q, k, v))
        o = torch.cat([F.scaled_dot_product_attention(q[i:i + step], k[i:i + step], v[i:i + step])
                       for i in range(0, b * heads, step)]).reshape(b, heads, n, d)
    o = o.permute(0, 2, 1, 3).reshape(b, n, c)
    return lin(o, sd, p + ".to_out.0")


def feed_forward(sd: SD, p: str, x: torch.Tensor) -> torch.Tensor:
    """FeedForward with GEGLU (attention.py:92-118): proj -> chunk(value, gate) -> value*gelu(gate) -> Linear."""
    v, g = lin(x, sd, p + ".net.0.proj").chunk(2, dim=-1)
    return lin(v * F.gelu(g), sd, p + ".net.2")


def basic_transformer_block(sd: SD, p: str, x, context, heads: int):
    """BasicTransformerBlock._forward (attention.py:556-577)."""
    x = attention(sd, p + ".attn1", layer_norm(x, sd, p + ".norm1"), None, heads) + x
    x = attention(sd, p + ".attn2", layer_norm(x, sd, p + ".norm2"), context, heads) + x
    x = feed_forward(sd, p + ".ff", layer_norm(x, sd, p + ".norm3")) + x
    return x


def video_transformer_block(sd: SD, p: str, x, context, T: int, heads: int):
    """VideoTransformerBlock._forward (video_attention.py:109-140), ff_in present, is_res True."""
    bt, s, c = x.shape
    b = bt // T
    x = x.reshape(b, T, s, c).permute(0, 2, 1, 3).reshape(b * s, T, c)  # "(b t) s c -> (b s) t c"
    x = feed_forward(sd, p + ".ff_in", layer_norm(x, sd, p + ".norm_in")) + x
    x = attention(sd, p + ".attn1", layer_norm(x, sd, p + ".norm1"), None, heads) + x
    x = attention(sd, p + ".attn2", layer_norm(x, sd, p + ".norm2"), context, heads) + x
    x = feed_forward(sd, p + ".ff", layer_norm(x, sd, p + ".norm3")) + x
    return x.reshape(b, s, T, c).permute(0, 2, 1, 3).reshape(bt, s, c)


def spatial_video_transformer(sd: SD, p: str, x, context, T: int, indicator, head_dim: int = 64):
    """SpatialVideoTransformer.forward (video_attention.py:230-301): use_linear, depth 1,
    use_spatial_context (time_context = context[::T] repeated over h*w)."""
    bt, c, h, w = x.shape
    heads = c // head_dim
    x_in = x
    assert context.ndim == 3
    time_context = context[::T].repeat_interleave(h * w, dim=0)  # "b ... -> (b n) ..."
    x = group_norm32(x, sd, p + ".norm", 1e-6)
    x = x.permute(0, 2, 3, 1).reshape(bt, h * w, c)
    x = lin(x, sd, p + ".proj_in")
    frames = torch.arange(T, device=x.device).repeat(bt // T)
    t_emb = timestep_embedding(frames, c).to(x.dtype)          # sinusoids in fp32 like the reference
    emb = lin(F.silu(lin(t_emb, sd, p + ".time_pos_embed.0")), sd, p + ".time_pos_embed.2")[:, None, :]
    x = basic_transformer_block(sd, p + ".transformer_blocks.0", x, context, heads)
    x_mix = video_transformer_block(sd, p + ".time_stack.0", x + emb, time_context, T, heads)
    x = alpha_blend(sd, p + ".time_mixer", x, x_mix, indicator, "b t -> (b t) 1 1")
    x = lin(x, sd, p + ".proj_out")
    x = x.reshape(bt, h, w, c).permute(0, 3, 1, 2)
    return x + x_in


def unet_embedding(sd: SD, spec: UNetSpec, timesteps: torch.Tensor, y: torch.Tensor) -> torch.Tensor:
    """time_embed(timestep_embedding(t)) + label_emb(y) (video_model.py:462-467), in y's dtype; the sinusoids are
    fp32 like the reference's."""
    t_emb = timestep_embedding(timesteps, spec.model_channels).to(y.dtype)
    emb = lin(F.silu(lin(t_emb, sd, "time_embed.0")), sd, "time_embed.2")
    return emb + lin(F.silu(lin(y, sd, "label_emb.0.0")), sd, "label_emb.0.2")


def unet_forward(sd: SD, spec: UNetSpec, x, timesteps, context, y, num_video_frames: int, image_only_indicator,
                 taps: Optional[dict] = None):
    """VideoUNet.forward (video_model.py:442-493). `taps`, if given, receives block outputs by name."""
    T = num_video_frames
    emb = unet_embedding(sd, spec, timesteps, y.to(x.dtype))
    assert y.shape[0] == x.shape[0]
    h = x
    hs = []
    for name, kind, prm in spec.blocks:
        if kind == "conv_in":
            h = F.conv2d(h, sd[name + ".weight"], sd[name + ".bias"], padding=1)
            hs.append(h)
        elif kind == "res":
            h = video_res_block(sd, name, h, emb, T, image_only_indicator)
        elif kind == "attn":
            h = spatial_video_transformer(sd, name, h, context, T, image_only_indicator, spec.num_head_channels)
        elif kind == "down":  # Downsample conv s2 p1 (openaimodel.py:202-217)
            h = F.conv2d(h, sd[name + ".op.weight"], sd[name + ".op.bias"], stride=2, padding=1)
        elif kind == "up":  # nearest 2x then conv (openaimodel.py:150-167)
            h = F.interpolate(h, scale_factor=2, mode="nearest")
            h = F.conv2d(h, sd[name + ".conv.weight"], sd[name + ".conv.bias"], padding=1)
        elif kind == "push":
            hs.append(h)
        elif kind == "pop_cat":
            h = torch.cat([h, hs.pop()], dim=1)
        elif kind == "out":
            h = F.silu(group_norm32(h.type(x.dtype), sd, "out.0", 1e-5))
            h = F.conv2d(h, sd["out.2.weight"], sd["out.2.bias"], padding=1)
        if taps is not None and kind in ("res", "attn", "down", "up", "conv_in", "out"):
            taps[name] = h
    return h


def openai_wrapper(sd: SD, spec: UNetSpec, x, t, c: dict, **kw):
    """OpenAIWrapper.forward (wrappers.py:23-34): channel-concat c['concat'], crossattn->context, vector->y."""
    x = torch.cat((x, c["concat"]), dim=1) if "concat" in c else x
    return unet_forward(sd, spec, x, t, c.get("crossattn"), c.get("vector"), **kw)


def unet_param_shapes(spec: UNetSpec) -> Dict[str, Tuple[int, ...]]:
    """state_dict layout of the reference VideoUNet (SURVEY.md App. D), derived from the spec."""
    mc, te = spec.model_channels, spec.model_channels * 4
    sh: Dict[str, Tuple[int, ...]] = {}

    def wb(p, w, bias=True):
        sh[p + ".weight"] = tuple(w)
        if bias:
            sh[p + ".bias"] = (w[0],)

    def norm(p, c):
        sh[p + ".weight"] = (c,)
        sh[p + ".bias"] = (c,)

    def res(p, cin, cout, three_d, emb_ch):
        k = (3, 1, 1) if three_d else (3, 3)
        norm(p + ".in_layers.0", cin)
        wb(p + ".in_layers.2", (cout, cin) + k)
        if emb_ch:
            wb(p + ".emb_layers.1", (cout, emb_ch))
        norm(p + ".out_layers.0", cout)
        wb(p + ".out_layers.3", (cout, cout) + k)
        if cin != cout:
            wb(p + ".skip_connection", (cout, cin, 1, 1))

    def attn(p, c, ctx):
        wb(p + ".to_q", (c, c), False)
        wb(p + ".to_k", (c, ctx), False)
        wb(p + ".to_v", (c, ctx), False)
        wb(p + ".to_out.0", (c, c))

    def ff(p, c):
        wb(p + ".net.0.proj", (8 * c, c))
        wb(p + ".net.2", (c, 4 * c))

    wb("time_embed.0", (te, mc)); wb("time_embed.2", (te, te))
    wb("label_emb.0.0", (te, spec.adm_in_channels)); wb("label_emb.0.2", (te, te))
    for name, kind, prm in spec.blocks:
        if kind == "conv_in":
            wb(name, (mc, spec.in_channels, 3, 3))
        elif kind == "res":
            res(name, prm["cin"], prm["cout"], False, te)
            res(name + ".time_stack", prm["cout"], prm["cout"], True, te)
            sh[name + ".time_mixer.mix_factor"] = (1,)
        elif kind == "attn":
            c = prm["ch"]
            norm(name + ".norm", c)
            wb(name + ".proj_in", (c, c))
            tb = name + ".transformer_blocks.0"
            attn(tb + ".attn1", c, c); attn(tb + ".attn2", c, spec.context_dim); ff(tb + ".ff", c)
            for n in ("norm1", "norm2", "norm3"):
                norm(f"{tb}.{n}", c)
            ts = name + ".time_stack.0"
            norm(ts + ".norm_in", c); ff(ts + ".ff_in", c)
            attn(ts + ".attn1", c, c); attn(ts + ".attn2", c, spec.context_dim); ff(ts + ".ff", c)
            for n in ("norm1", "norm2", "norm3"):
                norm(f"{ts}.{n}", c)
            wb(name + ".time_pos_embed.0", (4 * c, c)); wb(name + ".time_pos_embed.2", (c, 4 * c))
            sh[name + ".time_mixer.mix_factor"] = (1,)
            wb(name + ".proj_out", (c, c))
        elif kind == "down":
            wb(name + ".op", (prm["ch"], prm["ch"], 3, 3))
        elif kind == "up":
            wb(name + ".conv", (prm["ch"], prm["ch"], 3, 3))
        elif kind == "out":
            norm("out.0", mc)
            wb("out.2", (spec.out_channels, mc, 3, 3))
    return sh
