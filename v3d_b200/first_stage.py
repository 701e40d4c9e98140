"""FirstStage: what the first-stage Encoder and VideoDecoder (sgm/modules/diffusionmodules/model.py) share - the
ResnetBlock with temb = None and the single-head AttnBlock, each with its parameter shapes, packing and launches."""
from __future__ import annotations

import math

import torch

from . import ops
from .kernel_module import KernelModule


class FirstStage(KernelModule):
    # ---- parameter table ----------------------------------------------------------------------
    @staticmethod
    def _conv_shape(table: dict, key: str, co: int, ci: int, *ks: int) -> None:
        table[key + ".weight"] = (co, ci, *ks)
        table[key + ".bias"] = (co,)

    @staticmethod
    def _affine_shape(table: dict, key: str, c: int) -> None:
        table[key + ".weight"] = (c,)
        table[key + ".bias"] = (c,)

    def _resnet_block_shapes(self, table: dict, name: str, ci: int, co: int) -> None:
        self._affine_shape(table, name + ".norm1", ci)
        self._conv_shape(table, name + ".conv1", co, ci, 3, 3)
        self._affine_shape(table, name + ".norm2", co)
        self._conv_shape(table, name + ".conv2", co, co, 3, 3)
        if ci != co:
            self._conv_shape(table, name + ".nin_shortcut", co, ci, 1, 1)

    def _attn_block_shapes(self, table: dict, key: str, c: int) -> None:
        self._affine_shape(table, key + ".norm", c)
        for n in ("q", "k", "v", "proj_out"):
            self._conv_shape(table, f"{key}.{n}", c, c, 1, 1)

    def _init_value(self, key: str, shape) -> torch.Tensor:
        """Reference-like initialisation: unit norm scales, zero biases and norm shifts, conv weights
        uniform(-1/sqrt(fan_in), 1/sqrt(fan_in))."""
        if torch.empty(0).device.type == "meta":
            return torch.empty(shape)
        if len(shape) == 1:
            return torch.ones(shape) if key.endswith(".weight") else torch.zeros(shape)
        bound = 1.0 / math.sqrt(math.prod(shape[1:]))
        return (torch.rand(shape) * 2.0 - 1.0) * bound

    # ---- packing ------------------------------------------------------------------------------
    def _pack_resnet_block(self, P: dict, sd: dict, name: str, ci: int, co: int) -> None:
        self._pack_affine(P, sd, name + ".norm1")
        self._pack_affine(P, sd, name + ".norm2")
        for cname in (".conv1", ".conv2"):
            P[name + cname + ".weight"], P[name + cname + ".bias"] = self._pack_conv3x3(
                sd[name + cname + ".weight"], sd[name + cname + ".bias"])
        if ci != co:
            self._pack_1x1(P, sd, name + ".nin_shortcut")

    def _pack_attn_block(self, P: dict, sd: dict, key: str, c: int) -> None:
        """q | k stacked into one [2C, C] GEMM; v on its own (it is computed transposed, see `_attn`)."""
        self._pack_affine(P, sd, key + ".norm")
        wq, wk = sd[key + ".q.weight"].reshape(c, c), sd[key + ".k.weight"].reshape(c, c)
        P[key + ".qk.weight"] = self._bf(torch.cat([wq, wk], 0))
        P[key + ".qk.bias"] = self._f32(torch.cat([sd[key + ".q.bias"], sd[key + ".k.bias"]], 0))
        P[key + ".v.weight"] = self._bf(sd[key + ".v.weight"].reshape(c, c))
        P[key + ".v.bias"] = self._f32(sd[key + ".v.bias"])
        self._pack_1x1(P, sd, key + ".proj_out")

    # ---- launches -----------------------------------------------------------------------------
    def _resnet_block(self, P, name, ci, co, x, B, h, w):
        """ResnetBlock.forward with temb = None (model.py:131-151)."""
        hw = h * w
        a = self._gn(P, name + ".norm1", x, hw, B, ci, 1e-6, True)
        h1 = self._conv3x3(P, name + ".conv1", a, B, h, w, ci)
        a = self._gn(P, name + ".norm2", h1, hw, B, co, 1e-6, True)
        skip = x if ci == co else self._linear(P, name + ".nin_shortcut", x, B * hw)
        return self._conv3x3(P, name + ".conv2", a, B, h, w, co, r1=skip, s1=1.0, out=h1)

    def _attn(self, P, key, c, x, B, h, w):
        """AttnBlock (model.py:161-201): single head, d = C, over h*w tokens per frame.
        S = q k^T (fp32), softmax, O = P v; v's bias is added after P.v (rows of P sum to 1)."""
        hw = h * w
        rows = B * hw
        dev = x.device
        xn = self._gn(P, key + ".norm", x, hw, B, c, 1e-6, False)
        qk = self._linear(P, key + ".qk", xn, rows)                       # [rows, 2C]: q | k
        # V^T for all frames: vt[d, f*hw + j] = sum_k Wv[d,k] xn[f*hw + j, k]
        vt = torch.empty(c, rows, device=dev, dtype=torch.bfloat16)
        ops.gemm(P[key + ".v.weight"], xn, vt, K=c, N=rows, rows_per_batch=c)
        scores = torch.empty(B, hw, hw, device=dev, dtype=torch.float32)
        k_view = qk[:, c:]
        ops.gemm(qk, k_view, scores, K=c, N=hw, rows_per_batch=hw, batch=B, lda=2 * c, ldb=2 * c,
                 a_batch_stride=hw * 2 * c, b_batch_stride=hw * 2 * c)
        probs = torch.empty(B, hw, hw, device=dev, dtype=torch.bfloat16)
        ops.softmax_rows_f32(scores, probs, B * hw, hw, float(c) ** -0.5)
        del scores
        o = torch.empty(rows, c, device=dev, dtype=torch.bfloat16)
        ops.gemm(probs, vt, o, K=hw, N=c, rows_per_batch=hw, batch=B, a_batch_stride=hw * hw, ldb=rows,
                 b_batch_stride=hw, bias=P[key + ".v.bias"])
        return self._linear(P, key + ".proj_out", o, rows, out=xn, r1=x, s1=1.0)
