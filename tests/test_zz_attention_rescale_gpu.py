"""Spatial attention with PEAKED score rows: the wgmma kernel keeps a running row maximum and rescales its
register-resident output rows and running sum whenever a key tile raises it (csrc/attention_tc.cu).  Here the key
magnitude grows (or shrinks) along the sequence, so the row maximum jumps by far more than 2^8 between tiles and the
rescale path runs with large factors many times.  Checker: fp32 ATen SDPA on the
same bf16-rounded inputs.  (File name sorts last: this case was added after the round-1 GPU budget was spent.)
"""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.mark.parametrize("nb,ntok,heads", [(2, 512, 2), (1, 1000, 3), (1, 4096, 1)])
@pytest.mark.parametrize("order", ["growing", "shrinking"])
def test_attention_spatial_peaked_rows(nb, ntok, heads, order):
    from v3d_b200 import ops

    torch.manual_seed(3)
    c = heads * 64
    q = torch.randn(nb, ntok, c, device=DEV) * 4.0
    k = torch.randn(nb, ntok, c, device=DEV)
    v = torch.randn(nb, ntok, c, device=DEV)
    ramp = 1.0 + 6.0 * torch.arange(ntok, device=DEV, dtype=torch.float32) / ntok   # |k| grows 7x along the keys
    if order == "shrinking":                                                         # max is in the first tile:
        ramp = ramp.flip(0)                                                          # later tiles never overshoot
    k = k * ramp[None, :, None]
    qkv = torch.cat([q, k, v], dim=-1).reshape(nb * ntok, 3 * c).to(torch.bfloat16)
    out = torch.empty(nb * ntok, c, device=DEV, dtype=torch.bfloat16)
    ops.attention_spatial(qkv, out, nb, ntok, heads, 64 ** -0.5)
    qf, kf, vf = [t.reshape(nb, ntok, heads, 64).permute(0, 2, 1, 3).float() for t in qkv.split(c, dim=-1)]
    ref = F.scaled_dot_product_attention(qf, kf, vf).permute(0, 2, 1, 3).reshape(nb * ntok, c)
    # the branch this file is about: logits span tens of log2 units across key tiles
    logits = (qf[0, 0, :4] @ kf[0, 0].T) * 64 ** -0.5 * 1.4427
    assert (logits.max(dim=-1).values - logits[:, :64].max(dim=-1).values).max() > 8.0 or order == "shrinking"
    got = out.float()
    rel = ((got - ref).norm() / ref.norm()).item()
    assert torch.isfinite(got).all(), "non-finite attention output"
    assert rel <= 2e-2, f"peaked-row attention rel-L2 {rel:.4f}"
    # same inputs through the mma.sync twin (an independent online-softmax implementation): the two kernels must agree
    out2 = torch.empty_like(out)
    ops.attention_spatial_mma(qkv, out2, nb, ntok, heads, 64 ** -0.5)
    rel2 = ((got - out2.float()).norm() / ref.norm()).item()
    assert rel2 <= 2e-2, f"wgmma vs mma.sync rel-L2 {rel2:.4f}"
