"""Per-sample / per-frame views of the parity metrics (shared by the UNet, sampler and decoder parity tests).

A whole-tensor rel-L2 over a CFG batch of 36 samples lets a mistake confined to one frame through: that frame is
under 3 % of the tensor.  These helpers apply the same bound to every leading-index slice on its own."""
from __future__ import annotations

from typing import List, Optional, Tuple

import torch


def per_sample(got: torch.Tensor, ref: torch.Tensor) -> List[Tuple[int, float, float]]:
    """[(index, rel-L2, cosine)] of every slice along dim 0."""
    assert got.shape == ref.shape, (tuple(got.shape), tuple(ref.shape))
    a = got.detach().double().cpu().reshape(got.shape[0], -1)
    b = ref.detach().double().cpu().reshape(ref.shape[0], -1)
    rel = (a - b).norm(dim=1) / b.norm(dim=1).clamp_min(1e-12)
    cos = (a * b).sum(dim=1) / (a.norm(dim=1) * b.norm(dim=1)).clamp_min(1e-12)
    return [(i, float(r), float(c)) for i, (r, c) in enumerate(zip(rel, cos))]


def assert_per_sample(what: str, got: torch.Tensor, ref: torch.Tensor, rel: float,
                      cos: Optional[float] = None) -> Tuple[float, float]:
    """Every slice along dim 0 within rel-L2 `rel` (and cosine >= `cos`); returns the worst (rel-L2, cosine)."""
    rows = per_sample(got, ref)
    worst_r = max(r for _, r, _ in rows)
    worst_c = min(c for _, _, c in rows)
    bad = [(i, round(r, 5), round(c, 6)) for i, r, c in rows if r > rel or (cos is not None and c < cos)]
    assert not bad, f"{what}: {len(bad)} of {len(rows)} samples outside rel-L2 {rel} / cosine {cos}: {bad}"
    return worst_r, worst_c
