"""Per-sample / per-frame views of the parity metrics (shared by the UNet, sampler and decoder parity tests), and the
judge of the block-isolated fp64 checks.

A whole-tensor rel-L2 over a CFG batch of 36 samples lets a mistake confined to one frame through: that frame is
under 3 % of the tensor.  These helpers apply the same bound to every leading-index slice on its own; `judge` applies
a per-block error budget to every part of a caller-given partition of one block's output."""
from __future__ import annotations

from typing import Callable, Dict, List, Optional, Tuple

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


# ---------------------------------------------------------------------------------------------------------------
# block-isolated fp64 checks (tests/test_unet_blocks_fp64_gpu.py, tests/test_first_stage_clip_blocks_fp64_gpu.py)
# ---------------------------------------------------------------------------------------------------------------
LOCALITY_FACTOR, LOCALITY_FLOOR = 2.0, 0.1


def judge(name: str, kind: str, x_in: torch.Tensor, ref: torch.Tensor, got: torch.Tensor, c: float,
          partition: Callable[[torch.Tensor], Dict[str, torch.Tensor]], bf16_out: bool = True) -> dict:
    """Budget and locality of one block; returns a record, prints the BLOCK line.

    For every part p the error must satisfy ||err_p|| <= c ||upd_p|| + ||rnd_p||, with err = got - ref,
    upd = ref - x_in when the block keeps its shape (ref otherwise) and rnd = bf16(ref) - ref (0 when the block stores
    fp32).  `partition(sq)` maps a tensor of squares shaped like `ref` to {partition name: 1-D tensor of per-part sums};
    the budget is the ratio of the whole block, and every part's ratio must stay within LOCALITY_FACTOR x that +
    LOCALITY_FLOOR (the floor absorbs the statistical spread of small parts)."""
    def sums(d):
        sq = d.square()
        return sq.sum(), partition(sq)

    e = sums(got - ref)
    u = sums(ref - x_in if x_in.shape == ref.shape else ref)
    r = sums(ref.to(torch.bfloat16).to(ref.dtype) - ref) if bf16_out else (ref.new_zeros(()), {
        k: torch.zeros_like(v) for k, v in e[1].items()})
    tot = torch.stack([e[0], u[0], r[0]])
    parts = {k: torch.stack([e[1][k], u[1][k], r[1][k]]) for k in e[1]}

    def ratio(s):                                                             # s: [3, ...] sums of squares
        s = s.sqrt()
        return s[0] / (c * s[1] + s[2]).clamp_min(1e-300)

    whole = float(ratio(tot))
    worst, local_bad = ("whole", 0, whole), []
    limit = LOCALITY_FACTOR * whole + LOCALITY_FLOOR
    for pname, s in parts.items():
        rp = ratio(s).cpu()
        i = int(rp.argmax())
        if float(rp[i]) > worst[2]:
            worst = (pname, i, float(rp[i]))
        local_bad += [(pname, j, round(float(rp[j]), 3)) for j in range(rp.numel()) if float(rp[j]) > limit]
    s = tot.sqrt()
    c_meas = float((s[0] - s[2]).clamp_min(0.0) / s[1].clamp_min(1e-300))
    print(f"BLOCK {name} kind={kind} ratio={whole:.3f} worst={worst[0]}:{worst[1]}:{worst[2]:.3f} c={c_meas:.3e}")
    return dict(name=name, kind=kind, ratio=whole, worst=worst, c=c_meas, local_bad=local_bad,
                finite=bool(torch.isfinite(got).all()))


def groups(s: torch.Tensor, g: int) -> torch.Tensor:
    """Sums over consecutive runs of g entries of a 1-D tensor (the last run may be short)."""
    n = s.numel()
    return torch.nn.functional.pad(s, (0, -n % g)).reshape(-1, g).sum(1)


def ring_interior(sq_hw: torch.Tensor) -> torch.Tensor:
    """[ring, interior] of a [H, W] map of sums: the one-pixel border vs the rest."""
    inner = sq_hw[1:-1, 1:-1].sum()
    return torch.stack([sq_hw.sum() - inner, inner])
