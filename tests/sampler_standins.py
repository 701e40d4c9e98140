"""TEST INFRASTRUCTURE: torch stand-ins for the ancestral / DPM++ / LMS step kernels and CPU shims of their samplers.

Each stand-in restates one entry point of include/v3d_b200.h in fp32 torch, one operation per rounding in the kernel's
order, with every scalar held as a 0-dim tensor on the data's device (a python scalar would let CUDA torch divide by
multiplying with the reciprocal).  They are device-agnostic: tests/test_samplers_gpu.py holds them against the kernels
on the same CUDA tensors, tests/test_samplers_cpu.py runs the drop-in samplers on CPU through them.  `patched()`
installs them, together with tests/emu_ops.py, over `v3d_b200.ops`.
"""
from __future__ import annotations

import contextlib

import torch

import cpu_shims
import emu_ops
from v3d_b200 import ops as real_ops
from v3d_b200.sampling import (DPMPP2MSampler, DPMPP2SAncestralSampler, EulerAncestralSampler,
                               LinearMultistepSampler)


def _s(v: float, like: torch.Tensor) -> torch.Tensor:
    return torch.tensor(float(v), dtype=torch.float32, device=like.device)


def _with_noise(r, noise, s_noise, sigma_up, sigma_next):
    return r + (noise * _s(s_noise, r)) * _s(sigma_up, r) if sigma_next > 0 else r


def _euler(x, den, sigma, sigma_down):
    sg = _s(sigma, x)
    return x + (_s(sigma_down, x) - sg) * ((x - den) / sg)


def ancestral_euler_step(x, den, noise, out, sigma, sigma_down, sigma_up, sigma_next, s_noise, nsamples, per_sample):
    emu_ops._tick()
    out.copy_(_with_noise(_euler(x, den, sigma, sigma_down), noise, s_noise, sigma_up, sigma_next))
    return out


def dpmpp2s_stage(x, den, out, m1, m2, nsamples, per_sample):
    emu_ops._tick()
    out.copy_(_s(m1, x) * x - _s(m2, x) * den)
    return out


def dpmpp2s_step(x, den, den2, noise, out, sigma, sigma_down, sigma_up, sigma_next, s_noise, m3, m4, nsamples,
                 per_sample):
    emu_ops._tick()
    r = _s(m3, x) * x - _s(m4, x) * den2 if sigma_down > 0 else _euler(x, den, sigma, sigma_down)
    out.copy_(_with_noise(r, noise, s_noise, sigma_up, sigma_next))
    return out


def dpmpp2m_step(x, den, hist, out, m1, m2, m3, m4, second_order, nsamples, per_sample):
    emu_ops._tick()
    dd = _s(m3, x) * den - _s(m4, x) * hist if second_order else den
    r = _s(m1, x) * x - _s(m2, x) * dd
    hist.copy_(den)
    out.copy_(r)
    return out


def lms_step(x, den, ring, out, sigma, coeffs, slots, nsamples, per_sample):
    emu_ops._tick()
    assert 1 <= len(coeffs) <= 8 and len(coeffs) == len(slots) and ring.shape[0] >= len(coeffs)
    ring[slots[0]].copy_((x - den) / _s(sigma, x))
    acc = _s(coeffs[0], x) * ring[slots[0]]
    for c, k in zip(coeffs[1:], slots[1:]):
        acc = acc + _s(c, x) * ring[k]
    out.copy_(x + acc)
    return out


STANDINS = ["ancestral_euler_step", "dpmpp2s_stage", "dpmpp2s_step", "dpmpp2m_step", "lms_step"]


@contextlib.contextmanager
def patched():
    """emu_ops.patched() plus the stand-ins above on v3d_b200.ops."""
    saved = {n: getattr(real_ops, n) for n in STANDINS}
    with emu_ops.patched():
        try:
            for n in STANDINS:
                setattr(real_ops, n, globals()[n])
            yield
        finally:
            for n, f in saved.items():
                setattr(real_ops, n, f)


# the product samplers below their CUDA check (cpu_shims.py does the same for Euler / Heun)
class CpuEulerAncestral(EulerAncestralSampler):
    __call__ = EulerAncestralSampler._loop


class CpuDPMPP2SAncestral(DPMPP2SAncestralSampler):
    __call__ = DPMPP2SAncestralSampler._loop


class CpuDPMPP2M(DPMPP2MSampler):
    __call__ = DPMPP2MSampler._loop


class CpuLMS(LinearMultistepSampler):
    __call__ = LinearMultistepSampler._loop


CPU_SHIMS = {"EulerAncestralSampler": CpuEulerAncestral, "DPMPP2SAncestralSampler": CpuDPMPP2SAncestral,
             "DPMPP2MSampler": CpuDPMPP2M, "LinearMultistepSampler": CpuLMS}


def cpu_engine(sampler: str, num_frames: int, num_steps: int, **params):
    """cpu_shims.cpu_engine with its sampler replaced by the CPU shim of `sampler` (same schedule and guider)."""
    from v3d_b200 import engine

    eng, sd_u, sd_d = cpu_shims.cpu_engine(num_frames, num_steps)
    cfg = engine.v3d_512_config(num_frames=num_frames, num_steps=num_steps, min_cfg=1.5, max_cfg=3.5)
    eng.sampler = CPU_SHIMS[sampler](**cfg["sampler_config"]["params"], **params)
    return eng, sd_u, sd_d
