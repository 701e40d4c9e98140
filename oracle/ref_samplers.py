"""fp32 CPU restatement of the ancestral, DPM++ and linear-multistep samplers (TEST INFRASTRUCTURE).

EulerAncestralSampler, DPMPP2SAncestralSampler (sampling.py:136-173,240-287), DPMPP2MSampler (sampling.py:290-365),
LinearMultistepSampler (sampling.py:176-211) with the helpers of sampling_utils.py:7-43, around the denoiser / guider
restatements of oracle/ref_sampling.py.  The injected noise comes from an explicit `noise_fn(x)`, called once per step
(the last step included) exactly where the reference calls `self.noise_sampler(x)`.
"""
from __future__ import annotations

from typing import Callable, Dict

import torch
from scipy import integrate

from .ref_sampling import edm_sigmas, guider_combine, guider_prepare_inputs


def _bc(v: torch.Tensor, like: torch.Tensor) -> torch.Tensor:
    return v.reshape(-1, *([1] * (like.ndim - 1)))


def _start(x, num_steps: int, sigma_max: float):
    sigmas = edm_sigmas(num_steps, sigma_max=sigma_max)
    x = x * torch.sqrt(1.0 + sigmas[0] ** 2.0)
    return x, sigmas, x.new_ones([x.shape[0]])


def _guided(denoise_fn: Callable, cond: Dict, uc: Dict, scale: torch.Tensor, num_frames: int):
    return lambda xx, sig: guider_combine(denoise_fn(*guider_prepare_inputs(xx, sig, cond, uc)), scale, num_frames)


def ancestral_sigmas(sigma_from: torch.Tensor, sigma_to: torch.Tensor, eta: float):
    """sampling_utils.py:22-31 for eta > 0: (sigma_down, sigma_up)."""
    up = torch.minimum(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    return (sigma_to ** 2 - up ** 2) ** 0.5, up


def _add_noise(x, sigma_next, sigma_up, noise_fn, s_noise):
    """AncestralSampler.ancestral_step (sampling.py:150-156): the draw is made even where it is discarded."""
    return torch.where(_bc(sigma_next, x) > 0.0, x + noise_fn(x) * s_noise * _bc(sigma_up, x), x)


def euler_ancestral_sample(denoise_fn: Callable, x, cond: Dict, uc: Dict, num_steps: int, scale: torch.Tensor,
                           num_frames: int, noise_fn: Callable, eta: float = 1.0, s_noise: float = 1.0,
                           sigma_max: float = 700.0):
    x, sigmas, s_in = _start(x, num_steps, sigma_max)
    denoise = _guided(denoise_fn, cond, uc, scale, num_frames)
    for i in range(len(sigmas) - 1):
        sigma, nxt = s_in * sigmas[i], s_in * sigmas[i + 1]
        down, up = ancestral_sigmas(sigma, nxt, eta)
        d = (x - denoise(x, sigma)) / _bc(sigma, x)
        x = _add_noise(x + _bc(down - sigma, x) * d, nxt, up, noise_fn, s_noise)
    return x


def dpmpp2s_ancestral_sample(denoise_fn: Callable, x, cond: Dict, uc: Dict, num_steps: int, scale: torch.Tensor,
                             num_frames: int, noise_fn: Callable, eta: float = 1.0, s_noise: float = 1.0,
                             sigma_max: float = 700.0):
    x, sigmas, s_in = _start(x, num_steps, sigma_max)
    denoise = _guided(denoise_fn, cond, uc, scale, num_frames)
    for i in range(len(sigmas) - 1):
        sigma, nxt = s_in * sigmas[i], s_in * sigmas[i + 1]
        down, up = ancestral_sigmas(sigma, nxt, eta)
        den = denoise(x, sigma)
        x_euler = x + _bc(down - sigma, x) * ((x - den) / _bc(sigma, x))
        if torch.sum(down) < 1e-14:
            x_new = x_euler
        else:
            t, t_next = -sigma.log(), -down.log()
            h = t_next - t
            s = t + 0.5 * h
            x2 = _bc((-s).exp() / (-t).exp(), x) * x - _bc((-0.5 * h).expm1(), x) * den
            den2 = denoise(x2, (-s).exp())
            x_dpm = _bc((-t_next).exp() / (-t).exp(), x) * x - _bc((-h).expm1(), x) * den2
            x_new = torch.where(_bc(down, x) > 0.0, x_dpm, x_euler)
        x = _add_noise(x_new, nxt, up, noise_fn, s_noise)
    return x


def dpmpp2m_sample(denoise_fn: Callable, x, cond: Dict, uc: Dict, num_steps: int, scale: torch.Tensor,
                   num_frames: int, sigma_max: float = 700.0):
    x, sigmas, s_in = _start(x, num_steps, sigma_max)
    denoise = _guided(denoise_fn, cond, uc, scale, num_frames)
    old = None
    for i in range(len(sigmas) - 1):
        sigma, nxt = s_in * sigmas[i], s_in * sigmas[i + 1]
        den = denoise(x, sigma)
        t, t_next = -sigma.log(), -nxt.log()
        h = t_next - t
        m1, m2 = _bc((-t_next).exp() / (-t).exp(), x), _bc((-h).expm1(), x)
        x_std = m1 * x - m2 * den
        if old is None or torch.sum(nxt) < 1e-14:
            x_new = x_std
        else:
            r = (t - (-(s_in * sigmas[i - 1]).log())) / h
            den_d = _bc(1 + 1 / (2 * r), x) * den - _bc(1 / (2 * r), x) * old
            x_new = torch.where(_bc(nxt, x) > 0.0, m1 * x - m2 * den_d, x_std)
        x, old = x_new, den
    return x


def lms_coeff(order: int, t, i: int, j: int, epsrel: float = 1e-4) -> float:
    """linear_multistep_coeff (sampling_utils.py:7-19): quad over [t[i], t[i+1]] of the Lagrange basis polynomial of
    node i-j on nodes i, ..., i-order+1; with t the float32 numpy schedule the integrand is evaluated in float32."""
    assert order - 1 <= i

    def fn(tau):
        prod = 1.0
        for k in range(order):
            if k != j:
                prod *= (tau - t[i - k]) / (t[i - j] - t[i - k])
        return prod

    return integrate.quad(fn, t[i], t[i + 1], epsrel=epsrel)[0]


def lms_sample(denoise_fn: Callable, x, cond: Dict, uc: Dict, num_steps: int, scale: torch.Tensor, num_frames: int,
               order: int = 4, sigma_max: float = 700.0):
    x, sigmas, s_in = _start(x, num_steps, sigma_max)
    denoise = _guided(denoise_fn, cond, uc, scale, num_frames)
    t = sigmas.numpy()
    ds = []
    for i in range(len(sigmas) - 1):
        sigma = s_in * sigmas[i]
        ds = (ds + [(x - denoise(x, sigma)) / _bc(sigma, x)])[-order:]
        cur = min(i + 1, order)
        step = 0
        for j, d in enumerate(reversed(ds)):
            step = step + lms_coeff(cur, t, i, j) * d
        x = x + step
    return x
