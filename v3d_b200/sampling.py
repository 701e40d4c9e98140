"""Sampling-side drop-ins for the sgm plugin surface (reference sgm/modules/diffusionmodules/):
`EDMDiscretization` (discretizer.py:18-39), `LinearPredictionGuider` (guiders.py:60-101),
`VScalingWithEDMcNoise` + `Denoiser` (denoiser_scaling.py:51-59, denoiser.py:12-39), `OpenAIWrapper`
(wrappers.py:9-34), `EulerEDMSampler` (sampling.py:24-133,214-218) and - SURVEY 8(f)-3, same denoiser, no new
tensor-core work - `HeunEDMSampler` (sampling.py:221-237), `VanillaCFG` (guiders.py:23-42) and
`CentralPredictionGuider` (guiders.py:104-146); `EulerAncestralSampler`, `DPMPP2SAncestralSampler`, `DPMPP2MSampler`,
`LinearMultistepSampler` (sampling.py:136-211,240-365) with the helpers of sampling_utils.py:7-43.

Call shapes are the reference's: `sampler(denoiser, x, cond=c, uc=uc) -> x`, `denoiser(network, input, sigma,
cond, **kw)`, `network(x, t, c, **kw)`; any denoiser closure works (scripts/pub/V3D_512.py:278-283).  The
per-step elementwise arithmetic runs in this package's own fp32 kernels (csrc/sampler.cu); the sigma schedule
lives on the host, so the loop has no device->host sync (the reference syncs once per step, sampling.py:118-122).
"""
from __future__ import annotations

import importlib
from typing import Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from . import ops


def get_obj_from_str(string: str):
    module, cls = string.rsplit(".", 1)
    return getattr(importlib.import_module(module, package=None), cls)


def instantiate_from_config(config):
    """Same contract as sgm.util.instantiate_from_config (sgm/util.py:170-187)."""
    if "target" not in config:
        raise KeyError("Expected key `target` to instantiate.")
    return get_obj_from_str(config["target"])(**config.get("params", dict()))


class EDMDiscretization:
    """Karras rho-schedule; `__call__` appends the final 0 (discretizer.py:18-39)."""

    def __init__(self, sigma_min: float = 0.002, sigma_max: float = 80.0, rho: float = 7.0):
        self.sigma_min, self.sigma_max, self.rho = sigma_min, sigma_max, rho

    def get_sigmas(self, n: int, device="cpu") -> torch.Tensor:
        # computed on the host in fp32 exactly like the reference's torch.linspace expression
        ramp = torch.linspace(0, 1, n, device="cpu")
        min_inv_rho = self.sigma_min ** (1 / self.rho)
        max_inv_rho = self.sigma_max ** (1 / self.rho)
        return ((max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** self.rho).to(device)

    def __call__(self, n: int, do_append_zero: bool = True, device="cpu", flip: bool = False) -> torch.Tensor:
        sigmas = self.get_sigmas(n, device=device)
        if do_append_zero:
            sigmas = torch.cat([sigmas, sigmas.new_zeros([1])])
        return sigmas if not flip else torch.flip(sigmas, (0,))


class _FrameScaleGuider:
    """Shared machinery of the classifier-free guiders: batch order [uc; c], `x_u + scale_t (x_c - x_u)` with one
    scale per frame of a video (`self.scale`, shape [1, T]); the combine runs in v3d_cfg_combine."""

    additional_cond_keys: List[str] = []
    num_frames: int = 1

    def _init_keys(self, additional_cond_keys) -> None:
        if additional_cond_keys is None:
            additional_cond_keys = []
        if isinstance(additional_cond_keys, str):
            additional_cond_keys = [additional_cond_keys]
        self.additional_cond_keys = additional_cond_keys
        self._scale_dev: Optional[Tuple[torch.Tensor, torch.Tensor]] = None

    def _scale_on(self, device) -> torch.Tensor:
        # `self.scale` may be re-assigned by callers (scripts/pub/V3D_512.py:84-100); re-upload only when it changes
        # (re-assignment or an in-place edit such as `guider.scale[:, i] = ...`: the tensor's version counter moves)
        scale = self._scale_tensor()
        tag = (id(scale), scale._version)
        if self._scale_dev is None or self._scale_dev[0] != tag or self._scale_dev[1].device != device:
            self._scale_dev = (tag, scale.reshape(-1).float().to(device).contiguous())
        return self._scale_dev[1]

    def _scale_tensor(self) -> torch.Tensor:
        return self.scale

    def __call__(self, x: torch.Tensor, sigma: torch.Tensor) -> torch.Tensor:
        T = self.num_frames
        n2 = x.shape[0]
        assert n2 % (2 * T) == 0, "guider expects [uc; c] halves of whole videos"
        half = n2 // 2
        per = x[0].numel()
        x = x.float().contiguous()
        out = torch.empty((half,) + tuple(x.shape[1:]), device=x.device, dtype=torch.float32)
        ops.cfg_combine(x, self._scale_on(x.device), out, half // T, T, per)
        return out

    def prepare_inputs(self, x: torch.Tensor, s: torch.Tensor, c: dict, uc: dict):
        c_out = dict()
        for k in c:
            if k in ["vector", "crossattn", "concat"] + self.additional_cond_keys:
                c_out[k] = torch.cat((uc[k], c[k]), 0)
            else:
                if k == "rgb":
                    continue
                assert c[k] == uc[k]
                c_out[k] = c[k]
        return torch.cat([x] * 2), torch.cat([s] * 2), c_out


class LinearPredictionGuider(_FrameScaleGuider):
    """Per-frame CFG scale linspace(min, max, T); batch order [uc; c] (guiders.py:60-101)."""

    def __init__(self, max_scale: float, num_frames: int, min_scale: float = 1.0,
                 additional_cond_keys: Optional[Union[List[str], str]] = None):
        self.min_scale, self.max_scale, self.num_frames = min_scale, max_scale, num_frames
        self.scale = torch.linspace(min_scale, max_scale, num_frames, device="cpu").unsqueeze(0)
        self._init_keys(additional_cond_keys)


class CentralPredictionGuider(_FrameScaleGuider):
    """Triangular per-frame scale: linspace(min, 2 max, T) mirrored about the middle frame (guiders.py:104-146)."""

    def __init__(self, max_scale: float, num_frames: int, min_scale: float = 1.0,
                 additional_cond_keys: Optional[Union[List[str], str]] = None):
        self.min_scale, self.max_scale, self.num_frames = min_scale, max_scale, num_frames
        scale = torch.linspace(min_scale, 2 * max_scale, num_frames, device="cpu")
        scale[num_frames // 2:] = 2 * max_scale - scale[num_frames // 2:]
        self.scale = scale.unsqueeze(0)
        self._init_keys(additional_cond_keys)


class VanillaCFG(_FrameScaleGuider):
    """One scale for every sample: `x_u + scale (x_c - x_u)` (guiders.py:23-42)."""

    def __init__(self, scale: float):
        self.num_frames = 1
        self.scale_value = float(scale)
        self._init_keys(None)

    # the reference keeps a python float in `.scale` (guiders.py:24-25) and so does the attribute here; the [1, 1]
    # tensor the combine kernel reads is derived from it
    @property
    def scale(self) -> float:
        return float(self._scale_t.reshape(-1)[0])

    def _scale_tensor(self) -> torch.Tensor:
        return self._scale_t

    @scale.setter
    def scale(self, v):
        self._scale_t = v if isinstance(v, torch.Tensor) else torch.tensor([[float(v)]])

    @property
    def scale_value(self) -> float:
        return float(self._scale_t.reshape(-1)[0])

    @scale_value.setter
    def scale_value(self, v: float) -> None:
        self.scale = v


class VScalingWithEDMcNoise:
    """c_skip, c_out, c_in, c_noise of denoiser_scaling.py:51-59 (kept for API parity; the Denoiser below
    evaluates the same expressions inside its fused kernels)."""

    def __call__(self, sigma: torch.Tensor):
        c_skip = 1.0 / (sigma ** 2 + 1.0)
        c_out = -sigma / (sigma ** 2 + 1.0) ** 0.5
        c_in = 1.0 / (sigma ** 2 + 1.0) ** 0.5
        c_noise = 0.25 * sigma.log()
        return c_skip, c_out, c_in, c_noise


class Denoiser(nn.Module):
    """`network(input * c_in, c_noise, cond) * c_out + input * c_skip` (denoiser.py:23-39)."""

    def __init__(self, scaling_config: Dict):
        super().__init__()
        self.scaling = instantiate_from_config(scaling_config)
        if not isinstance(self.scaling, VScalingWithEDMcNoise):
            raise NotImplementedError("only VScalingWithEDMcNoise is implemented on the native path")

    def possibly_quantize_sigma(self, sigma: torch.Tensor) -> torch.Tensor:
        return sigma

    def possibly_quantize_c_noise(self, c_noise: torch.Tensor) -> torch.Tensor:
        return c_noise

    def forward(self, network: nn.Module, input: torch.Tensor, sigma: torch.Tensor, cond: Dict,
                **additional_model_inputs) -> torch.Tensor:
        sigma = self.possibly_quantize_sigma(sigma).float().contiguous()
        x = input.float().contiguous()
        n = x.shape[0]
        per = x[0].numel()
        assert sigma.numel() == n
        scaled = torch.empty_like(x)
        c_noise = torch.empty(n, device=x.device, dtype=torch.float32)
        ops.edm_scale_input(x, sigma, scaled, c_noise, n, per)
        c_noise = self.possibly_quantize_c_noise(c_noise.reshape(sigma.shape))
        net = network(scaled, c_noise, cond, **additional_model_inputs).float().contiguous()
        out = torch.empty_like(x)
        ops.edm_denoise_combine(net, x, sigma, out, n, per)
        return out


class IdentityWrapper(nn.Module):
    def __init__(self, diffusion_model, compile_model: bool = False):
        super().__init__()
        # compile_model is accepted and ignored: the network is already a fixed schedule of native kernels
        self.diffusion_model = diffusion_model

    def forward(self, *args, **kwargs):
        return self.diffusion_model(*args, **kwargs)


class OpenAIWrapper(IdentityWrapper):
    """wrappers.py:23-34: x = cat(x, c['concat']); context <- crossattn; y <- vector."""

    def forward(self, x: torch.Tensor, t: torch.Tensor, c: dict, **kwargs) -> torch.Tensor:
        if "concat" in c:
            x = torch.cat((x, c["concat"].type_as(x)), dim=1)
        return self.diffusion_model(x, timesteps=t, context=c.get("crossattn", None), y=c.get("vector", None),
                                    **kwargs)


DEFAULT_GUIDER = {"target": "v3d_b200.sampling.IdentityGuider"}


class IdentityGuider:
    def __call__(self, x, sigma):
        return x

    def prepare_inputs(self, x, s, c, uc):
        return x, s, {k: c[k] for k in c}


# ---------------------------------------------------------------------------------------------------------------------
# sampling_utils.py:7-43 (also exported at v3d_b200.sgm.modules.diffusionmodules.sampling_utils)
# ---------------------------------------------------------------------------------------------------------------------
def _append_dims(v: torch.Tensor, ndim: int) -> torch.Tensor:
    if v.ndim > ndim:
        raise ValueError(f"input has {v.ndim} dims but target_dims is {ndim}, which is less")
    return v.reshape(tuple(v.shape) + (1,) * (ndim - v.ndim))


def linear_multistep_coeff(order: int, t, i: int, j: int, epsrel: float = 1e-4) -> float:
    """Integral over [t[i], t[i+1]] of the Lagrange basis polynomial of node t[i-j] on the nodes t[i], ..., t[i-order+1]
    (sampling_utils.py:7-19).  `t` is the float32 numpy schedule, as the reference passes it: the integrand then runs in
    float32 and the adaptive quadrature sees exactly the reference's values."""
    from scipy import integrate

    if order - 1 > i:
        raise ValueError(f"Order {order} too high for step {i}")
    nodes = [k for k in range(order) if k != j]

    def basis(tau):
        prod = 1.0
        for k in nodes:
            prod *= (tau - t[i - k]) / (t[i - j] - t[i - k])
        return prod

    return integrate.quad(basis, t[i], t[i + 1], epsrel=epsrel)[0]


def get_ancestral_step(sigma_from: torch.Tensor, sigma_to: torch.Tensor, eta: float = 1.0):
    """(sigma_down, sigma_up) of an ancestral step with noise fraction eta (sampling_utils.py:22-31)."""
    if not eta:
        return sigma_to, 0.0
    sigma_up = torch.minimum(sigma_to, eta * (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5)
    sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
    return sigma_down, sigma_up


def to_d(x: torch.Tensor, sigma: torch.Tensor, denoised: torch.Tensor) -> torch.Tensor:
    return (x - denoised) / _append_dims(sigma, x.ndim)


def to_neg_log_sigma(sigma: torch.Tensor) -> torch.Tensor:
    return sigma.log().neg()


def to_sigma(neg_log_sigma: torch.Tensor) -> torch.Tensor:
    return neg_log_sigma.neg().exp()


# ---------------------------------------------------------------------------------------------------------------------
# Ancestral, DPM++ and linear-multistep samplers (sampling.py:136-211,240-365)
# ---------------------------------------------------------------------------------------------------------------------
LMS_MAX_ORDER = 8  # V3D_LMS_MAX_ORDER of include/v3d_b200.h


def _f32(v: float) -> torch.Tensor:
    """One schedule value as the fp32 tensor the reference computes its multipliers with (every sample of a step shares
    the step's sigma, so one element stands for the reference's `s_in * sigmas[i]`)."""
    return torch.tensor([v], dtype=torch.float32)


def _sigma_rows(values: List[float], n: int, device) -> torch.Tensor:
    """[len(values), n] fp32 per-sample sigma rows for the denoiser, uploaded once per call from pinned memory without a
    host sync."""
    rows = torch.tensor(values, dtype=torch.float32).reshape(-1, 1).expand(len(values), n).contiguous()
    if torch.device(device).type == "cuda":
        return rows.pin_memory().to(device, non_blocking=True)
    return rows


class _ScheduleSampler:
    """BaseDiffusionSampler (sampling.py:24-74) for the samplers below: the sigma schedule and every multiplier derived
    from it live on the host (computed in fp32 with the reference's expressions), the state, the denoised estimates and
    the sampler history on the device; each step's arithmetic is one native kernel (csrc/sampler.cu)."""

    def __init__(self, discretization_config, num_steps: Optional[int] = None, guider_config=None,
                 verbose: bool = False, device: str = "cuda"):
        self.num_steps = num_steps
        self.discretization = instantiate_from_config(discretization_config)
        self.guider = instantiate_from_config(guider_config if guider_config is not None else DEFAULT_GUIDER)
        self.verbose = verbose
        self.device = device

    def prepare_sampling_loop(self, x, cond, uc=None, num_steps=None):
        sigmas = self.discretization(self.num_steps if num_steps is None else num_steps, device="cpu")
        uc = cond if uc is None else uc
        x *= float(torch.sqrt(1.0 + sigmas[0] ** 2.0))  # in place on the caller's noise, like sampling.py:50
        return x, sigmas, len(sigmas), cond, uc

    def denoise(self, x, denoiser, sigma, cond, uc, **kwargs):
        denoised = denoiser(*self.guider.prepare_inputs(x, sigma, cond, uc), **kwargs)
        return self.guider(denoised, sigma).float().contiguous()

    def _steps(self, num_sigmas: int):
        steps = range(num_sigmas - 1)
        if self.verbose:
            from tqdm import tqdm

            steps = tqdm(steps, total=num_sigmas - 1, desc=f"Sampling with {type(self).__name__}")
        return steps

    def __call__(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        ops.require_current_device(x, f"v3d_b200.{type(self).__name__}")
        return self._loop(denoiser, x, cond, uc, num_steps, **kwargs)

    def _start(self, x, cond, uc, num_steps):
        assert x.dtype == torch.float32, "sampler state is fp32 (denoiser.py:36-39)"
        x, sigmas, num_sigmas, cond, uc = self.prepare_sampling_loop(x, cond, uc, num_steps)
        return x.contiguous(), sigmas.float(), num_sigmas, cond, uc


class EulerEDMSampler(_ScheduleSampler):
    """EDM Euler sampler (sampling.py:24-133,214-218). s_churn > 0 (noise injection) keeps the reference
    semantics via torch.randn_like; V3D_512 runs with s_churn = 0."""

    def __init__(self, discretization_config, num_steps: Optional[int] = None, guider_config=None,
                 verbose: bool = False, device: str = "cuda", s_churn: float = 0.0, s_tmin: float = 0.0,
                 s_tmax: float = float("inf"), s_noise: float = 1.0):
        super().__init__(discretization_config, num_steps, guider_config, verbose, device)
        self.s_churn, self.s_tmin, self.s_tmax, self.s_noise = s_churn, s_tmin, s_tmax, s_noise

    def possible_correction_step(self, euler_step, x, d, dt, next_sigma, denoiser, cond, uc):
        return euler_step

    def _churn(self, x, sigma, gamma: float):
        """-> (x, sigma_hat): the state with the churn noise added and the raised sigma (sampling.py:97-101)."""
        sigma_hat = sigma if gamma == 0 else sigma * (gamma + 1.0)
        if gamma > 0:
            eps = torch.randn_like(x) * self.s_noise
            x = x + eps * (sigma_hat ** 2 - sigma ** 2).reshape(-1, *([1] * (x.ndim - 1))) ** 0.5
        return x, sigma_hat

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, gamma: float = 0.0):
        x, sigma_hat = self._churn(x, sigma, gamma)
        denoised = self.denoise(x, denoiser, sigma_hat, cond, uc)
        out = torch.empty_like(x)
        ops.euler_step(x, denoised, sigma_hat, next_sigma, out, x.shape[0], x[0].numel())
        return out

    def _loop(self, denoiser, x, cond, uc=None, num_steps=None):
        """EDMSampler.__call__ (sampling.py:112-133)."""
        x, sigmas, num_sigmas, cond, uc = self._start(x, cond, uc, num_steps)
        n = x.shape[0]
        host = [float(s) for s in sigmas]
        rows = _sigma_rows(host, n, x.device)
        for i in self._steps(num_sigmas):
            gamma = min(self.s_churn / (num_sigmas - 1), 2 ** 0.5 - 1) if self.s_tmin <= host[i] <= self.s_tmax else 0.0
            x = self._step(host[i + 1] * n, rows[i], rows[i + 1], denoiser, x, cond, uc, gamma)
        return x

    def _step(self, next_sigma_sum: float, *step_args):
        return self.sampler_step(*step_args)


class HeunEDMSampler(EulerEDMSampler):
    """Second-order EDM sampler (sampling.py:221-237): after the Euler proposal the denoiser is evaluated once more at
    sigma_next and the step is redone with the averaged slope; the last step (sigma_next = 0) stays first order, which
    also saves the network evaluation exactly as the reference does (`torch.sum(next_sigma) < 1e-14`)."""

    _next_sigma_host: Optional[float] = None  # set by _step: lets the step skip the device->host sync

    def sampler_step(self, sigma, next_sigma, denoiser, x, cond, uc=None, gamma: float = 0.0):
        x, sigma_hat = self._churn(x, sigma, gamma)
        n, per = x.shape[0], x[0].numel()
        denoised = self.denoise(x, denoiser, sigma_hat, cond, uc)
        x_euler = torch.empty_like(x)
        ops.euler_step(x, denoised, sigma_hat, next_sigma, x_euler, n, per)
        nsum = self._next_sigma_host if self._next_sigma_host is not None else float(next_sigma.sum())
        if nsum < 1e-14:
            return x_euler
        denoised2 = self.denoise(x_euler, denoiser, next_sigma, cond, uc)
        out = torch.empty_like(x)
        ops.heun_step(x, denoised, x_euler, denoised2, sigma_hat.float().contiguous(),
                      next_sigma.float().contiguous(), out, n, per)
        return out

    def _step(self, next_sigma_sum: float, *step_args):
        self._next_sigma_host = next_sigma_sum
        try:
            return self.sampler_step(*step_args)
        finally:
            self._next_sigma_host = None


class _AncestralSampler(_ScheduleSampler):
    """AncestralSampler (sampling.py:136-173).  `noise_sampler(x)` is called once per step with the current state,
    the last step included (where ancestral_step discards the draw because sigma_next = 0), so a caller who replaces it
    or seeds torch's generator gets the reference's draws in the reference's order.

    eta = 0 is refused: the reference fails at the first step there (get_ancestral_step returns the python float 0.0
    as sigma_up and append_dims cannot take it, sampling_utils.py:24, util.py:194-201)."""

    def __init__(self, eta: float = 1.0, s_noise: float = 1.0, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.eta = eta
        self.s_noise = s_noise
        self.noise_sampler = lambda x: torch.randn_like(x)
        self._check_eta()

    def _check_eta(self) -> None:
        if not self.eta:
            raise ValueError(f"{type(self).__name__}: eta = 0 is not supported (the reference sampler fails on it); "
                             "use eta > 0, or DPMPP2MSampler / EulerEDMSampler for deterministic sampling")

    def _ancestral(self, sigma: float, sigma_next: float):
        sigma_down, sigma_up = get_ancestral_step(_f32(sigma), _f32(sigma_next), eta=self.eta)
        return sigma_down, sigma_up

    def _noise(self, x: torch.Tensor) -> torch.Tensor:
        noise = self.noise_sampler(x)
        if tuple(noise.shape) != tuple(x.shape) or noise.device != x.device:
            raise RuntimeError(f"noise_sampler returned {tuple(noise.shape)} on {noise.device}; expected "
                               f"{tuple(x.shape)} on {x.device}")
        return noise.float().contiguous()


class EulerAncestralSampler(_AncestralSampler):
    """sampling.py:240-247: one network evaluation per step; v3d_ancestral_euler_step does the Euler step to
    sigma_down and adds the sigma_up noise."""

    def _loop(self, denoiser, x, cond, uc=None, num_steps=None):
        self._check_eta()
        x, sigmas, num_sigmas, cond, uc = self._start(x, cond, uc, num_steps)
        n, per = x.shape[0], x[0].numel()
        host = [float(s) for s in sigmas]
        rows = _sigma_rows(host, n, x.device)
        out = torch.empty_like(x)          # the caller's (scaled) noise is not overwritten, like the reference
        for i in self._steps(num_sigmas):
            sigma_down, sigma_up = self._ancestral(host[i], host[i + 1])
            den = self.denoise(x, denoiser, rows[i], cond, uc)
            ops.ancestral_euler_step(x, den, self._noise(x), out, host[i], float(sigma_down), float(sigma_up),
                                     host[i + 1], self.s_noise, n, per)
            x = out
        return x


class DPMPP2SAncestralSampler(_AncestralSampler):
    """sampling.py:250-287: a midpoint evaluation at sigma(s) = sqrt(sigma * sigma_down) and the second-order update,
    except where every sigma_down is 0 (the last step), which takes the ancestral Euler step instead and saves the
    evaluation: 2N - 1 network evaluations for N steps."""

    def _loop(self, denoiser, x, cond, uc=None, num_steps=None):
        self._check_eta()
        x, sigmas, num_sigmas, cond, uc = self._start(x, cond, uc, num_steps)
        n, per = x.shape[0], x[0].numel()
        host = [float(s) for s in sigmas]
        plan, mid_sigmas = [], []
        for i in range(num_sigmas - 1):
            sigma_down, sigma_up = self._ancestral(host[i], host[i + 1])
            step = {"down": float(sigma_down), "up": float(sigma_up), "mid": None}
            if float(sigma_down) * n >= 1e-14:          # torch.sum(sigma_down) < 1e-14 skips the midpoint
                t, t_next = to_neg_log_sigma(_f32(host[i])), to_neg_log_sigma(sigma_down)
                h = t_next - t
                s = t + 0.5 * h
                step.update(mid=len(mid_sigmas), m1=float(to_sigma(s) / to_sigma(t)), m2=float((-0.5 * h).expm1()),
                            m3=float(to_sigma(t_next) / to_sigma(t)), m4=float((-h).expm1()))
                mid_sigmas.append(float(to_sigma(s)))
            plan.append(step)
        rows = _sigma_rows(host[:-1] + mid_sigmas, n, x.device)
        out, x2 = torch.empty_like(x), torch.empty_like(x)
        for i in self._steps(num_sigmas):
            p = plan[i]
            den = self.denoise(x, denoiser, rows[i], cond, uc)
            if p["mid"] is None:
                ops.ancestral_euler_step(x, den, self._noise(x), out, host[i], p["down"], p["up"], host[i + 1],
                                         self.s_noise, n, per)
            else:
                ops.dpmpp2s_stage(x, den, x2, p["m1"], p["m2"], n, per)
                den2 = self.denoise(x2, denoiser, rows[num_sigmas - 1 + p["mid"]], cond, uc)
                ops.dpmpp2s_step(x, den, den2, self._noise(x), out, host[i], p["down"], p["up"], host[i + 1],
                                 self.s_noise, p["m3"], p["m4"], n, per)
            x = out
        return x


class DPMPP2MSampler(_ScheduleSampler):
    """sampling.py:290-365: one network evaluation per step; the previous denoised estimate stays on the device
    (v3d_dpmpp2m_step reads it and stores the new one).  The first step and a step to sigma_next = 0 are first order."""

    def _loop(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        # extra keyword arguments are accepted and ignored, as by the reference's __call__ (sampling.py:347)
        x, sigmas, num_sigmas, cond, uc = self._start(x, cond, uc, num_steps)
        n, per = x.shape[0], x[0].numel()
        host = [float(s) for s in sigmas]
        rows = _sigma_rows(host, n, x.device)
        out, old_denoised = torch.empty_like(x), torch.empty_like(x)
        for i in self._steps(num_sigmas):
            t, t_next = to_neg_log_sigma(_f32(host[i])), to_neg_log_sigma(_f32(host[i + 1]))
            h = t_next - t
            m1, m2 = float(to_sigma(t_next) / to_sigma(t)), float((-h).expm1())
            m3 = m4 = 0.0
            second_order = i > 0 and host[i + 1] * n >= 1e-14
            if second_order:
                r = (t - to_neg_log_sigma(_f32(host[i - 1]))) / h
                m3, m4 = float(1 + 1 / (2 * r)), float(1 / (2 * r))
            den = self.denoise(x, denoiser, rows[i], cond, uc)
            ops.dpmpp2m_step(x, den, old_denoised, out, m1, m2, m3, m4, second_order, n, per)
            x = out
        return x


class LinearMultistepSampler(_ScheduleSampler):
    """sampling.py:176-211: one network evaluation per step; the last `order` slopes d = (x - D) / sigma live in a
    device ring and the linear_multistep_coeff weights are integrated on the host once per call.  order is at most
    LMS_MAX_ORDER (8)."""

    def __init__(self, order: int = 4, *args, **kwargs):
        super().__init__(*args, **kwargs)
        if not 1 <= int(order) <= LMS_MAX_ORDER:
            raise ValueError(f"LinearMultistepSampler: order {order} is outside 1..{LMS_MAX_ORDER}")
        self.order = int(order)

    def _loop(self, denoiser, x, cond, uc=None, num_steps=None, **kwargs):
        if not 1 <= int(self.order) <= LMS_MAX_ORDER:
            raise ValueError(f"LinearMultistepSampler: order {self.order} is outside 1..{LMS_MAX_ORDER}")
        order = int(self.order)
        x, sigmas, num_sigmas, cond, uc = self._start(x, cond, uc, num_steps)
        n, per = x.shape[0], x[0].numel()
        host = [float(s) for s in sigmas]
        sigmas_np = sigmas.numpy()
        coeffs = []
        for i in range(num_sigmas - 1):
            cur = min(i + 1, order)
            coeffs.append([linear_multistep_coeff(cur, sigmas_np, i, j) for j in range(cur)])
        rows = _sigma_rows(host, n, x.device)
        out = torch.empty_like(x)
        ring = torch.empty((order,) + tuple(x.shape), device=x.device, dtype=torch.float32)
        for i in self._steps(num_sigmas):
            den = self.denoise(x, denoiser, rows[i], cond, uc, **kwargs)
            slots = [(i - j) % order for j in range(len(coeffs[i]))]
            ops.lms_step(x, den, ring, out, host[i], coeffs[i], slots, n, per)
            x = out
        return x

