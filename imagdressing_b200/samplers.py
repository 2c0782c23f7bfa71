"""Multistep samplers with the diffusers-0.24 surface (the `scheduler` the reference pipelines accept besides DDIM,
dressing_sd/pipelines/IMAGDressing_v1_pipeline*.py:2-32): DPMSolverMultistepScheduler (dpmsolver++, order 1 / 2,
midpoint), EulerDiscreteScheduler, EulerAncestralDiscreteScheduler and UniPCMultistepScheduler (bh1 / bh2, orders 1-3).

Each update is linear in the latents x, the CFG-combined model output eps, one history tensor H (the previous step's
data prediction) and one noise tensor z. A scheduler therefore only computes, on the host, a per-step row
{dx, de, cx, ce, ch, cz} (include/imagd_b200.h, `imagd_cfg_sampler_step`):
    D = dx x + de eps ;  x' = cx x + ce eps + ch H + cz z ;  H <- D
and the fused kernel applies it. UniPC's corrector rewrites the current sample from the previous corrected sample and up
to three previous data predictions, so it runs on a second kernel (`imagd_cfg_sampler_pc_step`) over a bank of four
latents-sized slots, from a 16-wide row (UniPCMultistepScheduler). Options that change the FORM of an update (DPM order
3, SDE / dpmsolver algorithm types, s_churn > 0, non-epsilon prediction, thresholding, UniPC predict_x0=False /
solver_p) raise NotImplementedError; options that only change the tables (timestep_spacing, steps_offset, beta
schedule, Karras sigmas) are implemented.

Line references are to diffusers-0.24.0 src/diffusers/schedulers/scheduling_{dpmsolver_multistep,euler_discrete,
euler_ancestral_discrete,unipc_multistep}.py. diffusers is not a dependency, so parity with it is restated here and
anchored by identities in tests/test_samplers_cpu.py and tests/test_unipc_cpu.py (DESIGN.md §4).
"""
from __future__ import annotations

import math
from typing import NamedTuple, Optional

import numpy as np
import torch

from . import ops
from .modeling import FrozenConfig


class SchedulerOutput:
    def __init__(self, prev_sample, pred_original_sample=None):
        self.prev_sample = prev_sample
        self.pred_original_sample = pred_original_sample


class SamplerTables(NamedTuple):
    """Device tables of one (sliced) schedule, S rows. `t`: fp32 timesteps (the UNet's time embedding); `scale`: fp32
    model-input scale or None (identity); `coef`: fp32 [S, 6] update rows ([S, 16] predictor-corrector rows when
    `predictor_corrector`); `blend`: fp32 [S, 2] inpaint add_noise coefficients at t_{i+1} (last row {1, 0});
    `history` / `noise`: whether the update reads H / z; `predictor_corrector`: the rows are for
    imagd_cfg_sampler_pc_step and its slot bank."""
    t: torch.Tensor
    scale: Optional[torch.Tensor]
    coef: torch.Tensor
    blend: torch.Tensor
    history: bool
    noise: bool
    predictor_corrector: bool = False


def _alphas_cumprod(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas) -> torch.Tensor:
    """betas as every diffusers-0.24 scheduler builds them (fp32 torch), then cumprod(1 - beta)."""
    if trained_betas is not None:
        betas = torch.tensor(trained_betas, dtype=torch.float32)
    elif beta_schedule == "linear":
        betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    elif beta_schedule == "scaled_linear":
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    elif beta_schedule == "squaredcos_cap_v2":
        ab = lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2
        betas = torch.tensor([min(1 - ab((i + 1) / num_train_timesteps) / ab(i / num_train_timesteps), 0.999)
                              for i in range(num_train_timesteps)], dtype=torch.float32)
    else:
        raise NotImplementedError(beta_schedule)
    return torch.cumprod(1.0 - betas, dim=0)


def _karras(in_sigmas: np.ndarray, n: int) -> np.ndarray:
    """_convert_to_karras (rho = 7) between in_sigmas[-1] (min) and in_sigmas[0] (max)."""
    sigma_min, sigma_max = float(in_sigmas[-1]), float(in_sigmas[0])
    rho = 7.0
    ramp = np.linspace(0, 1, n)
    min_inv, max_inv = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return (max_inv + ramp * (min_inv - max_inv)) ** rho


def _sigma_to_t(sigma: np.ndarray, log_sigmas: np.ndarray) -> np.ndarray:
    """_sigma_to_t: piecewise-linear inverse of log sigma(t) over the training timesteps (fractional t)."""
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    return ((1 - w) * low_idx + w * high_idx).reshape(sigma.shape)


def _spaced(spacing: str, T: int, n: int, steps_offset: int, extra: int) -> np.ndarray:
    """The float timesteps of `timestep_spacing` before any rounding / dtype cast. `extra` = 1 for DPM-Solver, which
    spaces n + 1 points and drops the last (dpmsolver_multistep.py:255-275); 0 for Euler (euler_discrete.py:232-250).
    Neither is DDIM's formula: DDIM `linspace` spaces n points over [0, T-1] and rounds."""
    if spacing == "linspace":
        ts = np.linspace(0, T - 1, n + extra).round()[::-1][: n].copy()
    elif spacing == "leading":
        ratio = T // (n + extra)
        ts = (np.arange(0, n + extra) * ratio).round()[::-1][: n].copy() + steps_offset
    elif spacing == "trailing":
        ratio = T / n
        ts = np.arange(T, 0, -ratio).round().copy() - 1
    else:
        raise ValueError(f"timestep_spacing {spacing!r}")
    return ts


class _SamplerBase:
    """Shared surface: config / from_config, the cached device tables, step-index bookkeeping."""

    order = 1
    _needs_noise = False
    _predictor_corrector = False

    def _finish(self, **config):
        self.config = FrozenConfig(**config)
        self.alphas_cumprod = _alphas_cumprod(config["num_train_timesteps"], config["beta_start"], config["beta_end"],
                                              config["beta_schedule"], config.get("trained_betas"))
        self.num_inference_steps = None
        self._step_index = None
        self._dev = {}

    @classmethod
    def from_config(cls, config, **kw):
        """Foreign keys are dropped, so `X.from_config(ddim.config)` works and inherits timestep_spacing / steps_offset."""
        return cls(**{**{k: v for k, v in dict(config).items() if k in cls.__init__.__code__.co_varnames}, **kw})

    @property
    def step_index(self):
        return self._step_index

    def _init_step_index(self, timestep):
        """_init_step_index: the position of `timestep` in the schedule (the second match when it repeats)."""
        t = timestep.to(self.timesteps.device) if torch.is_tensor(timestep) else timestep
        idx = (self.timesteps == t).nonzero()
        if len(idx) == 0:
            self._step_index = len(self.timesteps) - 1
        else:
            self._step_index = int(idx[1 if len(idx) > 1 else 0])

    def _slice_start(self, timesteps) -> int:
        """Index in the full schedule of the first row of `timesteps`, which must be a suffix of it (inpainting with
        strength < 1 samples timesteps[t_start:]). Its rows are the matching rows of the full schedule."""
        full = self.timesteps.detach().cpu()
        ts = timesteps.detach().cpu()
        k = full.numel() - ts.numel()
        if k < 0 or not torch.equal(full[k:].to(ts.dtype), ts):
            raise ValueError("timesteps must be a suffix of the schedule set by set_timesteps")
        return k

    def sampler_tables(self, device, timesteps: Optional[torch.Tensor] = None) -> SamplerTables:
        """Device tables for `timesteps` (default: the whole schedule), cached per (device, timesteps) so their
        addresses stay fixed for a captured step graph."""
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        ts = self.timesteps if timesteps is None else timesteps
        key = (str(device), tuple(float(t) for t in self.timesteps), tuple(float(t) for t in ts))
        hit = self._dev.get(key)
        if hit is None:
            k = self._slice_start(ts)
            S = ts.numel()
            rows = [self._row(k + j, j) for j in range(S)]
            blend = [self._blend_row(k + j) if k + j + 1 < len(self.timesteps) else [1.0, 0.0] for j in range(S)]
            f32 = dict(dtype=torch.float32, device=device)
            scale = self._scale_rows(k, S)
            hit = SamplerTables(torch.tensor([float(t) for t in ts], **f32),
                                None if scale is None else torch.tensor(scale, **f32), torch.tensor(rows, **f32),
                                torch.tensor(blend, **f32), self._uses_history(), self._needs_noise,
                                self._predictor_corrector)
            self._dev[key] = hit
        return hit

    def _scale_rows(self, k, S):
        return None

    def _uses_history(self) -> bool:
        return False

    def _run_row(self, row, model_output, sample, history=None, step_noise=None):
        """Host step through the fused kernel with a one-row table (like DDIMScheduler.step)."""
        x = sample.float().contiguous()
        out = x.clone()
        coef = torch.tensor([row], dtype=torch.float32, device=x.device)
        step = torch.zeros(2, dtype=torch.int32, device=x.device)
        ops.cfg_sampler_step(model_output.float().contiguous(), None, 1.0, out, coef, step, history=history,
                             step_noise=step_noise)
        return out.to(sample.dtype)


# ====================================================================================================== DPM-Solver++
class _VPSampler(_SamplerBase):
    """What DPM-Solver++ and UniPC share: DPM-Solver's schedule (below), the VP inpaint blend rows, the identity
    scale_model_input and add_noise on alphas_cumprod."""

    def _set_vp_schedule(self, num_inference_steps: int, device):
        T = self.config.num_train_timesteps
        ts = _spaced(self.config.timestep_spacing, T, num_inference_steps, self.config.steps_offset, 1).astype(np.int64)
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        if self.config.use_karras_sigmas:
            log_sigmas = np.log(sig)
            sigmas = _karras(np.flip(sig).copy(), num_inference_steps)
            ts = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas]).round().astype(np.int64)
            sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(np.float32)
        else:
            sigmas = np.interp(ts, np.arange(0, len(sig)), sig)
            a0 = float(self.alphas_cumprod[0])
            sigmas = np.concatenate([sigmas, [((1 - a0) / a0) ** 0.5]]).astype(np.float32)
        _, first = np.unique(ts, return_index=True)
        if len(first) != len(ts):
            if self.config.use_karras_sigmas:
                raise NotImplementedError("Karras schedule with repeated timesteps (too many steps)")
            keep = np.sort(first)
            ts = ts[keep]
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(ts).to(device=device, dtype=torch.int64)
        self.num_inference_steps = len(ts)

    def _blend_row(self, i: int):
        a_n = float(self.alphas_cumprod[int(self.timesteps[i + 1])])
        return [math.sqrt(a_n), math.sqrt(1 - a_n)]

    def scale_model_input(self, sample, timestep=None):
        return sample

    def add_noise(self, original_samples, noise, timesteps):
        a = self.alphas_cumprod.to(original_samples.device)[timesteps.long()].to(original_samples.dtype)
        while a.dim() < original_samples.dim():
            a = a.unsqueeze(-1)
        return a.sqrt() * original_samples + (1 - a).sqrt() * noise


class DPMSolverMultistepScheduler(_VPSampler):
    """DPM-Solver++ (multistep, data prediction), solver_order 1 or 2, midpoint.

    Schedule (set_timesteps, dpmsolver_multistep.py:243-316):
      * spacing over n + 1 points, the last dropped: linspace -> linspace(0, T-1, n+1).round()[::-1][:-1];
        leading -> arange(n+1) * (T // (n+1)), reversed, [:-1], + steps_offset; trailing -> arange(T, 0, -T/n).round() - 1;
      * sigma_i = sqrt((1 - ab) / ab) interpolated at t_i; the FINAL sigma is sigma at alphas_cumprod[0] (sigma_last,
        :290-292), not 0 — so the last step ends at t = 0, like DDIM with set_alpha_to_one=False;
      * use_karras_sigmas: Karras sigmas between sigma(0) and sigma(T-1), timesteps = round(_sigma_to_t(sigma)), the
        final sigma a copy of the last one (:283-287);
      * duplicate timesteps are dropped (:295-297); a Karras schedule that loses rows that way is refused here.
    Update (dpm_solver_first_order_update :492-540, multistep_dpm_solver_second_order_update :542-650), with
    alpha = 1/sqrt(sigma^2+1), sigma_vp = sigma alpha, lambda = log(alpha) - log(sigma_vp), h = lambda_t - lambda_s:
      D_i = (x - sigma_vp_s eps) / alpha_s                           (convert_model_output, :424-490)
      order 1: x' = (sigma_vp_t / sigma_vp_s) x - alpha_t (e^-h - 1) D_i
      order 2: x' = (sigma_vp_t / sigma_vp_s) x - alpha_t (e^-h - 1) [(1 + 1/2r) D_i - 1/2r D_{i-1}],  r = h_{i-1} / h
    The first step after set_timesteps (lower_order_nums = 0) is first order, also when a sliced schedule starts late;
    lower_order_final: the last step is first order when the schedule has fewer than 15 steps (or euler_at_final)
    (:870-877). scale_model_input is the identity, init_noise_sigma = 1, add_noise is the VP form on alphas_cumprod."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995,
                 sample_max_value: float = 1.0, algorithm_type: str = "dpmsolver++", solver_type: str = "midpoint",
                 lower_order_final: bool = True, euler_at_final: bool = False, use_karras_sigmas: bool = False,
                 use_lu_lambdas: bool = False, lambda_min_clipped: float = -float("inf"), variance_type=None,
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        if solver_order not in (1, 2):
            raise NotImplementedError("solver_order 3 needs two history slots; orders 1 and 2 are built")
        if algorithm_type != "dpmsolver++" or solver_type != "midpoint":
            raise NotImplementedError("only algorithm_type='dpmsolver++' with solver_type='midpoint' is built")
        if prediction_type != "epsilon" or thresholding:
            raise NotImplementedError("only epsilon prediction without thresholding is built")
        if use_lu_lambdas or lambda_min_clipped != -float("inf") or variance_type is not None:
            raise NotImplementedError("use_lu_lambdas / lambda_min_clipped / variance_type are not built")
        self._finish(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                     beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                     prediction_type=prediction_type, thresholding=thresholding, algorithm_type=algorithm_type,
                     solver_type=solver_type, lower_order_final=lower_order_final, euler_at_final=euler_at_final,
                     use_karras_sigmas=use_karras_sigmas, timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        self.init_noise_sigma = 1.0
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy().astype(np.int64))
        self.sigmas = None
        self.lower_order_nums = 0
        self._hist = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        self._set_vp_schedule(num_inference_steps, device)
        self.lower_order_nums = 0
        self._step_index = None
        self._hist = None

    def _lower_order_final(self, i: int) -> bool:
        n = len(self.timesteps)
        return i == n - 1 and (self.config.euler_at_final or (self.config.lower_order_final and n < 15))

    def _row(self, i: int, j: int):
        """Row of full-schedule step i, the j-th step taken since the (sliced) schedule started."""
        s = self.sigmas.double().tolist()
        alpha = lambda k: 1.0 / math.sqrt(s[k] ** 2 + 1.0)
        svp = lambda k: s[k] * alpha(k)
        lam = lambda k: math.log(alpha(k)) - math.log(svp(k))
        a_s, s_s, a_t, s_t = alpha(i), svp(i), alpha(i + 1), svp(i + 1)
        h = lam(i + 1) - lam(i)
        A = a_t * math.expm1(-h)  # alpha_t (e^-h - 1)
        dx, de = 1.0 / a_s, -s_s / a_s
        if self.config.solver_order == 1 or j == 0 or self._lower_order_final(i):
            q = 0.0
        else:
            q = h / (2.0 * (lam(i) - lam(i - 1)))  # 1 / (2 r)
        k = 1.0 + q
        return [dx, de, s_t / s_s - A * k * dx, -A * k * de, A * q, 0.0]

    def _uses_history(self) -> bool:
        return self.config.solver_order > 1

    def step(self, model_output, timestep, sample, generator=None, variance_noise=None, return_dict: bool = True):
        """One DPM-Solver++ step (stateful: step index, lower-order counter, the previous data prediction)."""
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        if self._step_index is None:
            self._init_step_index(timestep)
        i = self._step_index
        hist = None
        if self._uses_history():
            if self._hist is None or self._hist.shape != sample.shape or self._hist.device != sample.device:
                self._hist = torch.zeros(sample.shape, dtype=torch.float32, device=sample.device)
            hist = self._hist
        j = 0 if self.lower_order_nums < 1 else 1
        out = self._run_row(self._row(i, j), model_output, sample, history=hist)
        if self.lower_order_nums < self.config.solver_order:
            self.lower_order_nums += 1
        self._step_index += 1
        return (out,) if not return_dict else SchedulerOutput(out)


# ====================================================================================================== Euler
class _EulerBase(_SamplerBase):
    """Schedule shared by Euler and Euler-ancestral (set_timesteps, euler_discrete.py:221-275):
      * FRACTIONAL fp32 timesteps: linspace -> linspace(0, T-1, n) unrounded; leading -> arange(n) * (T // n),
        reversed, + steps_offset; trailing -> arange(T, 0, -T/n).round() - 1;
      * sigma_i = interp(t_i) of sqrt((1 - ab) / ab), then a final sigma of 0;
      * model input x / sqrt(sigma_i^2 + 1) (scale_model_input :190-212), applied on the device from a scale table;
      * init_noise_sigma (:180-186) = max sigma for linspace / trailing spacing, sqrt(max sigma^2 + 1) for leading;
      * add_noise(x, noise, t) = x + sigma(t) noise with sigma looked up by t's position in the schedule."""

    def _euler_init(self, timestep_spacing, **config):
        self._finish(timestep_spacing=timestep_spacing, **config)
        T = config["num_train_timesteps"]
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        self.sigmas = torch.from_numpy(np.concatenate([sig[::-1], [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(np.linspace(0, T - 1, T, dtype=float)[::-1].copy()).to(torch.float32)

    @property
    def init_noise_sigma(self):
        m = float(self.sigmas.max())
        return m if self.config.timestep_spacing in ("linspace", "trailing") else (m ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps: int, device=None):
        self.num_inference_steps = num_inference_steps
        T = self.config.num_train_timesteps
        sp = self.config.timestep_spacing
        if sp == "linspace":
            ts = np.linspace(0, T - 1, num_inference_steps, dtype=np.float32)[::-1].copy()
        else:
            ts = _spaced(sp, T, num_inference_steps, self.config.steps_offset, 0).astype(np.float32)
        sig = (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()
        sigmas = np.interp(ts, np.arange(0, len(sig)), sig)
        if getattr(self.config, "use_karras_sigmas", False):
            sigmas = _karras(sigmas, num_inference_steps)
            ts = np.array([_sigma_to_t(s, np.log(sig)) for s in sigmas])
        self.sigmas = torch.from_numpy(np.concatenate([sigmas, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(np.float32)).to(device=device)
        self._step_index = None

    def _scale_rows(self, k, S):
        s = self.sigmas.double().tolist()
        return [1.0 / math.sqrt(s[i] ** 2 + 1.0) for i in range(k, k + S)]

    def _blend_row(self, i: int):
        return [1.0, float(self.sigmas[i + 1])]

    def scale_model_input(self, sample, timestep=None):
        if self._step_index is None:
            self._init_step_index(timestep)
        sigma = self.sigmas[self._step_index]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def add_noise(self, original_samples, noise, timesteps):
        sched = self.timesteps.to(original_samples.device)
        idx = [int((sched == t).nonzero()[0]) for t in timesteps.to(original_samples.device).reshape(-1)]
        sigma = self.sigmas.to(original_samples.device, original_samples.dtype)[idx]
        while sigma.dim() < original_samples.dim():
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma


class EulerDiscreteScheduler(_EulerBase):
    """Euler (Karras et al. Algorithm 2 without churn): x' = x + (sigma_{i+1} - sigma_i) eps (step, :320-410)."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon",
                 interpolation_type: str = "linear", use_karras_sigmas: bool = False,
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        if prediction_type != "epsilon":
            raise NotImplementedError("only epsilon prediction is built")
        if interpolation_type != "linear":
            raise NotImplementedError("only interpolation_type='linear' is built")
        self._euler_init(timestep_spacing, num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                         beta_end=beta_end, beta_schedule=beta_schedule, trained_betas=trained_betas,
                         prediction_type=prediction_type, interpolation_type=interpolation_type,
                         use_karras_sigmas=use_karras_sigmas, steps_offset=steps_offset)

    def _row(self, i: int, j: int):
        s = self.sigmas.double().tolist()
        return [0.0, 0.0, 1.0, s[i + 1] - s[i], 0.0, 0.0]

    def step(self, model_output, timestep, sample, s_churn: float = 0.0, s_tmin: float = 0.0,
             s_tmax: float = float("inf"), s_noise: float = 1.0, generator=None, return_dict: bool = True):
        """(diffusers also draws an unused noise tensor here when s_churn = 0; nothing is drawn.)"""
        if s_churn > 0.0:
            raise NotImplementedError("s_churn > 0 adds a stochastic sigma_hat; only s_churn = 0 is built")
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        if self._step_index is None:
            self._init_step_index(timestep)
        out = self._run_row(self._row(self._step_index, 0), model_output, sample)
        self._step_index += 1
        return (out,) if not return_dict else SchedulerOutput(out)


class EulerAncestralDiscreteScheduler(_EulerBase):
    """Euler-ancestral (step, euler_ancestral_discrete.py:296-385), sigma_f = sigma_i, sigma_t = sigma_{i+1}:
      sigma_up = sqrt(sigma_t^2 (sigma_f^2 - sigma_t^2) / sigma_f^2),  sigma_down = sqrt(sigma_t^2 - sigma_up^2)
      x' = x + (sigma_down - sigma_f) eps + sigma_up z,  z = randn_tensor(model_output.shape, generator)
    The last step (sigma_t = 0) adds no noise."""

    _needs_noise = True

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon",
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        if prediction_type != "epsilon":
            raise NotImplementedError("only epsilon prediction is built")
        self._euler_init(timestep_spacing, num_train_timesteps=num_train_timesteps, beta_start=beta_start,
                         beta_end=beta_end, beta_schedule=beta_schedule, trained_betas=trained_betas,
                         prediction_type=prediction_type, steps_offset=steps_offset)

    def sigma_up_down(self, i: int):
        s = self.sigmas.double().tolist()
        sf, st = s[i], s[i + 1]
        up = math.sqrt(st ** 2 * (sf ** 2 - st ** 2) / sf ** 2)
        return up, math.sqrt(st ** 2 - up ** 2)

    def _row(self, i: int, j: int):
        up, down = self.sigma_up_down(i)
        return [0.0, 0.0, 1.0, down - float(self.sigmas[i]), 0.0, up]

    def step(self, model_output, timestep, sample, generator=None, return_dict: bool = True):
        from .pipelines import randn_tensor

        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        if self._step_index is None:
            self._init_step_index(timestep)
        z = randn_tensor(model_output.shape, generator=generator, device=model_output.device, dtype=torch.float32)
        out = self._run_row(self._row(self._step_index, 0), model_output, sample, step_noise=z[None].contiguous())
        self._step_index += 1
        return (out,) if not return_dict else SchedulerOutput(out)


# ====================================================================================================== UniPC
def _unipc_rhos(h: float, rks, order: int, bh1: bool, corrector: bool):
    """(h_phi_1, B_h, rhos) of multistep_uni_p_bh_update / multistep_uni_c_bh_update in fp64, for the step
    h in lambda and the ratios rks = [r_1 .. r_{order-1}]. R / b follow the h_phi_k / factorial recursion; the predictor
    uses rhos_p = [0.5] at order 2 and solve(R[:-1, :-1], b[:-1]) at order 3, the corrector rhos_c = [0.5] at order 1
    and solve(R, b) above. Only the rhos the update reads are formed (at h = 0 the recursion divides by zero)."""
    hh = -h
    h_phi_1 = math.expm1(hh)
    B_h = hh if bh1 else math.expm1(hh)
    if corrector and order == 1:
        return h_phi_1, B_h, [0.5]
    if not corrector and order <= 2:
        return h_phi_1, B_h, [0.5] * (order - 1)
    r = np.array(list(rks) + [1.0])
    R, b = [], []
    h_phi_k, fact = h_phi_1 / hh - 1.0, 1
    for i in range(1, order + 1):
        R.append(r ** (i - 1))
        b.append(h_phi_k * fact / B_h)
        fact *= i + 1
        h_phi_k = h_phi_k / hh - 1.0 / fact
    R, b = np.array(R), np.array(b)
    rhos = np.linalg.solve(R, b) if corrector else np.linalg.solve(R[:-1, :-1], b[:-1])
    return h_phi_1, B_h, [float(v) for v in rhos]


class UniPCMultistepScheduler(_VPSampler):
    """UniPC (Zhao et al. 2023): the UniP predictor and the UniC corrector, predict_x0, solver_type bh1 / bh2, solver
    orders 1-3.

    Schedule: DPM-Solver's (set_timesteps), see _VPSampler — n + 1 spaced points with the
    last dropped, the final sigma at alphas_cumprod[0], Karras sigmas with the final sigma repeated; a Karras schedule
    that loses rows to duplicate timesteps is refused. scale_model_input is the identity, init_noise_sigma = 1,
    add_noise is the VP form on alphas_cumprod.
    Update (step, multistep_uni_{p,c}_bh_update), with alpha = 1/sqrt(sigma^2+1), sigma_vp = sigma alpha,
    lambda = log(alpha) - log(sigma_vp), hh = -h, h_phi_1 = expm1(hh), B_h = hh (bh1) or expm1(hh) (bh2), rhos from
    _unipc_rhos:
      m_i = (x - sigma_vp_i eps) / alpha_i                           (convert_model_output, from the UNCORRECTED x)
      corrector at step i > 0 when i-1 is not in disable_corrector (x = S, the previous corrected sample; m0 = m_{i-1};
      the previous step's order q; h = lambda_i - lambda_{i-1}; r_k = (lambda_{i-1-k} - lambda_{i-1}) / h):
        c = (sigma_vp_i / sigma_vp_{i-1}) S - alpha_i h_phi_1 m0
            - alpha_i B_h (sum_k rhos_c[k-1] (m_{i-1-k} - m0) / r_k + rhos_c[-1] (m_i - m0))
      else c = x;  S <- c (last_sample, before any inpaint blend)
      predictor of order p from c, m0 = m_i, h = lambda_{i+1} - lambda_i, r_k = (lambda_{i-k} - lambda_i) / h:
        x' = (sigma_vp_{i+1} / sigma_vp_i) c - alpha_{i+1} h_phi_1 m0
             - alpha_{i+1} B_h sum_k rhos_p[k-1] (m_{i-k} - m0) / r_k
      p = min(solver_order, n - i) with lower_order_final (at every step count, unlike DPM-Solver's n < 15 rule), then
      min(p, lower_order_nums + 1). A step sequence that starts late (inpainting, strength < 1) restarts the warm-up:
      first order and no corrector at its first step, so its rows are not rows of the full table (_row(i, j)).
    At h = 0 (the last Karras step, whose sigma repeats) the predictor returns c, which is diffusers' result at orders
    1 and 2 (at order 3 its solve has a NaN system).
    Each step is linear in x, eps, the stash S and the previous data predictions, and is one row of
    imagd_cfg_sampler_pc_step. Slot k < 3 holds the data prediction of the j-th step taken with j % 3 = k, slot 3 the
    stash: fixed addresses, and every slot a row reads was written by an earlier row of the same sequence.
    Options that change the form of the update raise NotImplementedError: predict_x0=False, solver_p, thresholding,
    non-epsilon prediction, solver_order > 3."""

    _predictor_corrector = True
    _STASH = 3

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False,
                 dynamic_thresholding_ratio: float = 0.995, sample_max_value: float = 1.0, predict_x0: bool = True,
                 solver_type: str = "bh2",
                 lower_order_final: bool = True, disable_corrector=(), solver_p=None, use_karras_sigmas: bool = False,
                 timestep_spacing: str = "linspace", steps_offset: int = 0):
        if solver_order not in (1, 2, 3):
            raise NotImplementedError("solver_order 1-3 are built (a higher order needs more slots)")
        if solver_type in ("midpoint", "heun", "logrho"):  # diffusers registers these as bh2
            solver_type = "bh2"
        if solver_type not in ("bh1", "bh2"):
            raise NotImplementedError(f"solver_type {solver_type!r}")
        if not predict_x0 or solver_p is not None:
            raise NotImplementedError("only predict_x0=True without solver_p is built")
        if prediction_type != "epsilon" or thresholding:
            raise NotImplementedError("only epsilon prediction without thresholding is built")
        self._finish(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                     beta_schedule=beta_schedule, trained_betas=trained_betas, solver_order=solver_order,
                     prediction_type=prediction_type, thresholding=thresholding, predict_x0=predict_x0,
                     solver_type=solver_type, lower_order_final=lower_order_final,
                     disable_corrector=list(disable_corrector), use_karras_sigmas=use_karras_sigmas,
                     timestep_spacing=timestep_spacing, steps_offset=steps_offset)
        self.init_noise_sigma = 1.0
        self.timesteps = torch.from_numpy(np.linspace(0, num_train_timesteps - 1, num_train_timesteps,
                                                      dtype=np.float32)[::-1].copy().astype(np.int64))
        self.sigmas = None
        self._taken = 0
        self._bank = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        self._set_vp_schedule(num_inference_steps, device)
        self._step_index = None
        self._taken = 0
        self._bank = None

    def _order(self, i: int, j: int) -> int:
        """this_order of full-schedule step i, the j-th step taken (lower_order_nums = min(j, solver_order))."""
        p = self.config.solver_order
        if self.config.lower_order_final:
            p = min(p, len(self.timesteps) - i)
        return min(p, j + 1)

    def _row(self, i: int, j: int):
        """Row {dx, de, ax, am, a0..a3, bc, bm, b0..b3, w_m, w_c} of full-schedule step i, the j-th step taken."""
        s = self.sigmas.double().tolist()
        alpha = lambda k: 1.0 / math.sqrt(s[k] ** 2 + 1.0)
        svp = lambda k: s[k] * alpha(k)
        lam = lambda k: math.log(alpha(k)) - math.log(svp(k))
        slot = lambda jj: jj % 3  # the data prediction of the jj-th step taken
        bh1 = self.config.solver_type == "bh1"
        ax, am, a = 1.0, 0.0, [0.0] * 4
        if j > 0 and (i - 1) not in self.config.disable_corrector:
            q = self._order(i - 1, j - 1)
            h = lam(i) - lam(i - 1)
            rks = [(lam(i - 1 - k) - lam(i - 1)) / h for k in range(1, q)]
            h_phi_1, B_h, rc = _unipc_rhos(h, rks, q, bh1, corrector=True)
            A = alpha(i)
            ax, am = 0.0, -A * B_h * rc[-1]
            a[self._STASH] = svp(i) / svp(i - 1)
            a[slot(j - 1)] = -A * h_phi_1 + A * B_h * (rc[-1] + sum(rc[k - 1] / rks[k - 1] for k in range(1, q)))
            for k in range(1, q):
                a[slot(j - 1 - k)] -= A * B_h * rc[k - 1] / rks[k - 1]
        bc, bm, b = 1.0, 0.0, [0.0] * 4
        h = lam(i + 1) - lam(i)
        if h != 0.0:
            p = self._order(i, j)
            rks = [(lam(i - k) - lam(i)) / h for k in range(1, p)]
            h_phi_1, B_h, rp = _unipc_rhos(h, rks, p, bh1, corrector=False)
            A = alpha(i + 1)
            bc = svp(i + 1) / svp(i)
            bm = -A * h_phi_1 + A * B_h * sum(rp[k - 1] / rks[k - 1] for k in range(1, p))
            for k in range(1, p):
                b[slot(j - k)] -= A * B_h * rp[k - 1] / rks[k - 1]
        return [1.0 / alpha(i), -svp(i) / alpha(i), ax, am, *a, bc, bm, *b, float(slot(j)), float(self._STASH)]

    def step(self, model_output, timestep, sample, return_dict: bool = True):
        """One UniPC step (stateful: step index, steps taken, the slot bank) through the predictor-corrector kernel."""
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        if self._step_index is None:
            self._init_step_index(timestep)
        bank = self._bank
        if bank is None or bank.shape[1:] != sample.shape or bank.device != sample.device:
            bank = self._bank = torch.empty((ops.PC_SLOTS, *sample.shape), dtype=torch.float32, device=sample.device)
        x = sample.float().contiguous()
        out = x.clone()
        coef = torch.tensor([self._row(self._step_index, self._taken)], dtype=torch.float32, device=x.device)
        step = torch.zeros(2, dtype=torch.int32, device=x.device)
        ops.cfg_sampler_pc_step(model_output.float().contiguous(), None, 1.0, out, coef, step, bank)
        self._taken += 1
        self._step_index += 1
        out = out.to(sample.dtype)
        return (out,) if not return_dict else SchedulerOutput(out)
