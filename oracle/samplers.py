"""Oracle: DPMSolverMultistepScheduler (dpmsolver++, midpoint), EulerDiscreteScheduler and
EulerAncestralDiscreteScheduler of diffusers-0.24, restated the way diffusers writes them: fp32 torch sigma / lambda
arithmetic per step and an explicit list of previous data predictions, no coefficient tables. TEST INFRASTRUCTURE ONLY.

The product (imagdressing_b200/samplers.py) folds every update into a per-step row for one fused kernel; checking it
against this step-by-step formulation checks the table algebra. Defaults are the reference's DDIM configuration
(scaled_linear 0.00085..0.012, timestep_spacing="leading", steps_offset=1), which is what `X.from_config(ddim.config)`
gives a user of the reference scripts.
"""
from __future__ import annotations

import numpy as np
import torch


class _Oracle:
    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 timestep_spacing="leading", steps_offset=1, use_karras_sigmas=False):
        self.T = num_train_timesteps
        if beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        else:
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.spacing, self.steps_offset, self.karras = timestep_spacing, steps_offset, use_karras_sigmas
        self.step_index = None

    def _train_sigmas(self):
        return (((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5).numpy()

    @staticmethod
    def _karras(in_sigmas, n):
        rho = 7.0
        ramp = np.linspace(0, 1, n)
        lo, hi = in_sigmas[-1].item() ** (1 / rho), in_sigmas[0].item() ** (1 / rho)
        return (hi + ramp * (lo - hi)) ** rho

    @staticmethod
    def _sigma_to_t(sigma, log_sigmas):
        log_sigma = np.log(np.maximum(sigma, 1e-10))
        dists = log_sigma - log_sigmas[:, np.newaxis]
        low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
        low, high = log_sigmas[low_idx], log_sigmas[low_idx + 1]
        w = np.clip((low - log_sigma) / (low - high), 0, 1)
        return ((1 - w) * low_idx + w * (low_idx + 1)).reshape(sigma.shape)

    def _init_step_index(self, t):
        idx = (self.timesteps == t).nonzero()
        self.step_index = int(idx[1]) if len(idx) > 1 else int(idx[0])


class DPMSolverOracle(_Oracle):
    """dpmsolver++ multistep, data prediction, midpoint second order."""

    def __init__(self, solver_order=2, lower_order_final=True, **kw):
        super().__init__(**kw)
        self.solver_order, self.lower_order_final = solver_order, lower_order_final
        self.init_noise_sigma = 1.0
        self.order = 1

    def set_timesteps(self, n, device=None):
        T = self.T
        if self.spacing == "linspace":
            ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif self.spacing == "leading":
            ts = (np.arange(0, n + 1) * (T // (n + 1))).round()[::-1][:-1].copy().astype(np.int64) + self.steps_offset
        else:
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.int64) - 1
        sig = self._train_sigmas()
        if self.karras:
            sigmas = self._karras(np.flip(sig).copy(), n)
            ts = np.array([self._sigma_to_t(s, np.log(sig)) for s in sigmas]).round().astype(np.int64)
            sigmas = np.concatenate([sigmas, sigmas[-1:]]).astype(np.float32)
        else:
            sigmas = np.interp(ts, np.arange(0, len(sig)), sig)
            last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
            sigmas = np.concatenate([sigmas, [last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas)
        self.timesteps = torch.from_numpy(ts).to(device)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0
        self.step_index = None

    @staticmethod
    def _alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def scale_model_input(self, x, t=None):
        return x

    def step(self, eps, t, x):
        if self.step_index is None:
            self._init_step_index(t)
        i = self.step_index
        alpha_s0, sigma_s0 = self._alpha_sigma(self.sigmas[i])
        x0 = (x - sigma_s0 * eps) / alpha_s0
        self.model_outputs = self.model_outputs[1:] + [x0]
        n = len(self.timesteps)
        final = i == n - 1 and self.lower_order_final and n < 15
        alpha_t, sigma_t = self._alpha_sigma(self.sigmas[i + 1])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        h = lambda_t - lambda_s0
        if self.solver_order == 1 or self.lower_order_nums < 1 or final:
            out = (sigma_t / sigma_s0) * x - (alpha_t * (torch.exp(-h) - 1.0)) * x0
        else:
            alpha_s1, sigma_s1 = self._alpha_sigma(self.sigmas[i - 1])
            lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
            m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
            r0 = (lambda_s0 - lambda_s1) / h
            d0, d1 = m0, (1.0 / r0) * (m0 - m1)
            out = (sigma_t / sigma_s0) * x - (alpha_t * (torch.exp(-h) - 1.0)) * d0 \
                - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * d1
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return (out,)

    def add_noise(self, x, noise, t):
        a = self.alphas_cumprod.to(x.device)[t].reshape(-1, 1, 1, 1).to(x.dtype)
        return a.sqrt() * x + (1 - a).sqrt() * noise


class EulerOracle(_Oracle):
    """Euler, s_churn = 0. `ancestral=True` with a generator: Euler-ancestral."""

    def __init__(self, ancestral=False, generator=None, **kw):
        super().__init__(**kw)
        self.ancestral, self.generator = ancestral, generator
        self.order = 1

    def set_timesteps(self, n, device=None):
        T = self.T
        if self.spacing == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=np.float32)[::-1].copy()
        elif self.spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()[::-1].copy().astype(np.float32) + self.steps_offset
        else:
            ts = np.arange(T, 0, -T / n).round().copy().astype(np.float32) - 1
        sig = self._train_sigmas()
        sigmas = np.interp(ts, np.arange(0, len(sig)), sig)
        if self.karras:
            sigmas = self._karras(sigmas, n)
            ts = np.array([self._sigma_to_t(s, np.log(sig)) for s in sigmas])
        self.sigmas = torch.from_numpy(np.concatenate([sigmas, [0.0]]).astype(np.float32))
        self.timesteps = torch.from_numpy(ts.astype(np.float32)).to(device)
        self.step_index = None

    @property
    def init_noise_sigma(self):
        m = float(self.sigmas.max())
        return m if self.spacing in ("linspace", "trailing") else (m ** 2 + 1) ** 0.5

    def scale_model_input(self, x, t):
        if self.step_index is None:
            self._init_step_index(t)
        return x / ((self.sigmas[self.step_index] ** 2 + 1) ** 0.5)

    def step(self, eps, t, x):
        if self.step_index is None:
            self._init_step_index(t)
        sigma = self.sigmas[self.step_index]
        sigma_next = self.sigmas[self.step_index + 1]
        pred_original = x - sigma * eps
        derivative = (x - pred_original) / sigma
        if not self.ancestral:
            out = x + derivative * (sigma_next - sigma)
        else:
            sigma_up = (sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2) ** 0.5
            sigma_down = (sigma_next ** 2 - sigma_up ** 2) ** 0.5
            out = x + derivative * (sigma_down - sigma)
            z = torch.randn(eps.shape, generator=self.generator, dtype=torch.float32).to(eps.device)
            out = out + z * sigma_up
        self.step_index += 1
        return (out,)

    def add_noise(self, x, noise, t):
        idx = [int((self.timesteps.to(x.device) == tt).nonzero()[0]) for tt in t.reshape(-1)]
        return x + noise * self.sigmas.to(x.device)[idx].reshape(-1, 1, 1, 1)


@torch.no_grad()
def sample_one(unet, ref_unet, latents, prompt_embeds, negative_embeds, garment_tokens, ref_latents, guidance, steps,
               scheduler, controlnet=None, control_cond=None, control_scale=1.0, mask=None, image_latents=None,
               noise=None, strength=1.0):
    """The reference denoising loop (IMAGDressing_v1_pipeline.py:463-541; ControlNet ipa_controlnet.py:651-666;
    inpainting _controlnet_inpainting.py:385-500) with any scheduler of this module, at batch 1 in fp32, with the two
    separate UNet calls per step the reference makes. oracle/pipeline.py holds the same loop for DDIM; this one adds
    what a sigma-space scheduler needs: the start latents scaled by init_noise_sigma, scale_model_input on the UNet and
    ControlNet input, and the inpainting strength (the sliced schedule starts from add_noise(image_latents, noise,
    t_start), not rescaled). latents: unit-variance noise [1,4,h,w] (the inpainting `noise` when mask is given)."""
    sch = scheduler
    sch.set_timesteps(steps, device=latents.device)
    ts = sch.timesteps
    if mask is not None and strength < 1.0:
        ts = ts[steps - min(int(steps * strength), steps):]
        latents = sch.add_noise(image_latents, noise, ts[:1])
    else:
        latents = latents * sch.init_noise_sigma
    sa = None
    for i, t in enumerate(ts):
        if i == 0:  # :465-479 — garment pass at t = 0, keep the attn1 processor inputs
            ref_unet(ref_latents, torch.zeros_like(t), garment_tokens)
            sa = {n: p.cache["hidden_states"] for n, p in ref_unet.attn_processors.items()}
        x_in = sch.scale_model_input(latents, t)  # inpainting.py:390,411
        down_c = mid_c = down_u = mid_u = None
        if controlnet is not None:  # batch-2 call, [uncond, cond] text
            down, mid = controlnet(torch.cat([x_in] * 2), t, torch.cat([negative_embeds, prompt_embeds]), control_cond,
                                   conditioning_scale=control_scale)
            down_c, mid_c = [d[1:2] for d in down], mid[1:2]
            down_u, mid_u = [d[0:1] for d in down], mid[0:1]
        eps_c = unet(x_in, t, prompt_embeds, cross_attention_kwargs={"sa_hidden_states": sa},
                     down_block_additional_residuals=down_c, mid_block_additional_residual=mid_c)[0]
        eps_u = unet(x_in, t, negative_embeds, down_block_additional_residuals=down_u,
                     mid_block_additional_residual=mid_u)[0]  # (no garment stream)
        latents = sch.step(eps_u + guidance * (eps_c - eps_u), t, latents)[0]
        if mask is not None:  # inpainting.py:487-500
            proper = image_latents
            if i < len(ts) - 1:
                proper = sch.add_noise(image_latents, noise, ts[i + 1:i + 2])
            latents = (1 - mask) * proper + mask * latents
    return latents
