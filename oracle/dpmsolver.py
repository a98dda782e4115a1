"""ORACLE (test infrastructure, not product): DPMSolverMultistepScheduler restated step by step.

diffusers==0.27.0 schedulers/scheduling_dpmsolver_multistep.py (DPM-Solver++, Lu et al. 2022), restated from its
published source as recalled, in its loop form: `convert_model_output` (x0 prediction), the history shift of
`model_outputs`, `dpm_solver_first_order_update` / `multistep_dpm_solver_second_order_update`, `lower_order_final`
/ `euler_at_final` / `final_sigmas_type`, Karras sigmas. Epsilon prediction, algorithm_type dpmsolver++ and
sde-dpmsolver++, solver_order 1 and 2. Arithmetic in float64 torch (diffusers runs the same expressions in the
model dtype).
PARITY UNPINNED against diffusers (absent here: no golden vectors of the original exist). Held to the mathematics
instead: tests/test_solver_schedulers_cpu.py measures its order of accuracy on the closed-form Gaussian problem.
"""
from __future__ import annotations

import numpy as np
import torch


def train_sigmas(num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear"):
    """((1 - a) / a) ** 0.5 of the training schedule, fp32 like diffusers"""
    if beta_schedule == "linear":
        betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
    elif beta_schedule == "scaled_linear":
        betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
    else:
        raise NotImplementedError(beta_schedule)
    ac = torch.cumprod(1.0 - betas, dim=0)
    return ac, np.array(((1 - ac) / ac) ** 0.5)


def sigma_to_t(sigma, log_sigmas):
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.reshape(np.shape(sigma))


def convert_to_karras(in_sigmas, num_inference_steps, sigma_min=None, sigma_max=None):
    sigma_min = sigma_min if sigma_min is not None else in_sigmas[-1].item()
    sigma_max = sigma_max if sigma_max is not None else in_sigmas[0].item()
    rho = 7.0
    ramp = np.linspace(0, 1, num_inference_steps)
    min_inv_rho = sigma_min ** (1 / rho)
    max_inv_rho = sigma_max ** (1 / rho)
    return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho


class DPMSolverOracle:
    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 solver_order=2, algorithm_type="dpmsolver++", solver_type="midpoint", lower_order_final=True,
                 euler_at_final=False, use_karras_sigmas=False, final_sigmas_type="zero",
                 timestep_spacing="leading", steps_offset=1):
        self.T = num_train_timesteps
        self.alphas_cumprod, self._sigmas = train_sigmas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.solver_order, self.algorithm_type, self.solver_type = solver_order, algorithm_type, solver_type
        self.lower_order_final, self.euler_at_final = lower_order_final, euler_at_final
        self.use_karras_sigmas, self.final_sigmas_type = use_karras_sigmas, final_sigmas_type
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.init_noise_sigma = 1.0
        self.order = 1

    def scale_model_input(self, sample, timestep=None):
        return sample

    def set_timesteps(self, n: int):
        last_timestep = self.T  # lambda_min_clipped = -inf
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, last_timestep - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif self.timestep_spacing == "leading":
            step_ratio = last_timestep // (n + 1)
            ts = (np.arange(0, n + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += self.steps_offset
        elif self.timestep_spacing == "trailing":
            step_ratio = self.T / n
            ts = np.arange(last_timestep, 0, -step_ratio).round().copy().astype(np.int64)
            ts -= 1
        else:
            raise ValueError(self.timestep_spacing)
        sigmas = self._sigmas
        log_sigmas = np.log(sigmas)
        if self.use_karras_sigmas:
            sigmas = np.flip(sigmas).copy()
            sigmas = convert_to_karras(sigmas, n)
            ts = np.array([sigma_to_t(s, log_sigmas) for s in sigmas]).round()
        else:
            sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        if self.final_sigmas_type == "sigma_min":
            sigma_last = ((1 - self.alphas_cumprod[0]) / self.alphas_cumprod[0]) ** 0.5
        else:
            sigma_last = 0
        sigmas = np.concatenate([sigmas, [sigma_last]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas).double()
        self.timesteps = torch.from_numpy(np.asarray(ts)).to(torch.int64)
        self.num_inference_steps = len(ts)
        self.model_outputs = [None] * self.solver_order
        self.lower_order_nums = 0
        self.step_index = None

    def index_for_timestep(self, timestep):
        idx = (self.timesteps == timestep).nonzero()
        return int(idx[1 if len(idx) > 1 else 0])

    @staticmethod
    def _alpha_sigma(sigma):
        alpha_t = 1 / ((sigma ** 2 + 1) ** 0.5)
        return alpha_t, sigma * alpha_t

    def add_noise(self, original_samples, noise, timesteps):
        sigma = self.sigmas[[self.index_for_timestep(t) for t in timesteps]].to(original_samples.dtype)
        a, s = self._alpha_sigma(sigma)
        while a.dim() < original_samples.dim():
            a, s = a.unsqueeze(-1), s.unsqueeze(-1)
        return a * original_samples + s * noise

    def _convert(self, eps, sample):
        alpha_t, sigma_t = self._alpha_sigma(self.sigmas[self.step_index])
        return (sample - sigma_t * eps) / alpha_t

    def _first_order(self, m0, sample, noise):
        alpha_t, sigma_t = self._alpha_sigma(self.sigmas[self.step_index + 1])
        alpha_s, sigma_s = self._alpha_sigma(self.sigmas[self.step_index])
        h = (torch.log(alpha_t) - torch.log(sigma_t)) - (torch.log(alpha_s) - torch.log(sigma_s))
        if self.algorithm_type == "dpmsolver++":
            return (sigma_t / sigma_s) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * m0
        return ((sigma_t / sigma_s * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * m0
                + sigma_t * torch.sqrt(1.0 - torch.exp(-2 * h)) * noise)

    def _second_order(self, sample, noise):
        alpha_t, sigma_t = self._alpha_sigma(self.sigmas[self.step_index + 1])
        alpha_s0, sigma_s0 = self._alpha_sigma(self.sigmas[self.step_index])
        alpha_s1, sigma_s1 = self._alpha_sigma(self.sigmas[self.step_index - 1])
        lambda_t = torch.log(alpha_t) - torch.log(sigma_t)
        lambda_s0 = torch.log(alpha_s0) - torch.log(sigma_s0)
        lambda_s1 = torch.log(alpha_s1) - torch.log(sigma_s1)
        m0, m1 = self.model_outputs[-1], self.model_outputs[-2]
        h, h_0 = lambda_t - lambda_s0, lambda_s0 - lambda_s1
        r0 = h_0 / h
        D0, D1 = m0, (1.0 / r0) * (m0 - m1)
        if self.algorithm_type == "dpmsolver++":
            if self.solver_type == "midpoint":
                return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                        - 0.5 * (alpha_t * (torch.exp(-h) - 1.0)) * D1)
            return ((sigma_t / sigma_s0) * sample - (alpha_t * (torch.exp(-h) - 1.0)) * D0
                    + (alpha_t * ((torch.exp(-h) - 1.0) / h + 1.0)) * D1)
        if self.solver_type == "midpoint":
            return ((sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
                    + 0.5 * (alpha_t * (1 - torch.exp(-2.0 * h))) * D1
                    + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise)
        return ((sigma_t / sigma_s0 * torch.exp(-h)) * sample + (alpha_t * (1 - torch.exp(-2.0 * h))) * D0
                + (alpha_t * ((1.0 - torch.exp(-2.0 * h)) / (-2.0 * h) + 1.0)) * D1
                + sigma_t * torch.sqrt(1.0 - torch.exp(-2.0 * h)) * noise)

    def step(self, model_output, timestep, sample, generator=None, variance_noise=None, **unused):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(timestep)
        n = len(self.timesteps)
        lower_order_final = (self.step_index == n - 1) and (
            self.euler_at_final or (self.lower_order_final and n < 15) or self.final_sigmas_type == "zero")
        model_output = self._convert(model_output, sample)
        for i in range(self.solver_order - 1):
            self.model_outputs[i] = self.model_outputs[i + 1]
        self.model_outputs[-1] = model_output
        noise = None
        if self.algorithm_type == "sde-dpmsolver++":
            noise = variance_noise if variance_noise is not None else torch.randn(
                model_output.shape, generator=generator, dtype=torch.float32).to(model_output.dtype)
        if self.solver_order == 1 or self.lower_order_nums < 1 or lower_order_final:
            prev = self._first_order(model_output, sample, noise)
        else:
            prev = self._second_order(sample, noise)
        if self.lower_order_nums < self.solver_order:
            self.lower_order_nums += 1
        self.step_index += 1
        return prev
