"""ORACLE (test infrastructure, not product): EulerDiscreteScheduler / EulerAncestralDiscreteScheduler restated
step by step.

diffusers==0.27.0 schedulers/scheduling_euler_discrete.py and scheduling_euler_ancestral_discrete.py, restated from
the published source as recalled, in their loop form: `set_timesteps` (three spacings, linear sigma interpolation,
Karras sigmas), `init_noise_sigma`, `scale_model_input`, `add_noise` and `step` for epsilon prediction with
s_churn = 0. Euler's `step` draws one noise tensor per call and discards it at s_churn = 0; the ancestral step adds it
with scale sigma_up. Arithmetic in float64 torch.
PARITY UNPINNED against diffusers (absent here: no golden vectors of the original exist). Held to the mathematics
instead: tests/test_solver_schedulers_cpu.py measures its order of accuracy on the closed-form Gaussian problem.
"""
from __future__ import annotations

import numpy as np
import torch

from .dpmsolver import convert_to_karras, sigma_to_t, train_sigmas


class EulerOracle:
    ancestral = False

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 use_karras_sigmas=False, timestep_spacing="leading", steps_offset=1):
        self.T = num_train_timesteps
        self.alphas_cumprod, self._sigmas = train_sigmas(num_train_timesteps, beta_start, beta_end, beta_schedule)
        self.use_karras_sigmas = use_karras_sigmas
        self.timestep_spacing, self.steps_offset = timestep_spacing, steps_offset
        self.sigmas = torch.cat([torch.from_numpy(self._sigmas).flip(0), torch.zeros(1)]).double()
        self.order = 1
        self.step_index = None

    @property
    def init_noise_sigma(self):
        max_sigma = self.sigmas.max()
        if self.timestep_spacing in ["linspace", "trailing"]:
            return max_sigma
        return (max_sigma ** 2 + 1) ** 0.5

    def set_timesteps(self, n: int):
        T = self.T
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n, dtype=float if self.ancestral else np.float32)[::-1].copy()
        elif self.timestep_spacing == "leading":
            step_ratio = T // n
            ts = (np.arange(0, n) * step_ratio).round()[::-1].copy().astype(np.float32)
            ts += self.steps_offset
        elif self.timestep_spacing == "trailing":
            step_ratio = T / n
            ts = (np.arange(T, 0, -step_ratio)).round().copy().astype(np.float32)
            ts -= 1
        else:
            raise ValueError(self.timestep_spacing)
        sigmas = self._sigmas
        log_sigmas = np.log(sigmas)
        sigmas = np.interp(ts, np.arange(0, len(sigmas)), sigmas)
        if self.use_karras_sigmas:
            sigmas = convert_to_karras(sigmas, n)
            ts = np.array([sigma_to_t(s, log_sigmas) for s in sigmas])
        sigmas = np.concatenate([sigmas, [0.0]]).astype(np.float32)
        self.sigmas = torch.from_numpy(sigmas).double()
        self.timesteps = torch.from_numpy(np.asarray(ts, dtype=np.float32))
        self.num_inference_steps = n
        self.step_index = None

    def index_for_timestep(self, timestep):
        idx = (self.timesteps == timestep).nonzero()
        return int(idx[1 if len(idx) > 1 else 0])

    def scale_model_input(self, sample, timestep):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(timestep)
        sigma = self.sigmas[self.step_index]
        return sample / ((sigma ** 2 + 1) ** 0.5)

    def add_noise(self, original_samples, noise, timesteps):
        sigma = self.sigmas[[self.index_for_timestep(t) for t in timesteps]].to(original_samples.dtype)
        while sigma.dim() < original_samples.dim():
            sigma = sigma.unsqueeze(-1)
        return original_samples + noise * sigma

    def step(self, model_output, timestep, sample, generator=None, variance_noise=None, **unused):
        if self.step_index is None:
            self.step_index = self.index_for_timestep(timestep)
        sigma = self.sigmas[self.step_index]
        noise = variance_noise if variance_noise is not None else torch.randn(
            model_output.shape, generator=generator, dtype=torch.float32).to(model_output.dtype)
        pred_original_sample = sample - sigma * model_output
        derivative = (sample - pred_original_sample) / sigma
        if self.ancestral:
            sigma_from, sigma_to = sigma, self.sigmas[self.step_index + 1]
            sigma_up = (sigma_to ** 2 * (sigma_from ** 2 - sigma_to ** 2) / sigma_from ** 2) ** 0.5
            sigma_down = (sigma_to ** 2 - sigma_up ** 2) ** 0.5
            prev = sample + derivative * (sigma_down - sigma) + noise * sigma_up
        else:  # s_churn = 0: gamma = 0, sigma_hat = sigma, the drawn noise is unused
            prev = sample + derivative * (self.sigmas[self.step_index + 1] - sigma)
        self.step_index += 1
        return prev


class EulerAncestralOracle(EulerOracle):
    ancestral = True
