"""ORACLE (test infrastructure, not product): PNDMScheduler with skip_prk_steps=True (PLMS) restated step by step.

diffusers==0.27.0 schedulers/scheduling_pndm.py, restated from the published source as recalled, in its loop form:
`set_timesteps` (the three spacings, then the PLMS list with the last-but-one timestep repeated), `step_plms` with
its counter, eps history and Heun restart at counter 1, `_get_prev_sample`, `add_noise`. The scheduler stored by the
SD-1.5 inpainting checkpoint the v1 app loads (reference app.py:91-93). Arithmetic in float64 torch over the fp32
alpha_bar table diffusers keeps.
PARITY UNPINNED against diffusers (absent here: no golden vectors of the original exist). Held to the mathematics
instead: tests/test_pndm_cpu.py measures its order of accuracy on the closed-form Gaussian problem.
"""
from __future__ import annotations

import numpy as np
import torch


class PNDMOracle:
    order = 1
    init_noise_sigma = 1.0

    def __init__(self, num_train_timesteps=1000, beta_start=0.00085, beta_end=0.012, beta_schedule="scaled_linear",
                 set_alpha_to_one=False, steps_offset=1, timestep_spacing="leading"):
        self.T = num_train_timesteps
        if beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        else:
            assert beta_schedule == "linear", beta_schedule
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        self.alphas_cumprod = torch.cumprod(1.0 - betas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.steps_offset, self.timestep_spacing = steps_offset, timestep_spacing
        self.num_inference_steps = None

    def set_timesteps(self, n: int, device=None):
        T = self.T
        self.num_inference_steps = n
        if self.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round().astype(np.int64)
        elif self.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round()
            ts += self.steps_offset
        elif self.timestep_spacing == "trailing":
            ts = np.round(np.arange(T, 0, -T / n))[::-1].astype(np.int64)
            ts -= 1
        else:
            raise ValueError(self.timestep_spacing)
        plms = np.concatenate([ts[:-1], ts[-2:-1], ts[-1:]])[::-1].copy()
        self.timesteps = torch.from_numpy(plms.astype(np.int64))
        self.ets = []
        self.counter = 0
        self.cur_sample = None

    def scale_model_input(self, sample, timestep=None):
        return sample

    def step(self, model_output, timestep, sample):
        ratio = self.T // self.num_inference_steps
        timestep = int(timestep)
        prev_timestep = timestep - ratio
        if self.counter != 1:
            self.ets = self.ets[-3:]
            self.ets.append(model_output)
        else:
            prev_timestep = timestep
            timestep = timestep + ratio
        if len(self.ets) == 1 and self.counter == 0:
            self.cur_sample = sample
        elif len(self.ets) == 1 and self.counter == 1:
            model_output = (model_output + self.ets[-1]) / 2
            sample = self.cur_sample
            self.cur_sample = None
        elif len(self.ets) == 2:
            model_output = (3 * self.ets[-1] - self.ets[-2]) / 2
        elif len(self.ets) == 3:
            model_output = (23 * self.ets[-1] - 16 * self.ets[-2] + 5 * self.ets[-3]) / 12
        else:
            model_output = (1 / 24) * (55 * self.ets[-1] - 59 * self.ets[-2] + 37 * self.ets[-3] - 9 * self.ets[-4])
        prev = self._get_prev_sample(sample, timestep, prev_timestep, model_output)
        self.counter += 1
        return prev

    def _get_prev_sample(self, sample, timestep, prev_timestep, model_output):
        a_t = float(self.alphas_cumprod[timestep])
        a_p = float(self.alphas_cumprod[prev_timestep]) if prev_timestep >= 0 else float(self.final_alpha_cumprod)
        sample_coeff = (a_p / a_t) ** 0.5
        denom = a_t * (1 - a_p) ** 0.5 + (a_t * (1 - a_t) * a_p) ** 0.5
        return sample_coeff * sample - (a_p - a_t) * model_output / denom

    def add_noise(self, original, noise, timesteps):
        a = self.alphas_cumprod[timesteps].to(original.dtype)
        while a.dim() < original.dim():
            a = a[..., None]
        return a ** 0.5 * original + (1 - a) ** 0.5 * noise
