"""DDIMScheduler, UniPCMultistepScheduler, DPMSolverMultistepScheduler, EulerDiscreteScheduler and
EulerAncestralDiscreteScheduler with the diffusers surface the reference pipelines duck-type
(`.config`, `.set_timesteps`, `.timesteps`, `.order`, `.init_noise_sigma`, `.scale_model_input`,
`.step(..., eta=, generator=, return_dict=False)[0]`, `.add_noise`, `from_config`; SURVEY.md §8b),
restating diffusers==0.27.0 DDIMScheduler (SURVEY.md App. A.8) as called by
powerpaint/pipelines/pipeline_PowerPaint.py:906 (set_timesteps), :993 (scale_model_input),
:1023 (step), :642 (init_noise_sigma).

Host side only computes the schedule (numpy / CPU tensors). The arithmetic of `step` on CUDA
tensors runs in the fused CFG+DDIM kernel (`pp_cfg_ddim_step`); there is no CPU `step`.
`step_coefficients()` exports the per-step scalar table the captured CUDA graph indexes.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import List, Optional, Tuple, Union

import numpy as np
import torch

from .config import Config


class DDIMSchedulerOutput(SimpleNamespace):
    pass


class DDIMScheduler:
    order = 1
    _compatibles: List[str] = []

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.00085, beta_end: float = 0.012,
                 beta_schedule: str = "scaled_linear", trained_betas=None, clip_sample: bool = False,
                 set_alpha_to_one: bool = False, steps_offset: int = 1, prediction_type: str = "epsilon",
                 thresholding: bool = False, dynamic_thresholding_ratio: float = 0.995, clip_sample_range: float = 1.0,
                 sample_max_value: float = 1.0, timestep_spacing: str = "leading", rescale_betas_zero_snr: bool = False,
                 **unused):
        if prediction_type != "epsilon":
            raise NotImplementedError("only prediction_type='epsilon' is on the PowerPaint hot path")
        if clip_sample or thresholding or rescale_betas_zero_snr:
            raise NotImplementedError("clip_sample / thresholding / zero-SNR rescale are off in the SD config")
        self.config = Config(
            num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
            beta_schedule=beta_schedule, trained_betas=trained_betas, clip_sample=clip_sample,
            set_alpha_to_one=set_alpha_to_one, steps_offset=steps_offset, prediction_type=prediction_type,
            thresholding=thresholding, dynamic_thresholding_ratio=dynamic_thresholding_ratio,
            clip_sample_range=clip_sample_range, sample_max_value=sample_max_value,
            timestep_spacing=timestep_spacing, rescale_betas_zero_snr=rescale_betas_zero_snr)
        if trained_betas is not None:
            betas = torch.tensor(trained_betas, dtype=torch.float32)
        elif beta_schedule == "linear":
            betas = torch.linspace(beta_start, beta_end, num_train_timesteps, dtype=torch.float32)
        elif beta_schedule == "scaled_linear":
            betas = torch.linspace(beta_start ** 0.5, beta_end ** 0.5, num_train_timesteps, dtype=torch.float32) ** 2
        else:
            raise NotImplementedError(f"beta_schedule {beta_schedule}")
        self.betas = betas
        self.alphas = 1.0 - betas
        self.alphas_cumprod = torch.cumprod(self.alphas, dim=0)
        self.final_alpha_cumprod = torch.tensor(1.0) if set_alpha_to_one else self.alphas_cumprod[0]
        self.init_noise_sigma = 1.0
        self.num_inference_steps: Optional[int] = None
        self.timesteps = torch.from_numpy(np.arange(0, num_train_timesteps)[::-1].copy().astype(np.int64))

    @classmethod
    def from_config(cls, config, **kwargs):
        d = dict(config.__dict__) if hasattr(config, "__dict__") else dict(config)
        d = {k: v for k, v in d.items() if not k.startswith("_")}
        d.update(kwargs)
        return cls(**d)

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder=None, revision=None, local_files_only=False,
                        cache_dir=None, **kwargs):
        """`SchedulerMixin.from_pretrained`: `<dir>[/<subfolder>]/scheduler_config.json` of a checkpoint in the diffusers
        layout (keys of other scheduler classes that have no meaning here are dropped by the constructor)"""
        from .loading import load_json, resolve_checkpoint_dir

        d = resolve_checkpoint_dir(pretrained_model_name_or_path, subfolder, revision, local_files_only, cache_dir)
        return cls.from_config(load_json(d, "scheduler_config.json"), **kwargs)

    def save_pretrained(self, save_directory, **unused):
        import json
        import os

        os.makedirs(save_directory, exist_ok=True)
        cfg = {"_class_name": type(self).__name__, "_diffusers_version": "0.27.0"}
        cfg.update({k: v for k, v in vars(self.config).items() if not k.startswith("_")})
        with open(os.path.join(save_directory, "scheduler_config.json"), "w") as f:
            json.dump(cfg, f, indent=2, sort_keys=True)

    def scale_model_input(self, sample: torch.Tensor, timestep=None) -> torch.Tensor:
        return sample

    def set_timesteps(self, num_inference_steps: int, device: Union[str, torch.device, None] = None):
        c = self.config
        if num_inference_steps > c.num_train_timesteps:
            raise ValueError(f"`num_inference_steps`: {num_inference_steps} cannot be larger than "
                             f"`self.config.train_timesteps`: {c.num_train_timesteps}")
        self.num_inference_steps = num_inference_steps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, c.num_train_timesteps - 1, num_inference_steps).round()[::-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            ratio = c.num_train_timesteps // num_inference_steps
            ts = (np.arange(0, num_inference_steps) * ratio).round()[::-1].copy().astype(np.int64)
            ts += c.steps_offset
        elif c.timestep_spacing == "trailing":
            ratio = c.num_train_timesteps / num_inference_steps
            ts = np.round(np.arange(c.num_train_timesteps, 0, -ratio)).astype(np.int64) - 1
        else:
            raise ValueError(f"{c.timestep_spacing} is not supported")
        self.timesteps = torch.from_numpy(ts).to(device)

    # ---- schedule scalars
    def _alphas(self, timestep: int) -> Tuple[float, float]:
        prev = timestep - self.config.num_train_timesteps // self.num_inference_steps
        a_t = float(self.alphas_cumprod[timestep])
        a_prev = float(self.alphas_cumprod[prev]) if prev >= 0 else float(self.final_alpha_cumprod)
        return a_t, a_prev

    def step_coefficients(self, timesteps=None, eta: float = 0.0) -> torch.Tensor:
        """[n_steps, 8] fp32 rows {sqrt(a_t), sqrt(1-a_t), sqrt(a_prev), sqrt(1-a_prev-sigma^2), sigma,
        0, 0, 0} consumed by pp_cfg_ddim_step (include/powerpaint_b200.h)."""
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        ts = self.timesteps if timesteps is None else timesteps
        rows = []
        for t in [int(x) for x in ts]:
            a_t, a_prev = self._alphas(t)
            var = (1 - a_prev) / (1 - a_t) * (1 - a_t / a_prev)
            sigma = eta * math.sqrt(max(var, 0.0))
            rows.append([math.sqrt(a_t), math.sqrt(1 - a_t), math.sqrt(a_prev),
                         math.sqrt(max(1 - a_prev - sigma * sigma, 0.0)), sigma, 0.0, 0.0, 0.0])
        return torch.tensor(rows, dtype=torch.float32)

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor, eta: float = 0.0,
             use_clipped_model_output: bool = False, generator=None, variance_noise: Optional[torch.Tensor] = None,
             return_dict: bool = True):
        """x_t -> x_{t-1} on CUDA tensors through the fused kernel (no CFG: model_output is used as is)."""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after "
                             "creating the scheduler")
        if not sample.is_cuda:
            raise RuntimeError("DDIMScheduler.step runs in the CUDA kernel pp_cfg_ddim_step; "
                               "CPU tensors are not supported (no CPU fallback on the hot path)")
        from . import ops

        nb, c, h, w = sample.shape
        if c != 4:
            raise ValueError("the fused step kernel handles 4-channel latents")
        coef = self.step_coefficients([int(timestep)], eta).to(sample.device)
        lat = ops.nhwc_fp32_from_nchw(sample)
        eps = ops.nhwc_fp32_from_nchw(model_output)
        noise = None
        if eta > 0:
            if variance_noise is None:
                variance_noise = torch.randn(model_output.shape, generator=generator,
                                             device=generator.device if generator is not None else sample.device,
                                             dtype=torch.float32).to(sample.device)
            noise = ops.nhwc_fp32_from_nchw(variance_noise)
        ops.run(ops.cfg_ddim_desc(eps=eps, eps_fp32=True, eps_ld=4, latents=lat, coef=coef, step_idx=None,
                                  advance_step=False, noise=noise, guidance_scale=1.0, do_cfg=False, batch=nb,
                                  hw=h * w))
        prev = lat.view(nb, h, w, 4).permute(0, 3, 1, 2).contiguous().to(sample.dtype)
        if not return_dict:
            return (prev,)
        # x0 prediction of the output object (diffusers' `pred_original_sample`, epsilon parametrisation); the loop never
        # reads it: one elementwise expression on the caller's tensors, outside the fused kernel
        a_t, _ = self._alphas(int(timestep))
        x0 = ((sample.float() - math.sqrt(1 - a_t) * model_output.float()) / math.sqrt(a_t)).to(sample.dtype)
        return DDIMSchedulerOutput(prev_sample=prev, pred_original_sample=x0)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        a = self.alphas_cumprod.to(original_samples.device)[timesteps.to(original_samples.device)]
        a = a.to(original_samples.dtype)
        while a.dim() < original_samples.dim():
            a = a.unsqueeze(-1)
        return a ** 0.5 * original_samples + (1 - a) ** 0.5 * noise

    def __len__(self):
        return self.config.num_train_timesteps


class UniPCMultistepScheduler(DDIMScheduler):
    """diffusers `UniPCMultistepScheduler` as the v2 app builds it — `UniPCMultistepScheduler.from_config(
    pipe.scheduler.config)` (reference app.py:197): solver_order 2, solver_type "bh2", predict_x0, epsilon
    prediction, lower_order_final, beta schedule / spacing / steps_offset inherited from the DDIM config.

    The multistep predictor-corrector update is linear in the tensors it touches (current sample, last corrected
    sample, the previous x0 predictions), so `unipc_coefficients()` folds the whole schedule (log-SNR steps, the
    B(h) terms, the 2x2 solve of the corrector) into 10 scalars per step, computed in float64 on the host; the
    arithmetic on the latents runs in the fused CFG + UniPC kernel (`pp_unipc_step`), like DDIM's."""

    order = 1
    kind = "unipc"

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False, predict_x0: bool = True,
                 solver_type: str = "bh2", lower_order_final: bool = True, disable_corrector=(),
                 use_karras_sigmas: bool = False, timestep_spacing: str = "linspace", steps_offset: int = 0, **unused):
        if solver_order != 2 or not predict_x0 or solver_type != "bh2" or use_karras_sigmas or disable_corrector:
            raise NotImplementedError("only the app's UniPC configuration is built: solver_order=2, bh2, predict_x0, "
                                      "no Karras sigmas, corrector on")
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, steps_offset=steps_offset,
                         prediction_type=prediction_type, thresholding=thresholding, timestep_spacing=timestep_spacing)
        self.config.solver_order = solver_order
        self.config.predict_x0 = predict_x0
        self.config.solver_type = solver_type
        self.config.lower_order_final = lower_order_final
        self.config.use_karras_sigmas = use_karras_sigmas
        self.sigmas = None
        self._state = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        T = c.num_train_timesteps
        n = num_inference_steps
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            step_ratio = T // (n + 1)
            ts = (np.arange(0, n + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += c.steps_offset
        elif c.timestep_spacing == "trailing":
            step_ratio = T / n
            ts = np.arange(T, 0, -step_ratio).round().copy().astype(np.int64) - 1
        else:
            raise ValueError(f"{c.timestep_spacing} is not supported")
        ac = self.alphas_cumprod.numpy().astype(np.float64)
        sig = ((1 - ac) / ac) ** 0.5
        sig = np.interp(ts, np.arange(0, len(sig)), sig)
        self.sigmas = np.concatenate([sig, [((1 - ac[0]) / ac[0]) ** 0.5]]).astype(np.float32).astype(np.float64)
        self.timesteps = torch.from_numpy(ts).to(device)
        self.num_inference_steps = n
        self._state = None

    def step_coefficients(self, timesteps=None, eta: float = 0.0) -> torch.Tensor:
        """the shared 8-float rows (guidance / side-net scale are filled in by the denoiser); DDIM columns unused"""
        n = len(self.timesteps if timesteps is None else timesteps)
        return torch.zeros(n, 8, dtype=torch.float32)

    def unipc_coefficients(self, first: int = 0) -> torch.Tensor:
        """[n, 12] fp32 rows for `pp_unipc_step` (include/powerpaint_b200.h), starting at schedule index `first`
        (strength < 1 starts part-way: the multistep history then starts empty there, like the reference)."""
        if self.sigmas is None:
            raise ValueError("call set_timesteps first")
        sg = self.sigmas
        n = len(sg) - 1

        def alpha_sigma(s):
            a = 1.0 / math.sqrt(s * s + 1.0)
            return a, s * a

        def lam(s):
            a, st = alpha_sigma(s)
            return math.log(a) - math.log(st)

        rows = []
        lower = 0
        this_order = 1
        for i in range(first, n):
            a_i, s_i = alpha_sigma(sg[i])
            u = [1.0 / a_i, -s_i / a_i, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]
            if i > first:  # corrector with the order chosen at the previous step
                order = this_order
                a_t, s_t = a_i, s_i
                _, s_s0 = alpha_sigma(sg[i - 1])
                h = lam(sg[i]) - lam(sg[i - 1])
                hh = -h
                h_phi_1 = math.expm1(hh)
                B_h = math.expm1(hh)
                h_phi_k = h_phi_1 / hh - 1.0
                if order == 1:
                    rho_last, rho0_over_rk = 0.5, 0.0
                else:
                    rk = (lam(sg[i - 2]) - lam(sg[i - 1])) / h
                    b1 = h_phi_k / B_h
                    b2 = (h_phi_k / hh - 0.5) * 2.0 / B_h
                    # R = [[1, 1], [rk, 1]] rhos = [b1, b2]
                    rho0 = (b1 - b2) / (1.0 - rk)
                    rho_last = b1 - rho0
                    rho0_over_rk = rho0 / rk
                u[2] = 1.0
                u[3] = s_t / s_s0
                u[4] = -a_t * h_phi_1 + a_t * B_h * (rho0_over_rk + rho_last)
                u[5] = -a_t * B_h * rho0_over_rk
                u[6] = -a_t * B_h * rho_last
            order = min(2, n - i) if self.config.lower_order_final else 2
            this_order = min(order, lower + 1)
            # predictor towards sigma[i + 1]
            a_t, s_t = alpha_sigma(sg[i + 1])
            h = lam(sg[i + 1]) - lam(sg[i])
            hh = -h
            h_phi_1 = math.expm1(hh)
            B_h = math.expm1(hh)
            u[7] = s_t / s_i
            u[8] = -a_t * h_phi_1
            if this_order == 2:
                rk = (lam(sg[i - 1]) - lam(sg[i])) / h
                u[8] += a_t * B_h * 0.5 / rk
                u[9] = -a_t * B_h * 0.5 / rk
            if lower < 2:
                lower += 1
            rows.append(u)
        return torch.tensor(rows, dtype=torch.float32)

    def step(self, model_output: torch.Tensor, timestep: int, sample: torch.Tensor, return_dict: bool = True, **unused):
        """eager x_t -> x_{t-1} on CUDA tensors through the fused kernel; keeps the multistep state like diffusers
        (reset by `set_timesteps`)"""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after "
                             "creating the scheduler")
        if not sample.is_cuda:
            raise RuntimeError("UniPCMultistepScheduler.step runs in the CUDA kernel pp_unipc_step; CPU tensors are "
                               "not supported (no CPU fallback on the hot path)")
        from . import ops

        nb, c, h, w = sample.shape
        if c != 4:
            raise ValueError("the fused step kernel handles 4-channel latents")
        st = self._state
        if st is None:
            z = lambda: torch.zeros(nb, h * w, 4, dtype=torch.float32, device=sample.device)  # noqa: E731
            st = self._state = dict(i=0, last=z(), m1=z(), m2=z(), ucoef=self.unipc_coefficients().to(sample.device),
                                    coef=torch.zeros(len(self.sigmas) - 1, 8, device=sample.device),
                                    idx=torch.zeros(1, dtype=torch.int32, device=sample.device))
        st["idx"].fill_(st["i"])
        lat = ops.nhwc_fp32_from_nchw(sample)
        eps = ops.nhwc_fp32_from_nchw(model_output)
        ops.run(ops.unipc_desc(eps=eps, eps_fp32=True, eps_ld=4, latents=lat, last_sample=st["last"], m1=st["m1"],
                               m2=st["m2"], coef=st["coef"], ucoef=st["ucoef"], step_idx=st["idx"], advance_step=False,
                               do_cfg=False, batch=nb, hw=h * w))
        st["i"] += 1
        prev = lat.view(nb, h, w, 4).permute(0, 3, 1, 2).contiguous().to(sample.dtype)
        if not return_dict:
            return (prev,)
        return DDIMSchedulerOutput(prev_sample=prev)


# ---------------------------------------------------------------------------------------------------------------------
# DPM-Solver++ and Euler / Euler-ancestral: one folded row per step for `pp_solver_step`
# ---------------------------------------------------------------------------------------------------------------------
def _sigma_to_t(sigma: float, log_sigmas: np.ndarray) -> float:
    """diffusers' `_sigma_to_t`: the (fractional) training timestep whose sigma is `sigma`, by linear interpolation of
    log sigma between the two neighbouring training steps"""
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    return float(((1 - w) * low_idx + w * high_idx).reshape(np.shape(sigma)))


def karras_sigmas(sigma_min: float, sigma_max: float, n: int, rho: float = 7.0) -> np.ndarray:
    """Karras et al. (2022) eq. 5: n sigmas from sigma_max down to sigma_min, evenly spaced in sigma^(1/rho)"""
    ramp = np.linspace(0, 1, n)
    min_inv_rho, max_inv_rho = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
    return (max_inv_rho + ramp * (min_inv_rho - max_inv_rho)) ** rho


class _SolverScheduler(DDIMScheduler):
    """Shared surface of the schedulers stepped by `pp_solver_step`. `solver_coefficients(first)` folds every step into
    one row of 8 scalars (include/powerpaint_b200.h, pp_solver_desc), computed in float64 from the fp32 sigma table:

        m_t = r0 x + r1 eps;  x_next = r2 x + r3 m_t + r4 m1 + r5 noise;  next input = r6 x_next;  r7 = input scale

    Subclasses set `self.sigmas` (float64 holding the fp32 values diffusers keeps, one more than the steps) and
    `self.timesteps` in `set_timesteps`, and implement `_rows(first)`."""

    kind = "solver"
    order = 1
    #: the update uses fresh Gaussian noise every step (SDE / ancestral variants)
    stochastic = False
    #: diffusers' `step` draws one `randn_tensor(model_output.shape)` per call (used or not)
    draws_noise = False

    def _base_init(self, num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas, prediction_type,
                   thresholding, timestep_spacing, steps_offset, rescale_betas_zero_snr, config: dict):
        if timestep_spacing not in ("linspace", "leading", "trailing"):
            raise NotImplementedError(f"timestep_spacing={timestep_spacing!r}: linspace, leading and trailing are built")
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, prediction_type=prediction_type,
                         thresholding=thresholding, timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                         rescale_betas_zero_snr=rescale_betas_zero_snr)
        self.config = Config(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                                   beta_schedule=beta_schedule, trained_betas=trained_betas,
                                   prediction_type=prediction_type, thresholding=thresholding,
                                   timestep_spacing=timestep_spacing, steps_offset=steps_offset,
                                   rescale_betas_zero_snr=rescale_betas_zero_snr, **config)
        # ((1 - a) / a) ** 0.5 in fp32 torch, as diffusers computes it
        self._train_sigmas = np.array(((1 - self.alphas_cumprod) / self.alphas_cumprod) ** 0.5)
        self.sigmas: Optional[np.ndarray] = None
        self._state = None

    def _finish_set_timesteps(self, timesteps, sigmas, device):
        self.sigmas = np.asarray(sigmas, dtype=np.float32).astype(np.float64)
        self.timesteps = torch.from_numpy(np.asarray(timesteps)).to(device)
        self.num_inference_steps = len(self.timesteps)
        self._state = None

    def step_coefficients(self, timesteps=None, eta: float = 0.0) -> torch.Tensor:
        """the shared 8-float rows (guidance / side-net scale are filled in by the denoiser); DDIM columns unused"""
        n = len(self.timesteps if timesteps is None else timesteps)
        return torch.zeros(n, 8, dtype=torch.float32)

    def index_for_timestep(self, timestep) -> int:
        """diffusers' `index_for_timestep`: the second match when a timestep repeats, so a schedule that starts
        part-way (strength < 1) does not skip a step"""
        idx = (self.timesteps.cpu() == torch.as_tensor(timestep).cpu().to(self.timesteps.dtype)).nonzero()
        if len(idx) == 0:
            raise ValueError(f"timestep {timestep} is not in the schedule")
        return int(idx[1 if len(idx) > 1 else 0])

    def solver_coefficients(self, first: int = 0) -> torch.Tensor:
        """[n - first, 8] fp32 rows for `pp_solver_step`, starting at schedule index `first` (strength < 1 starts
        part-way; the multistep history then starts empty there, like the reference's scheduler)"""
        if self.sigmas is None:
            raise ValueError("call set_timesteps first")
        return torch.tensor(self._rows(first), dtype=torch.float32)

    def input_scale(self, index: int) -> float:
        """`scale_model_input` factor of schedule index `index`"""
        return 1.0

    def scale_model_input(self, sample: torch.Tensor, timestep=None) -> torch.Tensor:
        if self.sigmas is None:
            raise ValueError("call set_timesteps first")
        i = self._state["i"] if self._state is not None else self.index_for_timestep(timestep)
        return sample * self.input_scale(i)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, generator=None,
             return_dict: bool = True, **unused):
        """eager x_t -> x_{t-1} on CUDA tensors through `pp_solver_step`; keeps the multistep state like diffusers (its
        step index starts at `timestep`'s place in the schedule, reset by `set_timesteps`). Stochastic variants draw
        their noise as diffusers does: one `randn_tensor(model_output.shape, generator=generator)` per call."""
        if self.sigmas is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after "
                             "creating the scheduler")
        if not sample.is_cuda:
            raise RuntimeError(f"{type(self).__name__}.step runs in the CUDA kernel pp_solver_step; CPU tensors are "
                               "not supported (no CPU fallback on the hot path)")
        from . import ops
        from .pipelines.common import randn_tensor

        nb, c, h, w = sample.shape
        if c != 4:
            raise ValueError("the fused step kernel handles 4-channel latents")
        st = self._state
        if st is None:
            first = self.index_for_timestep(timestep)
            st = self._state = dict(i=first, first=first,
                                    m1=torch.zeros(nb, h * w, 4, dtype=torch.float32, device=sample.device),
                                    scoef=self.solver_coefficients(first).to(sample.device),
                                    coef=torch.zeros(len(self.timesteps) - first, 8, device=sample.device),
                                    idx=torch.zeros(1, dtype=torch.int32, device=sample.device))
        if st["i"] >= len(self.timesteps):
            raise ValueError("step called more often than the schedule has steps")
        st["idx"].fill_(st["i"] - st["first"])
        noise = None
        if self.draws_noise:
            drawn = randn_tensor(model_output.shape, generator=generator, device=model_output.device,
                                 dtype=model_output.dtype)
            if self.stochastic:
                noise = ops.nhwc_fp32_from_nchw(drawn)
        lat = ops.nhwc_fp32_from_nchw(sample)
        if lat.untyped_storage().data_ptr() == sample.untyped_storage().data_ptr():
            lat = lat.clone()  # an fp32 channels_last sample: the kernel updates `lat` in place, never the caller's
        eps = ops.nhwc_fp32_from_nchw(model_output)
        ops.run(ops.solver_desc(eps=eps, eps_fp32=True, eps_ld=4, latents=lat, m1=st["m1"], coef=st["coef"],
                                scoef=st["scoef"], step_idx=st["idx"], advance_step=False, do_cfg=False, batch=nb,
                                hw=h * w, noise=noise))
        st["i"] += 1
        prev = lat.view(nb, h, w, 4).permute(0, 3, 1, 2).contiguous().to(sample.dtype)
        if not return_dict:
            return (prev,)
        return DDIMSchedulerOutput(prev_sample=prev)

    def _add_noise_sigmas(self, timesteps: torch.Tensor) -> torch.Tensor:
        return torch.tensor([self.sigmas[self.index_for_timestep(t)] for t in timesteps.reshape(-1).cpu()],
                            dtype=torch.float32)

    def _spaced_timesteps(self, n: int, dtype) -> np.ndarray:
        """the three `timestep_spacing` rules of diffusers' Euler schedulers (n timesteps, no terminal one)"""
        c = self.config
        T = c.num_train_timesteps
        if c.timestep_spacing == "linspace":
            return np.linspace(0, T - 1, n, dtype=dtype)[::-1].copy()
        if c.timestep_spacing == "leading":
            ratio = T // n
            return (np.arange(0, n) * ratio).round()[::-1].copy().astype(dtype) + c.steps_offset
        ratio = T / n
        return np.arange(T, 0, -ratio).round().copy().astype(dtype) - 1


class DPMSolverMultistepScheduler(_SolverScheduler):
    """diffusers `DPMSolverMultistepScheduler` (DPM-Solver++, Lu et al. 2022) for epsilon prediction:
    algorithm_type `dpmsolver++` / `sde-dpmsolver++`, solver_order 1 / 2, solver_type `midpoint` / `heun`,
    `lower_order_final`, `euler_at_final`, Karras sigmas, `final_sigmas_type` `zero` / `sigma_min`. The latent is VP
    (x = alpha x0 + sigma eps, model input = x). Timesteps, sigmas and the update restate diffusers 0.27.0
    (schedulers/scheduling_dpmsolver_multistep.py) as recalled from its published source — they cannot be run here;
    oracle/dpmsolver.py restates the same step by step, and tests/test_solver_schedulers_cpu.py holds both to the
    orders of accuracy of the mathematics. One deliberate difference: a step of length zero (Karras sigmas end at
    sigma_min, and `final_sigmas_type="sigma_min"` appends it again) is the identity here, where diffusers' heun
    update evaluates 0 / 0."""

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, solver_order: int = 2,
                 prediction_type: str = "epsilon", thresholding: bool = False, algorithm_type: str = "dpmsolver++",
                 solver_type: str = "midpoint", lower_order_final: bool = True, euler_at_final: bool = False,
                 use_karras_sigmas: bool = False, use_lu_lambdas: bool = False, final_sigmas_type: str = "zero",
                 lambda_min_clipped: float = -float("inf"), variance_type=None, timestep_spacing: str = "linspace",
                 steps_offset: int = 0, rescale_betas_zero_snr: bool = False, **unused):
        if algorithm_type not in ("dpmsolver++", "sde-dpmsolver++"):
            raise NotImplementedError(f"algorithm_type={algorithm_type!r}: dpmsolver++ and sde-dpmsolver++ are built")
        if solver_order not in (1, 2):
            raise NotImplementedError(f"solver_order={solver_order}: orders 1 and 2 are built")
        if solver_type in ("logrho", "bh1", "bh2"):  # diffusers maps the UniPC names onto midpoint
            solver_type = "midpoint"
        if solver_type not in ("midpoint", "heun"):
            raise NotImplementedError(f"solver_type={solver_type!r}: midpoint and heun are built")
        if use_lu_lambdas:
            raise NotImplementedError("use_lu_lambdas is not built")
        if final_sigmas_type not in ("zero", "sigma_min"):
            raise NotImplementedError(f"final_sigmas_type={final_sigmas_type!r}: zero and sigma_min are built")
        if variance_type is not None:
            raise NotImplementedError(f"variance_type={variance_type!r}: only epsilon prediction without a learned "
                                      "variance is built")
        self._base_init(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas, prediction_type,
                        thresholding, timestep_spacing, steps_offset, rescale_betas_zero_snr,
                        dict(solver_order=solver_order, algorithm_type=algorithm_type, solver_type=solver_type,
                             lower_order_final=lower_order_final, euler_at_final=euler_at_final,
                             use_karras_sigmas=use_karras_sigmas, use_lu_lambdas=use_lu_lambdas,
                             final_sigmas_type=final_sigmas_type, lambda_min_clipped=lambda_min_clipped,
                             variance_type=variance_type))
        self.stochastic = self.draws_noise = algorithm_type == "sde-dpmsolver++"

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        n = num_inference_steps
        ac = self.alphas_cumprod
        lambda_t = torch.log(ac ** 0.5) - torch.log((1 - ac) ** 0.5)
        clipped_idx = torch.searchsorted(torch.flip(lambda_t, [0]), c.lambda_min_clipped)
        last = int((c.num_train_timesteps - clipped_idx).numpy().item())
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, last - 1, n + 1).round()[::-1][:-1].copy().astype(np.int64)
        elif c.timestep_spacing == "leading":
            step_ratio = last // (n + 1)
            ts = (np.arange(0, n + 1) * step_ratio).round()[::-1][:-1].copy().astype(np.int64)
            ts += c.steps_offset
        else:
            step_ratio = c.num_train_timesteps / n
            ts = np.arange(last, 0, -step_ratio).round().copy().astype(np.int64) - 1
        sig = self._train_sigmas
        if c.use_karras_sigmas:
            sig = karras_sigmas(float(sig[0]), float(sig[-1]), n)
            ts = np.array([_sigma_to_t(s, np.log(self._train_sigmas)) for s in sig]).round().astype(np.int64)
        else:
            sig = np.interp(ts, np.arange(0, len(sig)), sig)
        last_sigma = float(self._train_sigmas[0]) if c.final_sigmas_type == "sigma_min" else 0.0
        self._finish_set_timesteps(ts, np.concatenate([sig, [last_sigma]]), device)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        """x = alpha x0 + sigma eps at the schedule's sigma of each timestep"""
        s = self._add_noise_sigmas(timesteps).to(original_samples.device, original_samples.dtype)
        a = 1 / (s ** 2 + 1) ** 0.5
        s = s * a
        while a.dim() < original_samples.dim():
            a, s = a.unsqueeze(-1), s.unsqueeze(-1)
        return a * original_samples + s * noise

    def _rows(self, first: int):
        c = self.config
        sg = self.sigmas
        n = len(sg) - 1
        sde = c.algorithm_type == "sde-dpmsolver++"

        def alpha_sigma(s):
            a = 1.0 / math.sqrt(s * s + 1.0)
            return a, s * a

        def lam(s):
            a, st = alpha_sigma(s)
            return math.log(a) - math.log(st)

        rows, lower = [], 0
        for i in range(first, n):
            a_s, s_s = alpha_sigma(sg[i])
            a_t, s_t = alpha_sigma(sg[i + 1])
            r = [1.0 / a_s, -s_s / a_s, 0.0, 0.0, 0.0, 0.0, 1.0, 1.0]
            final = i == n - 1 and (c.euler_at_final or (c.lower_order_final and n < 15)
                                    or c.final_sigmas_type == "zero")
            if s_t == 0.0:  # final sigma zero: h = inf, exp(-h) = 0
                h, e = math.inf, 0.0
            else:
                h = lam(sg[i + 1]) - lam(sg[i])
                e = math.exp(-h)
            r[2] = s_t / s_s * (e if sde else 1.0)
            if sde:
                r[5] = s_t * math.sqrt(1.0 - e * e)
            A = a_t * (1.0 - e * e) if sde else -a_t * (e - 1.0)  # coefficient of D0 = m_t
            if h == 0.0:  # Karras sigmas ending at sigma_min, then final_sigmas_type sigma_min: a step of length 0
                r[2:6] = [1.0, 0.0, 0.0, 0.0]
            elif c.solver_order == 1 or lower < 1 or final:
                r[3] = A
            else:
                rr = (lam(sg[i]) - lam(sg[i - 1])) / h
                if c.solver_type == "midpoint":
                    b = 0.5 * A
                elif sde:
                    b = a_t * ((1.0 - e * e) / (-2.0 * h) + 1.0)
                else:
                    b = a_t * ((e - 1.0) / h + 1.0)
                # D1 = (m_t - m1) / rr
                r[3] = A + b / rr
                r[4] = -b / rr
            lower = min(lower + 1, c.solver_order)
            rows.append(r)
        return rows


class EulerDiscreteScheduler(_SolverScheduler):
    """diffusers `EulerDiscreteScheduler` (Karras et al. 2022, Algorithm 2 with s_churn = 0) for epsilon prediction,
    linear sigma interpolation, optional Karras sigmas, the three timestep spacings. The latent is VE
    (x = x0 + s eps, model input = x / sqrt(s^2 + 1), `init_noise_sigma` != 1); timesteps can be fractional (Karras)
    and reach the UNet unrounded. Restates diffusers 0.27.0 (schedulers/scheduling_euler_discrete.py) as recalled from
    its published source; oracle/euler.py restates the same step by step. diffusers' `step` draws one noise tensor
    per call even at s_churn = 0 and discards it; `draws_noise` reports that so a caller can keep a generator's
    stream where the reference leaves it."""

    _linspace_dtype = np.float32
    _karras_config = True

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, prediction_type: str = "epsilon",
                 interpolation_type: str = "linear", use_karras_sigmas: bool = False, sigma_min=None, sigma_max=None,
                 timestep_spacing: str = "linspace", timestep_type: str = "discrete", steps_offset: int = 0,
                 rescale_betas_zero_snr: bool = False, **unused):
        if interpolation_type != "linear":
            raise NotImplementedError(f"interpolation_type={interpolation_type!r}: linear is built")
        if timestep_type != "discrete":
            raise NotImplementedError(f"timestep_type={timestep_type!r}: discrete is built")
        self._base_init(num_train_timesteps, beta_start, beta_end, beta_schedule, trained_betas, prediction_type,
                        False, timestep_spacing, steps_offset, rescale_betas_zero_snr,
                        dict(interpolation_type=interpolation_type, use_karras_sigmas=use_karras_sigmas,
                             sigma_min=sigma_min, sigma_max=sigma_max, timestep_type=timestep_type))
        del self.config.thresholding
        self.draws_noise = True
        self.init_noise_sigma = self._init_noise_sigma(float(self._train_sigmas.max()))

    def _init_noise_sigma(self, max_sigma: float) -> float:
        if self.config.timestep_spacing in ("linspace", "trailing"):
            return max_sigma
        return (max_sigma ** 2 + 1) ** 0.5

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        n = num_inference_steps
        ts = self._spaced_timesteps(n, self._linspace_dtype)
        sig = np.interp(ts, np.arange(0, len(self._train_sigmas)), self._train_sigmas)
        if c.use_karras_sigmas:
            smin = c.get("sigma_min") if self._karras_config else None
            smax = c.get("sigma_max") if self._karras_config else None
            sig = karras_sigmas(float(sig[-1]) if smin is None else smin, float(sig[0]) if smax is None else smax, n)
            ts = np.array([_sigma_to_t(s, np.log(self._train_sigmas)) for s in sig])
        ts = np.asarray(ts, dtype=np.float32)
        self._finish_set_timesteps(ts, np.concatenate([sig, [0.0]]), device)
        self.init_noise_sigma = self._init_noise_sigma(float(self.sigmas.max()))

    def input_scale(self, index: int) -> float:
        return 1.0 / math.sqrt(self.sigmas[index] ** 2 + 1.0)

    def add_noise(self, original_samples: torch.Tensor, noise: torch.Tensor, timesteps: torch.Tensor) -> torch.Tensor:
        """x = x0 + s eps at the schedule's sigma of each timestep"""
        s = self._add_noise_sigmas(timesteps).to(original_samples.device, original_samples.dtype)
        while s.dim() < original_samples.dim():
            s = s.unsqueeze(-1)
        return original_samples + noise * s

    def _update(self, s: float, s_next: float, r: list):
        r[2] = s_next / s
        r[3] = 1.0 - s_next / s

    def _rows(self, first: int):
        sg = self.sigmas
        rows = []
        for i in range(first, len(sg) - 1):
            s, s_next = sg[i], sg[i + 1]
            r = [1.0, -s, 0.0, 0.0, 0.0, 0.0, self.input_scale(i + 1), self.input_scale(i)]
            self._update(s, s_next, r)
            rows.append(r)
        return rows


class EulerAncestralDiscreteScheduler(EulerDiscreteScheduler):
    """diffusers `EulerAncestralDiscreteScheduler` for epsilon prediction: the Euler step to sigma_down plus fresh
    noise of scale sigma_up (sigma_up^2 + sigma_down^2 = sigma_next^2), VE latent, the same schedule options as
    `EulerDiscreteScheduler`. Restates diffusers 0.27.0 (schedulers/scheduling_euler_ancestral_discrete.py) as
    recalled from its published source (linspace timesteps in float64 there, float32 in the Euler scheduler)."""

    _linspace_dtype = np.float64
    _karras_config = False

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.stochastic = True

    def _update(self, s: float, s_next: float, r: list):
        s_up = math.sqrt(s_next ** 2 * (s ** 2 - s_next ** 2) / s ** 2)
        s_down = math.sqrt(s_next ** 2 - s_up ** 2)
        r[2] = s_down / s
        r[3] = 1.0 - s_down / s
        r[5] = s_up


# ---------------------------------------------------------------------------------------------------------------------
# PNDM with skip_prk_steps (PLMS): one folded row per step for `pp_plms_step`
# ---------------------------------------------------------------------------------------------------------------------
PLMS_RING = 3  # physical eps history slots: a 4-entry Adams-Bashforth step reads the 3 previous entries


class _PlmsFold:
    """The state machine of diffusers' `PNDMScheduler.step_plms`, run on symbols instead of tensors: `row(t)` returns
    the step at timestep `t` as one row of 8 floats for `pp_plms_step`

        x_next = r0 x + r1 cur_sample + r2 eps + r3 ets[0] + r4 ets[1] + r5 ets[2]
        ets[r6] <- eps (r6 >= 0);  cur_sample <- x (r7 != 0)

    Appended history entries go to slots 0, 1, 2, 0, ... so a new entry replaces the oldest of the three it can
    see, which this step reads before the kernel writes it. `alpha(t)` is alpha_bar as diffusers indexes it."""

    AB = {1: (1.0,), 2: (3 / 2, -1 / 2), 3: (23 / 12, -16 / 12, 5 / 12), 4: (55 / 24, -59 / 24, 37 / 24, -9 / 24)}

    def __init__(self, ratio: int, alpha, final_alpha: float):
        self.ratio, self.alpha, self.final_alpha = ratio, alpha, final_alpha
        self.counter = 0
        self.appended = 0
        self.hist: List[int] = []  # slots of the remembered eps, oldest first (at most 3)

    def row(self, timestep) -> List[float]:
        t = int(timestep)
        prev = t - self.ratio
        r = [0.0] * 8
        r[6] = -1.0
        old = self.hist[-3:]
        if self.counter != 1:
            slot = self.appended % PLMS_RING
            r[6] = float(slot)
            self.hist = (old + [slot])[-PLMS_RING:]
            self.appended += 1
            weights = self.AB[len(old) + 1]
        else:  # Heun restart: average with the first eps, from the sample the first step started at
            prev, t = t, t + self.ratio
            weights = (0.5, 0.5)
            old = old[-1:]
        a_t = self.alpha(t)
        a_p = self.alpha(prev) if prev >= 0 else self.final_alpha
        sc = math.sqrt(a_p / a_t)
        k = (a_p - a_t) / (a_t * math.sqrt(1 - a_p) + math.sqrt(a_t * (1 - a_t) * a_p))
        r[1 if self.counter == 1 else 0] = sc
        r[7] = 1.0 if self.counter == 0 else 0.0
        r[2] = -k * weights[0]
        for w, s in zip(weights[1:], reversed(old)):  # weights[1] belongs to the newest remembered entry
            r[3 + s] += -k * w
        self.counter += 1
        return r


class PNDMScheduler(DDIMScheduler):
    """diffusers `PNDMScheduler` with `skip_prk_steps=True` (PLMS), the scheduler the SD-1.5 inpainting checkpoint
    stores and the v1 app samples with (reference app.py:91-93): N inference steps make N + 1 UNet evaluations, a
    first Euler-like step, a Heun restart from the first step's sample (counter 1), then Adams-Bashforth of order
    2, 3 and 4 on the guided eps. Restates diffusers 0.27.0 (schedulers/scheduling_pndm.py) as recalled from its
    published source; oracle/pndm.py restates the same step by step. The Runge-Kutta warm-up (`skip_prk_steps=False`,
    diffusers' default, used by no stored SD-1.x configuration) and v-prediction are not built.

    Every step is linear in (x, the first step's sample, the new eps, up to 3 earlier eps), with weights that depend
    on the step index only, so `plms_coefficients()` folds the schedule into one 8-float row per step (`_PlmsFold`)
    and the arithmetic on the latents runs in the fused CFG + PLMS kernel (`pp_plms_step`)."""

    order = 1
    kind = "plms"

    def __init__(self, num_train_timesteps: int = 1000, beta_start: float = 0.0001, beta_end: float = 0.02,
                 beta_schedule: str = "linear", trained_betas=None, skip_prk_steps: bool = False,
                 set_alpha_to_one: bool = False, prediction_type: str = "epsilon", timestep_spacing: str = "leading",
                 steps_offset: int = 0, **unused):
        if not skip_prk_steps:
            raise NotImplementedError("skip_prk_steps=False (the Runge-Kutta warm-up) is not built: PLMS with "
                                      "skip_prk_steps=True is, as stored by the SD-1.x checkpoints")
        if prediction_type != "epsilon":
            raise NotImplementedError(f"prediction_type={prediction_type!r}: only epsilon prediction is built")
        if timestep_spacing not in ("linspace", "leading", "trailing"):
            raise NotImplementedError(f"timestep_spacing={timestep_spacing!r}: linspace, leading and trailing are built")
        super().__init__(num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
                         beta_schedule=beta_schedule, trained_betas=trained_betas, set_alpha_to_one=set_alpha_to_one,
                         steps_offset=steps_offset, prediction_type=prediction_type, timestep_spacing=timestep_spacing)
        self.config = Config(
            num_train_timesteps=num_train_timesteps, beta_start=beta_start, beta_end=beta_end,
            beta_schedule=beta_schedule, trained_betas=trained_betas, skip_prk_steps=skip_prk_steps,
            set_alpha_to_one=set_alpha_to_one, prediction_type=prediction_type, timestep_spacing=timestep_spacing,
            steps_offset=steps_offset)
        self._state = None

    def set_timesteps(self, num_inference_steps: int, device=None):
        c = self.config
        T, n = c.num_train_timesteps, num_inference_steps
        if n > T:
            raise ValueError(f"`num_inference_steps`: {n} cannot be larger than `self.config.train_timesteps`: {T}")
        self.num_inference_steps = n
        if c.timestep_spacing == "linspace":
            ts = np.linspace(0, T - 1, n).round().astype(np.int64)
        elif c.timestep_spacing == "leading":
            ts = (np.arange(0, n) * (T // n)).round().astype(np.int64) + c.steps_offset
        else:
            ts = np.round(np.arange(T, 0, -T / n))[::-1].astype(np.int64) - 1
        # the last-but-one timestep is repeated: the Heun restart evaluates the net there a second time
        plms = np.concatenate([ts[:-1], ts[-2:-1], ts[-1:]])[::-1].copy()
        self.timesteps = torch.from_numpy(plms.astype(np.int64)).to(device)
        self._state = None

    def step_coefficients(self, timesteps=None, eta: float = 0.0) -> torch.Tensor:
        """the shared 8-float rows (guidance / side-net scale / blend are filled in by the denoiser); DDIM columns
        unused"""
        n = len(self.timesteps if timesteps is None else timesteps)
        return torch.zeros(n, 8, dtype=torch.float32)

    def _fold(self) -> _PlmsFold:
        ac = self.alphas_cumprod
        return _PlmsFold(self.config.num_train_timesteps // self.num_inference_steps, lambda t: float(ac[t]),
                         float(self.final_alpha_cumprod))

    def plms_coefficients(self, first: int = 0, dtype=torch.float32) -> torch.Tensor:
        """[len(timesteps) - first, 8] rows for `pp_plms_step` (folded in float64, returned as `dtype`), starting at
        schedule index `first` (strength < 1 slices the schedule; the step counter and the history then start at 0
        there, like diffusers' scheduler)"""
        if self.num_inference_steps is None:
            raise ValueError("call set_timesteps first")
        fold = self._fold()
        return torch.tensor([fold.row(t) for t in self.timesteps[first:].tolist()], dtype=dtype)

    def step(self, model_output: torch.Tensor, timestep, sample: torch.Tensor, return_dict: bool = True):
        """eager x_t -> x_{t-1} on CUDA tensors through `pp_plms_step`; keeps diffusers' counter and eps history
        (reset by `set_timesteps`)"""
        if self.num_inference_steps is None:
            raise ValueError("Number of inference steps is 'None', you need to run 'set_timesteps' after "
                             "creating the scheduler")
        if not sample.is_cuda:
            raise RuntimeError("PNDMScheduler.step runs in the CUDA kernel pp_plms_step; CPU tensors are not "
                               "supported (no CPU fallback on the hot path)")
        from . import ops

        nb, c, h, w = sample.shape
        if c != 4:
            raise ValueError("the fused step kernel handles 4-channel latents")
        st = self._state
        if st is None or st["shape"] != (nb, h, w) or st["device"] != sample.device:
            z = lambda *s: torch.zeros(*s, nb, h * w, 4, dtype=torch.float32, device=sample.device)  # noqa: E731
            st = self._state = dict(fold=self._fold() if st is None else st["fold"], shape=(nb, h, w),
                                    device=sample.device, cur=z(), ets=z(PLMS_RING),
                                    coef=torch.zeros(1, 8, device=sample.device))
        row = torch.tensor([st["fold"].row(timestep)], dtype=torch.float32).to(sample.device)
        lat = ops.nhwc_fp32_from_nchw(sample)
        if lat.untyped_storage().data_ptr() == sample.untyped_storage().data_ptr():
            lat = lat.clone()  # an fp32 channels_last sample: the kernel updates `lat` in place, never the caller's
        eps = ops.nhwc_fp32_from_nchw(model_output)
        ops.run(ops.plms_desc(eps=eps, eps_fp32=True, eps_ld=4, latents=lat, cur_sample=st["cur"], ets=st["ets"],
                              coef=st["coef"], pcoef=row, step_idx=None, advance_step=False, do_cfg=False, batch=nb,
                              hw=h * w))
        prev = lat.view(nb, h, w, 4).permute(0, 3, 1, 2).contiguous().to(sample.dtype)
        if not return_dict:
            return (prev,)
        return DDIMSchedulerOutput(prev_sample=prev)
