"""`StableDiffusionControlNetInpaintPipeline` (PowerPaint v1 + ControlNet) — drop-in for the
reference class (powerpaint/pipelines/pipeline_PowerPaint_ControlNet.py:225; `__call__` :1347-1771).
The loop (:1663-1735: ControlNet on the 4-channel latents + control image, 9-channel UNet with the
12 down residuals + mid residual, CFG, scheduler.step) runs as one recorded CUDA program per step
(`FusedDenoiser(mode="controlnet")`); the t-independent `controlnet_cond_embedding(control_image)`
is evaluated once per call instead of once per step (SURVEY.md App. C (3)).

Several ControlNets (a list, wrapped in `MultiControlNetModel` as :306 does), `guess_mode` and pooled
(`global_pool_conditions`) ControlNets run on the same fused loop (see `powerpaint_b200.denoise`).

Out of scope like upstream's dead code: `predict_woControl` (:996-1345, a buggy copy of the v1 `__call__`).
"""
from __future__ import annotations

import logging
from typing import Callable, List, Optional, Union

import torch

from ..denoise import FusedDenoiser
from ..models.unet_2d_condition import ControlNetModel, MultiControlNetModel, UNet2DConditionModel
from .common import (LoopInputs, callback_fires, check_control_guidance, check_image, check_prompt_arguments,
                     prepare_mask_and_masked_image, preprocess_image,
                     randn_tensor, solver_loop_inputs, step_noise, uint8_device_inputs)
from .pipeline_PowerPaint import StableDiffusionInpaintPipeline

logger = logging.getLogger(__name__)


class StableDiffusionControlNetInpaintPipeline(StableDiffusionInpaintPipeline):
    def __init__(self, vae, text_encoder, tokenizer, unet, controlnet, scheduler, safety_checker=None,
                 feature_extractor=None, requires_safety_checker: bool = False):
        super().__init__(vae, text_encoder, tokenizer, unet, scheduler, safety_checker, feature_extractor,
                         requires_safety_checker)
        if isinstance(controlnet, (list, tuple)):
            controlnet = MultiControlNetModel(controlnet)
        self.controlnet = controlnet
        self._denoiser_side = None

    def denoiser(self) -> FusedDenoiser:
        nets = self.controlnet.nets if isinstance(self.controlnet, MultiControlNetModel) else [self.controlnet]
        if not isinstance(self.unet, UNet2DConditionModel) or not all(isinstance(n, ControlNetModel) for n in nets):
            assert False, "unet / controlnet must be powerpaint_b200 UNet2DConditionModel / ControlNetModel(s)"
        if self._denoiser is None or self._denoiser_unet is not self.unet or self._denoiser_side is not self.controlnet:
            self._denoiser = FusedDenoiser(self.unet, self.controlnet, mode="controlnet")
            self._denoiser_unet, self._denoiser_side = self.unet, self.controlnet
        return self._denoiser

    def check_inputs_controlnet(self, prompt, image, height, width, callback_steps, negative_prompt=None,
                                prompt_embeds=None, negative_prompt_embeds=None, controlnet_conditioning_scale=1.0,
                                control_guidance_start=0.0, control_guidance_end=1.0):
        """the reference's `check_inputs` (:651-786; `image` = the control image) in its order, same exception types
        and messages. Unlike the v1 pipeline it does not look at `strength`."""
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if callback_steps is None or not isinstance(callback_steps, int) or callback_steps <= 0:
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type"
                             f" {type(callback_steps)}.")
        check_prompt_arguments(prompt, negative_prompt, prompt_embeds, negative_prompt_embeds)
        multi = isinstance(self.controlnet, MultiControlNetModel)
        if multi and isinstance(prompt, list):
            logger.warning(f"You have {len(self.controlnet.nets)} ControlNets and you have passed {len(prompt)}"
                           " prompts. The conditionings will be fixed across the prompts.")
        if isinstance(self.controlnet, ControlNetModel):
            check_image(image, prompt, prompt_embeds)
        elif multi:
            if not isinstance(image, list):
                raise TypeError("For multiple controlnets: `image` must be type `list`")
            elif any(isinstance(i, list) for i in image):
                raise ValueError("A single batch of multiple conditionings are supported at the moment.")
            elif len(image) != len(self.controlnet.nets):
                raise ValueError("For multiple controlnets: `image` must have the same length as the number of "
                                 f"controlnets, but got {len(image)} images and {len(self.controlnet.nets)} "
                                 "ControlNets.")
            for image_ in image:
                check_image(image_, prompt, prompt_embeds)
        else:
            assert False
        if isinstance(self.controlnet, ControlNetModel):
            if not isinstance(controlnet_conditioning_scale, float):
                raise TypeError("For single controlnet: `controlnet_conditioning_scale` must be type `float`.")
        elif isinstance(controlnet_conditioning_scale, list):
            # the reference's length check sits in an `elif` its `if` always shadows, so a scale list of the wrong
            # length passes here (and `zip` later drops the nets it has no scale for)
            if any(isinstance(i, list) for i in controlnet_conditioning_scale):
                raise ValueError("A single batch of multiple conditionings are supported at the moment.")
        if len(control_guidance_start) != len(control_guidance_end):
            raise ValueError(f"`control_guidance_start` has {len(control_guidance_start)} elements, but "
                             f"`control_guidance_end` has {len(control_guidance_end)} elements. Make sure to provide "
                             "the same number of elements to each list.")
        if multi and len(control_guidance_start) != len(self.controlnet.nets):
            n = len(self.controlnet.nets)
            raise ValueError(f"`control_guidance_start`: {control_guidance_start} has {len(control_guidance_start)} "
                             f"elements but there are {n} controlnets available. Make sure to provide {n}.")
        check_control_guidance(control_guidance_start, control_guidance_end)

    def check_image(self, image, prompt, prompt_embeds):
        """ref:pipeline_PowerPaint_ControlNet.py:788-827"""
        check_image(image, prompt, prompt_embeds)

    def _default_height_width(self, height, width, image):
        """missing sizes come from the init image, rounded down to a multiple of 8 (:914-937)"""
        while isinstance(image, list):
            image = image[0]
        if height is None:
            height = image.height if hasattr(image, "height") else image.shape[2]
            height = (height // 8) * 8
        if width is None:
            width = image.width if hasattr(image, "width") else image.shape[3]
            width = (width // 8) * 8
        return height, width

    def prepare_control_image(self, image, width, height, batch_size, num_images_per_prompt, device, dtype,
                              do_classifier_free_guidance=False, guess_mode=False):
        """control images are NOT normalised to [-1, 1] (do_normalize=False, :320-322)"""
        image = preprocess_image(image, height=height, width=width, do_normalize=False).to(dtype=torch.float32)
        repeat_by = batch_size if image.shape[0] == 1 else num_images_per_prompt
        image = image.repeat_interleave(repeat_by, dim=0).to(device=device, dtype=dtype)
        if do_classifier_free_guidance and not guess_mode:
            image = torch.cat([image] * 2)
        return image

    @torch.no_grad()
    def prepare_loop(self, promptA: Union[str, List[str]] = None, promptB: Union[str, List[str]] = None, image=None,
                 mask=None, control_image=None, height: Optional[int] = None, width: Optional[int] = None,
                 strength: float = 1.0, tradoff: float = 1.0, tradoff_nag: float = 1.0, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, negative_promptA: Optional[Union[str, List[str]]] = None,
                 negative_promptB: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                 eta: float = 0.0, generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 latents: Optional[torch.FloatTensor] = None, prompt_embeds: Optional[torch.FloatTensor] = None,
                 negative_prompt_embeds: Optional[torch.FloatTensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback: Optional[Callable[[int, int, torch.FloatTensor], None]] = None,
                 callback_steps: int = 1, cross_attention_kwargs=None,
                 controlnet_conditioning_scale: Union[float, List[float]] = 0.5, guess_mode: bool = False,
                 control_guidance_start: Union[float, List[float]] = 0.0,
                 control_guidance_end: Union[float, List[float]] = 1.0):
        height, width = self._default_height_width(height, width, image)
        prompt, negative_prompt = promptA, negative_promptA
        # align format for control guidance (:1491-1502), then the reference's checks (:1505-1517)
        if not isinstance(control_guidance_start, list) and isinstance(control_guidance_end, list):
            control_guidance_start = len(control_guidance_end) * [control_guidance_start]
        elif not isinstance(control_guidance_end, list) and isinstance(control_guidance_start, list):
            control_guidance_end = len(control_guidance_start) * [control_guidance_end]
        elif not isinstance(control_guidance_start, list) and not isinstance(control_guidance_end, list):
            mult = len(self.controlnet.nets) if isinstance(self.controlnet, MultiControlNetModel) else 1
            control_guidance_start, control_guidance_end = mult * [control_guidance_start], mult * [control_guidance_end]
        self.check_inputs_controlnet(prompt, control_image, height, width, callback_steps, negative_prompt,
                                     prompt_embeds, negative_prompt_embeds, controlnet_conditioning_scale,
                                     control_guidance_start, control_guidance_end)
        # valid for the reference, outside the hot path here
        if cross_attention_kwargs:
            raise NotImplementedError("cross_attention_kwargs (LoRA scale) is outside the hot path")
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None and isinstance(prompt, list):
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        device = self._execution_device
        do_cfg = guidance_scale > 1.0
        nets = self.controlnet.nets if isinstance(self.controlnet, MultiControlNetModel) else [self.controlnet]
        multi = isinstance(self.controlnet, MultiControlNetModel)
        if multi and isinstance(controlnet_conditioning_scale, float):  # (:1533-1534)
            controlnet_conditioning_scale = [controlnet_conditioning_scale] * len(nets)
        guess_mode = guess_mode or nets[0].config.global_pool_conditions  # (:1536-1541)
        prompt_embeds = self._encode_prompt(promptA, promptB, tradoff, device, num_images_per_prompt, do_cfg,
                                            negative_promptA, negative_promptB, tradoff_nag,
                                            prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds)
        total = batch_size * num_images_per_prompt
        control = [self.prepare_control_image(ci, width, height, total, num_images_per_prompt, device, torch.float32,
                                              do_cfg, guess_mode) for ci in (control_image if multi else [control_image])]
        if uint8_device_inputs(self.vae, image, mask):  # see StableDiffusionInpaintPipeline.__call__
            if image.shape[-2:] != mask.shape[-2:] or image.shape[0] != mask.shape[0] or mask.shape[1] != 1:
                raise ValueError("uint8 image [B,3,H,W] and mask [B,1,H,W] must agree in batch and size")
            masked_image = init_image = image.contiguous()
        else:
            mask, masked_image, init_image = prepare_mask_and_masked_image(image, mask, height, width,
                                                                           return_image=True)
        self.scheduler.set_timesteps(num_inference_steps, device="cpu")
        timesteps, num_inference_steps = self.get_timesteps(num_inference_steps, strength, device)
        if self.unet.config.in_channels != 9:
            raise ValueError("the ControlNet inpainting path expects the 9-channel inpainting UNet")
        if num_inference_steps < 1:
            raise ValueError(f"After adjusting the num_inference_steps by strength parameter: {strength}, the number "
                             f"of pipeline steps is {num_inference_steps} which is < 1 and not appropriate for this "
                             "pipeline.")
        # strength < 1 (ref:pipeline_PowerPaint_ControlNet.py:1603-1625): noised image latents, shorter schedule
        latent_timestep = timesteps[:1].repeat(total)
        is_strength_max = strength == 1.0
        latents, noise = self.prepare_latents(total, self.vae.config.latent_channels, height, width, torch.float32,
                                              device, generator, latents, image=init_image,
                                              timestep=latent_timestep, is_strength_max=is_strength_max,
                                              return_noise=True, return_image_latents=False)
        mask, masked_image_latents = self.prepare_mask_latents(mask, masked_image, total, height, width, torch.float32,
                                                               device, generator, do_cfg)
        extra_step_kwargs = self.prepare_extra_step_kwargs(generator, eta)
        keeps = [[1.0 - float(i / len(timesteps) < s or (i + 1) / len(timesteps) > e) for i in range(len(timesteps))]
                 for s, e in zip(control_guidance_start, control_guidance_end)]
        # `controlnet_keep` (ref:pipeline_PowerPaint_ControlNet.py:1652-1658): the per-step scale
        # conditioning_scale * keep[i] sits in the device coefficient table the recorded program indexes
        coef = self.scheduler.step_coefficients(timesteps, eta=extra_step_kwargs.get("eta", 0.0))
        ucoef = scoef = pcoef = None
        finish = None
        kind = getattr(self.scheduler, "kind", "ddim")
        if kind == "unipc":
            ucoef = self.scheduler.unipc_coefficients(first=len(self.scheduler.timesteps) - len(timesteps))
        if kind == "plms":
            pcoef = self.scheduler.plms_coefficients(first=len(self.scheduler.timesteps) - len(timesteps))
        noise_kw = {}
        if eta > 0 and "eta" in extra_step_kwargs:  # schedulers without `eta` ignore it (signature sniffing, :536-551)
            noise_kw = step_noise(generator, latents.shape, device, len(timesteps))
        if kind == "solver":
            scoef, noise_kw, finish = solver_loop_inputs(self.scheduler, timesteps, latents.shape, generator, device)
        cb = None
        if callback is not None:
            n_ts = len(timesteps)
            warmup = n_ts - num_inference_steps * self.scheduler.order  # PNDM: 1, its first step is not reported

            def cb(i, t, lat):
                if callback_fires(i, n_ts, warmup, self.scheduler.order) and i % callback_steps == 0:
                    callback(i, t, lat)
                return None
        if multi:
            # `MultiControlNetModel` zips nets with scales: a net without a scale adds nothing (a zero scale)
            scales = [float(v) for v in controlnet_conditioning_scale][:len(nets)]
            side = dict(control_image=control, side_scale=scales + [0.0] * (len(nets) - len(scales)), side_keep=keeps)
        else:
            scale = controlnet_conditioning_scale
            side = dict(control_image=control[0], side_scale=float(scale[0] if isinstance(scale, list) else scale),
                        side_keep=keeps[0])
        # `guess_mode` / `scoef` are passed only when set: a denoiser whose `run` predates them keeps serving the
        # plain single-ControlNet call unchanged
        if guess_mode:
            side["guess_mode"] = True
        if scoef is not None:
            side["scoef"] = scoef
        if pcoef is not None:
            side["pcoef"] = pcoef
        if "randn_draws" in noise_kw:
            side["randn_draws"] = noise_kw["randn_draws"]
        run = dict(latents=latents, prompt_embeds=prompt_embeds, side_prompt_embeds=prompt_embeds, timesteps=timesteps,
                   coef=coef, guidance_scale=guidance_scale, extra=torch.cat([mask, masked_image_latents], dim=1),
                   noise_fn=noise_kw.get("noise_fn"), ucoef=ucoef, callback=cb, **side)
        return LoopInputs(run, finish, output_type, return_dict)
