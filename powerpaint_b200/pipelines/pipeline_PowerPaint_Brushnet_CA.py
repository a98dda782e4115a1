"""`StableDiffusionPowerPaintBrushNetPipeline` (PowerPaint v2) — drop-in for the reference class
(powerpaint/pipelines/pipeline_PowerPaint_Brushnet_CA.py:131; `__call__` :1024-1497). The loop
(:1384-1449: BrushNet forward with the task-prompt embeddings, UNet forward with the promptU
embeddings and the 12+1+15 add tensors, CFG, scheduler.step) runs as ONE recorded CUDA program per
step (`FusedDenoiser(mode="brushnet")`): the BrushNet zero-convs write straight into the buffers the
UNet epilogues add from, so the 28 add tensors never make a separate pass through HBM.

Kept from the reference API: constructor names (:179-192, incl. `text_encoder_brushnet`, `brushnet`),
`__call__` signature (:1026-1062), `brushnet_conditioning_scale` must be a float (TypeError, :827-828),
mask convention `original_mask = (sum_c(preprocessed mask) < 0)` (:1312), conditioning latents
`cat[vae.encode(image).latent_dist.sample() * scaling_factor, nearest(mask)]` (:1338-1345, sampled
with the GLOBAL RNG and for both CFG halves, exactly like upstream), `brushnet_keep` (:1369-1376),
`callback_on_step_end` semantics (:1451-1459).
"""
from __future__ import annotations

from typing import Any, Callable, Dict, List, Optional, Union

import torch

from ..denoise import FusedDenoiser
from ..models.unet_2d_condition import BrushNetModel, UNet2DConditionModel
from .common import (LoopInputs, callback_fires, check_control_guidance, check_image, check_prompt_arguments,
                     encode_text, preprocess_image, randn_tensor, step_noise,
                     solver_loop_inputs)
from .pipeline_PowerPaint import StableDiffusionInpaintPipeline


class StableDiffusionPowerPaintBrushNetPipeline(StableDiffusionInpaintPipeline):
    _callback_tensor_inputs = ["latents", "prompt_embeds", "negative_prompt_embeds"]

    def __init__(self, vae, text_encoder, text_encoder_brushnet, tokenizer, unet, brushnet, scheduler,
                 safety_checker=None, feature_extractor=None, image_encoder=None,
                 requires_safety_checker: bool = False):
        super().__init__(vae, text_encoder, tokenizer, unet, scheduler, safety_checker, feature_extractor,
                         requires_safety_checker)
        if image_encoder is not None:
            raise NotImplementedError("IP-adapter image_encoder is outside the hot path (unused by app.py)")
        self.text_encoder_brushnet = text_encoder_brushnet
        self.brushnet = brushnet
        self._denoiser_side = None

    def denoiser(self) -> FusedDenoiser:
        if not isinstance(self.unet, UNet2DConditionModel) or not isinstance(self.brushnet, BrushNetModel):
            assert False, "unet / brushnet must be powerpaint_b200 UNet2DConditionModel / BrushNetModel"
        if self._denoiser is None or self._denoiser_unet is not self.unet or self._denoiser_side is not self.brushnet:
            self._denoiser = FusedDenoiser(self.unet, self.brushnet, mode="brushnet")
            self._denoiser_unet, self._denoiser_side = self.unet, self.brushnet
        return self._denoiser

    def check_image(self, image, mask, prompt, prompt_embeds):
        """ref:pipeline_PowerPaint_Brushnet_CA.py:868-922"""
        check_image(image, prompt, prompt_embeds, mask=mask, with_mask=True)

    @property
    def clip_skip(self):
        # what `__call__` was given (:1006-1007, :1227). Like the reference's `__call__`, ours never hands it to
        # `encode_prompt` (:1268-1277), so it only shows here.
        return getattr(self, "_clip_skip", None)

    @property
    def cross_attention_kwargs(self):
        return None  # LoRA scaling is outside the hot path

    @property
    def num_timesteps(self):
        return getattr(self, "_num_timesteps", None)

    @property
    def guidance_scale(self):
        return self._guidance_scale

    @property
    def do_classifier_free_guidance(self):
        return self._guidance_scale > 1

    # ------------------------------------------------------------------ prompts
    def _encode_prompt(self, promptA, promptB, t, device, num_images_per_prompt, do_classifier_free_guidance,
                       negative_promptA=None, negative_promptB=None, t_nag=None, prompt_embeds=None,
                       negative_prompt_embeds=None, lora_scale=None):
        """task prompts go through `text_encoder_brushnet` (:228-439)"""
        te = self.text_encoder
        self.text_encoder = self.text_encoder_brushnet
        try:
            return super()._encode_prompt(promptA, promptB, t, device, num_images_per_prompt,
                                          do_classifier_free_guidance, negative_promptA, negative_promptB, t_nag,
                                          prompt_embeds, negative_prompt_embeds, lora_scale)
        finally:
            self.text_encoder = te

    def encode_prompt(self, prompt, device, num_images_per_prompt, do_classifier_free_guidance, negative_prompt=None,
                      prompt_embeds=None, negative_prompt_embeds=None, lora_scale=None, clip_skip=None):
        """plain promptU through `text_encoder` (:442-629); returns [neg; pos] like the reference's caller expects"""
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
            prompt = [prompt]
        elif prompt is not None:
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        if prompt_embeds is None and clip_skip is not None:
            # (:537-552) hidden state `clip_skip` layers before the last one, then the final LayerNorm; needs a text
            # encoder that returns its hidden states (transformers' CLIPTextModel; the kernel-backed one refuses)
            ids = self.tokenizer(prompt, padding="max_length", max_length=self.tokenizer.model_max_length,
                                 truncation=True, return_tensors="pt").input_ids
            hidden = self.text_encoder(ids.to(device), output_hidden_states=True)[-1][-(clip_skip + 1)]
            prompt_embeds = self.text_encoder.text_model.final_layer_norm(hidden)
        elif prompt_embeds is None:
            prompt_embeds = encode_text(self.tokenizer, self.text_encoder, prompt, device)
        prompt_embeds = prompt_embeds.to(device=device, dtype=torch.float32)
        bs, seq, _ = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, seq, -1)
        if do_classifier_free_guidance and negative_prompt_embeds is None:
            if negative_prompt is None:
                uncond = [""] * batch_size
            elif isinstance(negative_prompt, str):
                uncond = [negative_prompt]
            elif batch_size != len(negative_prompt):
                raise ValueError(f"`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but "
                                 f"`prompt` has batch size {batch_size}.")
            else:
                uncond = negative_prompt
            negative_prompt_embeds = encode_text(self.tokenizer, self.text_encoder, uncond, device, max_length=seq)
        if do_classifier_free_guidance:
            negative_prompt_embeds = negative_prompt_embeds.to(device=device, dtype=torch.float32)
            negative_prompt_embeds = negative_prompt_embeds.repeat(1, num_images_per_prompt, 1).view(
                batch_size * num_images_per_prompt, negative_prompt_embeds.shape[1], -1)
            return torch.cat([negative_prompt_embeds, prompt_embeds])
        return prompt_embeds

    # ------------------------------------------------------------------ checks (:753-922)
    _callback_tensor_inputs = ["latents", "prompt_embeds", "negative_prompt_embeds"]

    def check_inputs_brushnet(self, prompt, image, mask, callback_steps, negative_prompt=None, prompt_embeds=None,
                              negative_prompt_embeds=None, ip_adapter_image=None, ip_adapter_image_embeds=None,
                              brushnet_conditioning_scale=1.0, control_guidance_start=0.0, control_guidance_end=1.0,
                              callback_on_step_end_tensor_inputs=None):
        """the reference's `check_inputs` (:753-866) in its order, same exception types and messages"""
        if callback_steps is not None and (not isinstance(callback_steps, int) or callback_steps <= 0):
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type"
                             f" {type(callback_steps)}.")
        if callback_on_step_end_tensor_inputs is not None and not all(
                k in self._callback_tensor_inputs for k in callback_on_step_end_tensor_inputs):
            bad = [k for k in callback_on_step_end_tensor_inputs if k not in self._callback_tensor_inputs]
            raise ValueError(f"`callback_on_step_end_tensor_inputs` has to be in {self._callback_tensor_inputs}, but "
                             f"found {bad}")
        check_prompt_arguments(prompt, negative_prompt, prompt_embeds, negative_prompt_embeds)
        if not isinstance(self.brushnet, BrushNetModel):
            assert False
        check_image(image, prompt, prompt_embeds, mask=mask, with_mask=True)
        if not isinstance(brushnet_conditioning_scale, float):
            raise TypeError("For single brushnet: `brushnet_conditioning_scale` must be type `float`.")
        if not isinstance(control_guidance_start, (tuple, list)):
            control_guidance_start = [control_guidance_start]
        if not isinstance(control_guidance_end, (tuple, list)):
            control_guidance_end = [control_guidance_end]
        check_control_guidance(control_guidance_start, control_guidance_end)
        if ip_adapter_image is not None and ip_adapter_image_embeds is not None:
            raise ValueError("Provide either `ip_adapter_image` or `ip_adapter_image_embeds`. Cannot leave both "
                             "`ip_adapter_image` and `ip_adapter_image_embeds` defined.")
        if ip_adapter_image_embeds is not None:
            if not isinstance(ip_adapter_image_embeds, list):
                raise ValueError("`ip_adapter_image_embeds` has to be of type `list` but is "
                                 f"{type(ip_adapter_image_embeds)}")
            elif ip_adapter_image_embeds[0].ndim not in [3, 4]:
                raise ValueError("`ip_adapter_image_embeds` has to be a list of 3D or 4D tensors but is "
                                 f"{ip_adapter_image_embeds[0].ndim}D")

    def prepare_image(self, image, width, height, batch_size, num_images_per_prompt, device, dtype,
                      do_classifier_free_guidance=False, guess_mode=False):
        image = preprocess_image(image, height=height, width=width).to(dtype=torch.float32)
        repeat_by = batch_size if image.shape[0] == 1 else num_images_per_prompt
        image = image.repeat_interleave(repeat_by, dim=0).to(device=device, dtype=dtype)
        if do_classifier_free_guidance and not guess_mode:
            image = torch.cat([image] * 2)
        return image

    # ------------------------------------------------------------------ __call__ (:1024-1497)
    @torch.no_grad()
    def prepare_loop(self, promptA: Union[str, List[str]] = None, promptB: Union[str, List[str]] = None,
                 promptU: Union[str, List[str]] = None, tradoff: float = 1.0, tradoff_nag: float = 1.0, image=None,
                 mask=None, height: Optional[int] = None, width: Optional[int] = None, num_inference_steps: int = 50,
                 timesteps: List[int] = None, guidance_scale: float = 7.5,
                 negative_promptA: Optional[Union[str, List[str]]] = None,
                 negative_promptB: Optional[Union[str, List[str]]] = None,
                 negative_promptU: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                 eta: float = 0.0, generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 latents: Optional[torch.FloatTensor] = None, prompt_embeds: Optional[torch.FloatTensor] = None,
                 negative_prompt_embeds: Optional[torch.FloatTensor] = None, ip_adapter_image=None,
                 ip_adapter_image_embeds=None, output_type: Optional[str] = "pil", return_dict: bool = True,
                 cross_attention_kwargs: Optional[Dict[str, Any]] = None,
                 brushnet_conditioning_scale: Union[float, List[float]] = 1.0, guess_mode: bool = False,
                 control_guidance_start: Union[float, List[float]] = 0.0,
                 control_guidance_end: Union[float, List[float]] = 1.0, clip_skip: Optional[int] = None,
                 callback_on_step_end: Optional[Callable[[Any, int, int, Dict], Dict]] = None,
                 callback_on_step_end_tensor_inputs: List[str] = ["latents"], **kwargs):
        callback = kwargs.pop("callback", None)
        callback_steps = kwargs.pop("callback_steps", None)
        # the oracle-facing extension: pre-computed promptU embeddings ([neg; pos]) for offline benches
        prompt_embedsU = kwargs.pop("prompt_embedsU", None)
        if kwargs:
            raise TypeError(f"unexpected keyword arguments: {sorted(kwargs)}")
        # align format for control guidance (:1197-1205), then the reference's checks in the reference's order (:1208-1224)
        if not isinstance(control_guidance_start, list) and isinstance(control_guidance_end, list):
            control_guidance_start = len(control_guidance_end) * [control_guidance_start]
        elif not isinstance(control_guidance_end, list) and isinstance(control_guidance_start, list):
            control_guidance_end = len(control_guidance_start) * [control_guidance_end]
        elif not isinstance(control_guidance_start, list) and not isinstance(control_guidance_end, list):
            control_guidance_start, control_guidance_end = [control_guidance_start], [control_guidance_end]
        prompt, negative_prompt = promptA, negative_promptA
        self.check_inputs_brushnet(prompt, image, mask, callback_steps, negative_prompt, prompt_embeds,
                                   negative_prompt_embeds, ip_adapter_image, ip_adapter_image_embeds,
                                   brushnet_conditioning_scale, control_guidance_start, control_guidance_end,
                                   callback_on_step_end_tensor_inputs)
        # valid for the reference, outside the hot path here
        if ip_adapter_image is not None or ip_adapter_image_embeds is not None:
            raise NotImplementedError("IP-adapter inputs are outside the hot path (unused by app.py)")
        if cross_attention_kwargs:
            raise NotImplementedError("cross_attention_kwargs (LoRA scale) is outside the hot path")
        self._guidance_scale = guidance_scale
        self._clip_skip = clip_skip
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None and isinstance(prompt, list):
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        device = self._execution_device
        do_cfg = self.do_classifier_free_guidance
        guess_mode = guess_mode or self.brushnet.config.global_pool_conditions  # (:1240-1245)
        prompt_embeds = self._encode_prompt(promptA, promptB, tradoff, device, num_images_per_prompt, do_cfg,
                                            negative_promptA, negative_promptB, tradoff_nag,
                                            prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds)
        if prompt_embedsU is None:
            prompt_embedsU = self.encode_prompt(promptU, device, num_images_per_prompt, do_cfg, negative_promptU)
        else:
            prompt_embedsU = prompt_embedsU.to(device=device, dtype=torch.float32)
        total = batch_size * num_images_per_prompt
        image_t = self.prepare_image(image, width, height, total, num_images_per_prompt, device, torch.float32, do_cfg,
                                     guess_mode)
        original_mask = self.prepare_image(mask, width, height, total, num_images_per_prompt, device, torch.float32,
                                           do_cfg, guess_mode)
        original_mask = (original_mask.sum(1)[:, None, :, :] < 0).to(image_t.dtype)
        height, width = image_t.shape[-2:]
        if timesteps is not None:
            # `retrieve_timesteps` (:114-122): DDIM and UniPC take no custom schedule — neither diffusers 0.27.0's nor
            # the ones here — so the reference raises this ValueError at this point of the call
            import inspect

            if "timesteps" not in inspect.signature(self.scheduler.set_timesteps).parameters:
                raise ValueError(f"The current scheduler class {self.scheduler.__class__}'s `set_timesteps` does not "
                                 "support custom timestep schedules. Please check whether you are using the correct "
                                 "scheduler.")
            raise NotImplementedError("custom `timesteps`: the fused step kernels read the coefficient tables of "
                                      "DDIMScheduler / UniPCMultistepScheduler (uniform spacing)")
        self.scheduler.set_timesteps(num_inference_steps, device="cpu")
        ts = self.scheduler.timesteps
        self._num_timesteps = len(ts)
        num_channels_latents = self.unet.config.in_channels
        shape = (total, num_channels_latents, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != total:  # (:957-962)
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {total}. Make sure the batch size matches the length of the "
                             "generators.")
        if latents is None:
            noise = randn_tensor(shape, generator=generator, device=device, dtype=torch.float32)
        else:
            noise = latents.to(device)
        latents = noise * self.scheduler.init_noise_sigma
        # global RNG, 2B batch under CFG (B in guess mode, whose images are not doubled) — exactly as the reference
        # (:1338-1341)
        if do_cfg and not guess_mode and hasattr(self.vae, "decode_postprocessed"):
            # both CFG halves hold the same images: encode them once and duplicate the moments; the noise is still
            # drawn for all 2B samples in one call, so the RNG stream equals the reference's
            dist = self.vae.encode(image_t[:total]).latent_dist
            mean, std = torch.cat([dist.mean] * 2), torch.cat([dist.std] * 2)
            conditioning_latents = (mean + std * torch.randn(mean.shape, device=mean.device, dtype=mean.dtype)).float()
            conditioning_latents = conditioning_latents * self.vae.config.scaling_factor
        else:
            conditioning_latents = (self.vae.encode(image_t.to(self.vae.dtype)).latent_dist.sample().float()
                                    * self.vae.config.scaling_factor)
        mask_l = torch.nn.functional.interpolate(original_mask, size=conditioning_latents.shape[-2:])
        conditioning_latents = torch.cat([conditioning_latents, mask_l], 1)
        extra_step_kwargs = self.prepare_extra_step_kwargs(generator, eta)
        keep = [1.0 - float(i / len(ts) < control_guidance_start[0] or (i + 1) / len(ts) > control_guidance_end[0])
                for i in range(len(ts))]
        # `brushnet_keep` (:1369-1376) x brushnet_conditioning_scale (:1403-1409) = the per-step scale row of the
        # device coefficient table the recorded program indexes
        coef = self.scheduler.step_coefficients(ts, eta=extra_step_kwargs.get("eta", 0.0))
        # the v2 app runs UniPC (app.py:197): its folded per-step scalars select the UniPC step kernel
        kind = getattr(self.scheduler, "kind", "ddim")
        ucoef = self.scheduler.unipc_coefficients() if kind == "unipc" else None
        pcoef = self.scheduler.plms_coefficients() if kind == "plms" else None
        scoef = finish = None
        noise_kw = {}
        if eta > 0 and "eta" in extra_step_kwargs:  # schedulers without `eta` ignore it (signature sniffing, :536-551)
            noise_kw = step_noise(generator, shape, device, len(ts))
        if kind == "solver":
            scoef, noise_kw, finish = solver_loop_inputs(self.scheduler, ts, shape, generator, device)
        cb = None
        if callback_on_step_end is not None or callback is not None:
            pipe = self
            order = self.scheduler.order
            warmup = len(ts) - num_inference_steps * order  # PNDM: 1, its first step is not reported to `callback`

            def cb(i, t, lat):
                new = None
                if callback_on_step_end is not None:
                    # the reference hands out the encoded tensors (:1451-1459): [neg; pos] split again
                    neg_e, pos_e = (prompt_embeds.chunk(2) if do_cfg else (None, prompt_embeds))
                    kw = {k: {"latents": lat, "prompt_embeds": pos_e, "negative_prompt_embeds": neg_e}[k]
                          for k in callback_on_step_end_tensor_inputs}
                    outs = callback_on_step_end(pipe, i, t, kw) or {}
                    for k in ("prompt_embeds", "negative_prompt_embeds"):
                        if k in outs and outs[k] is not kw.get(k):
                            raise NotImplementedError(
                                f"callback_on_step_end returned a replacement `{k}`: the cross-attention K/V of the "
                                "prompt are projected once per call, replacing them mid-loop is not supported")
                    new = outs.pop("latents", lat)
                    lat = new
                fires = callback_fires(i, len(ts), warmup, order) and i % (callback_steps or 1) == 0
                if callback is not None and fires:
                    callback(i, t, lat)
                return new
        # `scoef` / `guess_mode` are passed only when set: a denoiser whose `run` predates them keeps serving DDIM
        # and UniPC unchanged
        opt = {k: v for k, v in (("scoef", scoef), ("pcoef", pcoef), ("randn_draws", noise_kw.get("randn_draws")))
               if v is not None}
        if guess_mode:
            opt["guess_mode"] = True
        run = dict(latents=latents, prompt_embeds=prompt_embedsU, side_prompt_embeds=prompt_embeds, timesteps=ts,
                   coef=coef, guidance_scale=guidance_scale, extra=conditioning_latents,
                   side_scale=float(brushnet_conditioning_scale), side_keep=keep, ucoef=ucoef, noise_fn=noise_kw.get("noise_fn"),
                   callback=cb, **opt)
        return LoopInputs(run, finish, output_type, return_dict)
