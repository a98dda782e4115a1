"""`StableDiffusionInpaintPipeline` of PowerPaint v1 — drop-in for the reference class
(powerpaint/pipelines/pipeline_PowerPaint.py:156; `__call__` :722-1071) with the denoising loop
(:988-1035) replaced by the fused CUDA program of `powerpaint_b200.denoise.FusedDenoiser`.

Kept verbatim from the reference API (SURVEY.md §8b): constructor argument names, plain settable
attributes `.tokenizer/.text_encoder/.unet/.vae/.scheduler` (the app re-assigns them,
app.py:94,111-112,130), the `__call__` signature including the `tradoff` / `tradoff_nag` spelling,
the task-prompt blend `E = t*E_A + (1-t)*E_B` (:423,:499) with negative embeddings first (:516),
`check_inputs` exceptions (:553-602), callback cadence (:1038-1041), return types (:1068-1071).
Everything outside the loop (PIL pre-processing, CLIP, VAE) is the reference's host dataflow
on torch; the VAE / text encoder / tokenizer are injected dependencies exactly as upstream.
"""
from __future__ import annotations

import inspect
from typing import Callable, List, Optional, Union

import torch

from ..denoise import FusedDenoiser
from ..models import AutoencoderKL, BrushNetModel, ControlNetModel, UNet2DConditionModel
from .common import (LoopInputs, callback_fires, decode_latents, encode_text, prepare_mask_and_masked_image, run_loop,
                     randn_tensor, solver_loop_inputs, step_noise, uint8_device_inputs, vae_encode)

# the components stored as diffusers model directories, by their name in model_index.json
_MODEL_COMPONENTS = {"unet": UNet2DConditionModel, "brushnet": BrushNetModel, "controlnet": ControlNetModel,
                     "vae": AutoencoderKL}


class StableDiffusionInpaintPipeline:
    _optional_components = ["safety_checker", "feature_extractor"]

    def __init__(self, vae, text_encoder, tokenizer, unet, scheduler, safety_checker=None, feature_extractor=None,
                 requires_safety_checker: bool = False):
        if safety_checker is not None:
            raise NotImplementedError("safety_checker must be None (the reference app passes None, app.py:131-132)")
        self.vae = vae
        self.text_encoder = text_encoder
        self.tokenizer = tokenizer
        self.unet = unet
        self.scheduler = scheduler
        self.safety_checker = None
        self.feature_extractor = feature_extractor
        # the reference force-sets steps_offset=1 / clip_sample=False on the scheduler config (:205-231)
        cfg = getattr(scheduler, "config", None)
        if cfg is not None:
            if getattr(cfg, "steps_offset", 1) != 1:
                cfg.steps_offset = 1
            if getattr(cfg, "clip_sample", False):
                cfg.clip_sample = False
        boc = getattr(getattr(vae, "config", None), "block_out_channels", (0, 0, 0, 0))
        self.vae_scale_factor = 2 ** (len(boc) - 1)
        self._denoiser: Optional[FusedDenoiser] = None
        self._denoiser_unet = None
        self._progress_bar_config = {}

    # ------------------------------------------------------------------ checkpoint directories (ref:app.py:91-93,157-164)
    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, torch_dtype=None, revision: Optional[str] = None,
                        variant: Optional[str] = None, local_files_only: bool = False,
                        cache_dir: Optional[str] = None, **kwargs):
        """`DiffusionPipeline.from_pretrained` for a local directory or a cached hub snapshot in the diffusers layout
        (`model_index.json` + one subfolder per component). Constructor arguments passed as keywords replace the
        stored component, like upstream (`brushnet=`, `text_encoder_brushnet=`, `safety_checker=None`, ...). The nets and
        the VAE load as this package's classes, text encoder and tokenizer through transformers (the injected
        dependencies they are upstream), the scheduler as DDIM (or UniPC) built from `scheduler_config.json`. A stored
        safety checker is not loaded. Everything is on the CPU afterwards: `pipe = pipe.to("cuda")` as in the app."""
        import inspect
        import os

        from ..loading import load_json, resolve_checkpoint_dir

        root = resolve_checkpoint_dir(pretrained_model_name_or_path, None, revision, local_files_only, cache_dir)
        index = load_json(root, "model_index.json")
        params = [p for p in inspect.signature(cls.__init__).parameters if p != "self"]
        passed = {k: kwargs.pop(k) for k in list(kwargs) if k in params}
        for ignored in ("low_cpu_mem_usage", "use_safetensors", "device_map", "force_download", "resume_download",
                        "proxies", "token", "use_auth_token", "custom_pipeline"):
            kwargs.pop(ignored, None)
        if kwargs:
            raise TypeError(f"unexpected keyword arguments: {sorted(kwargs)}")
        components = {}
        for name in params:
            if name in passed:
                components[name] = passed[name]
            elif name in ("safety_checker", "feature_extractor", "image_encoder"):
                if name == "safety_checker" and (index.get(name) or [None])[0] is not None:
                    import warnings

                    warnings.warn("powerpaint_b200: the stored safety checker is not loaded (outside the hot path; pass "
                                  "`safety_checker=None` like the app's v2 branch does to silence this)", stacklevel=2)
                components[name] = None
            elif name == "requires_safety_checker":
                components[name] = False
            else:
                entry = index.get(name)
                if not entry or entry[0] is None:
                    raise ValueError(f"Pipeline {cls} expected {name}, but it is neither stored in "
                                     f"{os.path.join(root, 'model_index.json')} nor passed as a keyword argument.")
                components[name] = cls._load_component(name, os.path.join(root, name), entry, torch_dtype, variant)
        return cls(**components)

    @staticmethod
    def _load_component(name: str, directory: str, entry, torch_dtype, variant):
        """one subfolder of a pipeline directory; `entry` = [library, class name] of model_index.json"""
        from ..loading import load_json
        from .. import schedulers
        from ..schedulers import DDIMScheduler

        if name in _MODEL_COMPONENTS:
            return _MODEL_COMPONENTS[name].from_pretrained(directory, torch_dtype=torch_dtype, variant=variant)
        if name in ("text_encoder", "text_encoder_brushnet"):
            import transformers

            te = transformers.CLIPTextModel.from_pretrained(directory)
            return te.to(torch_dtype) if torch_dtype is not None else te
        if name == "tokenizer":
            import transformers

            return transformers.CLIPTokenizer.from_pretrained(directory)
        if name == "scheduler":
            cfg = load_json(directory, "scheduler_config.json")
            stored = cfg.get("_class_name")
            if stored in ("UniPCMultistepScheduler", "DPMSolverMultistepScheduler", "EulerDiscreteScheduler",
                          "EulerAncestralDiscreteScheduler"):
                return getattr(schedulers, stored).from_config(cfg)
            if stored not in (None, "DDIMScheduler"):
                import warnings

                hint = (" (PLMS runs on the fused loop when chosen explicitly: pipe.scheduler = "
                        "PNDMScheduler.from_pretrained(checkpoint, subfolder='scheduler'))" if stored == "PNDMScheduler"
                        else "")
                warnings.warn(f"powerpaint_b200: the stored scheduler {stored} is replaced by DDIMScheduler built from "
                              "the same noise schedule (the fused step kernels implement DDIM, UniPC, DPM-Solver++, "
                              f"Euler and PNDM){hint}", stacklevel=3)
            return DDIMScheduler.from_config(cfg)
        raise ValueError(f"unknown pipeline component {name!r} ({entry})")

    # ------------------------------------------------------------------ small diffusers surface
    @property
    def _execution_device(self) -> torch.device:
        return self.unet.device

    @property
    def device(self) -> torch.device:
        return self.unet.device

    # every module the reference pipelines register (`register_modules`, ref:pipeline_PowerPaint.py:247-255,
    # ref:pipeline_PowerPaint_Brushnet_CA.py:212-222, ref:pipeline_PowerPaint_ControlNet.py:308-317)
    _components = ("vae", "text_encoder", "text_encoder_brushnet", "unet", "brushnet", "controlnet", "safety_checker")

    def to(self, device=None, dtype=None):
        """`DiffusionPipeline.to`: every registered module moves (the app does `pipe = pipe.to("cuda")`,
        ref:app.py:113,135,200). A dtype only selects the dtype of the tensors the hot-path nets return."""
        if isinstance(device, torch.dtype):
            device, dtype = None, device
        for name in self._components:
            m = getattr(self, name, None)
            if m is None or not hasattr(m, "to"):
                continue
            if device is not None:
                m.to(device)
            if dtype is not None and name in ("unet", "brushnet", "controlnet"):
                m.to(dtype=dtype)
        return self

    def set_progress_bar_config(self, **kwargs):
        self._progress_bar_config = kwargs

    def enable_model_cpu_offload(self, gpu_id=0):
        """The v2 app calls this right before `pipe.to("cuda")` (ref:app.py:199-200). Nothing is offloaded here: the
        recorded step programs hold device pointers into the packed weights, which stay resident (an H100 has 80 GB;
        UNet + BrushNet are 3.5 GB in bf16). Kept callable so the app runs unchanged; it only says so."""
        import warnings

        warnings.warn("powerpaint_b200: enable_model_cpu_offload() keeps all models resident on the GPU (the hot path "
                      "has no CPU side to offload to)", stacklevel=2)

    def denoiser(self) -> FusedDenoiser:
        if not isinstance(self.unet, UNet2DConditionModel):
            raise TypeError("`unet` must be a powerpaint_b200 UNet2DConditionModel: the denoising loop runs as a "
                            "recorded CUDA program and has no eager fallback")
        if self._denoiser is None or self._denoiser_unet is not self.unet:
            self._denoiser = FusedDenoiser(self.unet, mode="v1")
            self._denoiser_unet = self.unet
        return self._denoiser

    # ------------------------------------------------------------------ prompt encoding (:317-518)
    def _encode_prompt(self, promptA, promptB, t, device, num_images_per_prompt, do_classifier_free_guidance,
                       negative_promptA=None, negative_promptB=None, t_nag=None, prompt_embeds=None,
                       negative_prompt_embeds=None, lora_scale=None):
        prompt, negative_prompt = promptA, negative_promptA
        if promptA is not None and isinstance(promptA, str):
            batch_size = 1
        elif promptA is not None and isinstance(promptA, list):
            batch_size = len(promptA)
        else:
            batch_size = prompt_embeds.shape[0]
        if prompt_embeds is None:
            eA = encode_text(self.tokenizer, self.text_encoder, promptA, device)
            eB = encode_text(self.tokenizer, self.text_encoder, promptB, device)
            prompt_embeds = eA * t + (1 - t) * eB
        prompt_embeds = prompt_embeds.to(device=device, dtype=torch.float32)
        bs, seq, _ = prompt_embeds.shape
        prompt_embeds = prompt_embeds.repeat(1, num_images_per_prompt, 1).view(bs * num_images_per_prompt, seq, -1)
        if do_classifier_free_guidance and negative_prompt_embeds is None:
            if negative_prompt is None:
                uA, uB = [""] * batch_size, [""] * batch_size
            elif prompt is not None and type(prompt) is not type(negative_prompt):
                raise TypeError(f"`negative_prompt` should be the same type to `prompt`, but got "
                                f"{type(negative_prompt)} != {type(prompt)}.")
            elif isinstance(negative_prompt, str):
                uA, uB = [negative_promptA], [negative_promptB]
            elif batch_size != len(negative_prompt):
                raise ValueError(f"`negative_prompt`: {negative_prompt} has batch size {len(negative_prompt)}, but "
                                 f"`prompt`: {prompt} has batch size {batch_size}. Please make sure that passed "
                                 "`negative_prompt` matches the batch size of `prompt`.")
            else:
                uA, uB = negative_promptA, negative_promptB
            nA = encode_text(self.tokenizer, self.text_encoder, uA, device, max_length=seq)
            nB = encode_text(self.tokenizer, self.text_encoder, uB, device, max_length=seq)
            negative_prompt_embeds = nA * t_nag + (1 - t_nag) * nB
        if do_classifier_free_guidance:
            seq = negative_prompt_embeds.shape[1]
            negative_prompt_embeds = negative_prompt_embeds.to(dtype=torch.float32, device=device)
            negative_prompt_embeds = negative_prompt_embeds.repeat(1, num_images_per_prompt, 1)
            negative_prompt_embeds = negative_prompt_embeds.view(batch_size * num_images_per_prompt, seq, -1)
            prompt_embeds = torch.cat([negative_prompt_embeds, prompt_embeds])
        return prompt_embeds

    # ------------------------------------------------------------------ checks / helpers
    def check_inputs(self, prompt, height, width, strength, callback_steps, negative_prompt=None, prompt_embeds=None,
                     negative_prompt_embeds=None):
        if strength < 0 or strength > 1:
            raise ValueError(f"The value of strength should in [0.0, 1.0] but is {strength}")
        if height % 8 != 0 or width % 8 != 0:
            raise ValueError(f"`height` and `width` have to be divisible by 8 but are {height} and {width}.")
        if callback_steps is None or not isinstance(callback_steps, int) or callback_steps <= 0:
            raise ValueError(f"`callback_steps` has to be a positive integer but is {callback_steps} of type"
                             f" {type(callback_steps)}.")
        if prompt is not None and prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `prompt`: {prompt} and `prompt_embeds`: {prompt_embeds}. Please "
                             "make sure to only forward one of the two.")
        elif prompt is None and prompt_embeds is None:
            raise ValueError("Provide either `prompt` or `prompt_embeds`. Cannot leave both `prompt` and "
                             "`prompt_embeds` undefined.")
        elif prompt is not None and not isinstance(prompt, (str, list)):
            raise ValueError(f"`prompt` has to be of type `str` or `list` but is {type(prompt)}")
        if negative_prompt is not None and negative_prompt_embeds is not None:
            raise ValueError(f"Cannot forward both `negative_prompt`: {negative_prompt} and `negative_prompt_embeds`:"
                             f" {negative_prompt_embeds}. Please make sure to only forward one of the two.")
        if prompt_embeds is not None and negative_prompt_embeds is not None:
            if prompt_embeds.shape != negative_prompt_embeds.shape:
                raise ValueError("`prompt_embeds` and `negative_prompt_embeds` must have the same shape when passed "
                                 f"directly, but got: `prompt_embeds` {prompt_embeds.shape} != "
                                 f"`negative_prompt_embeds` {negative_prompt_embeds.shape}.")

    def prepare_extra_step_kwargs(self, generator, eta):
        kw = {}
        params = set(inspect.signature(self.scheduler.step).parameters.keys())
        if "eta" in params:
            kw["eta"] = eta
        if "generator" in params:
            kw["generator"] = generator
        return kw

    def get_timesteps(self, num_inference_steps, strength, device):
        init_timestep = min(int(num_inference_steps * strength), num_inference_steps)
        t_start = max(num_inference_steps - init_timestep, 0)
        timesteps = self.scheduler.timesteps[t_start * self.scheduler.order:]
        return timesteps, num_inference_steps - t_start

    def prepare_latents(self, batch_size, num_channels_latents, height, width, dtype, device, generator, latents=None,
                        image=None, timestep=None, is_strength_max=True, return_noise=False,
                        return_image_latents=False):
        shape = (batch_size, num_channels_latents, height // self.vae_scale_factor, width // self.vae_scale_factor)
        if isinstance(generator, list) and len(generator) != batch_size:
            raise ValueError(f"You have passed a list of generators of length {len(generator)}, but requested an "
                             f"effective batch size of {batch_size}. Make sure the batch size matches the length of "
                             "the generators.")
        if (image is None or timestep is None) and not is_strength_max:
            raise ValueError("Since strength < 1. initial latents are to be initialised as a combination of Image + "
                             "Noise.However, either the image or the noise timestep has not been provided.")
        image_latents = None
        if return_image_latents or (latents is None and not is_strength_max):
            if image.dtype == torch.uint8:  # device-resident uint8 request: normalised inside the encoder's first pass
                image_latents = self.vae.config.scaling_factor * self.vae.encode_uint8(image).sample(generator).float()
            else:
                image_latents = vae_encode(self.vae, image.to(device=device, dtype=dtype), generator)
        if latents is None:
            noise = randn_tensor(shape, generator=generator, device=device, dtype=dtype)
            latents = noise if is_strength_max else self.scheduler.add_noise(image_latents, noise, timestep)
            latents = latents * self.scheduler.init_noise_sigma if is_strength_max else latents
        else:
            noise = latents.to(device)
            latents = noise * self.scheduler.init_noise_sigma
        outputs = (latents,)
        if return_noise:
            outputs += (noise,)
        if return_image_latents:
            outputs += (image_latents,)
        return outputs

    def _encode_vae_image(self, image: torch.Tensor, generator=None) -> torch.Tensor:
        """ref:pipeline_PowerPaint.py:657-669: posterior sample (per-sample generators honoured) x scaling_factor"""
        return vae_encode(self.vae, image, generator)

    def run_safety_checker(self, image, device, dtype):
        """ref:pipeline_PowerPaint.py:521-533 with `safety_checker=None` (what the app passes): nothing is flagged"""
        return image, None

    def decode_latents(self, latents: torch.Tensor):
        """the deprecated helper of the ControlNet / BrushNet pipelines (ref:pipeline_PowerPaint_ControlNet.py:614-624):
        float32 NHWC numpy in [0, 1]"""
        return decode_latents(self.vae, latents, "np")

    def enable_vae_slicing(self):
        """accepted: decoding a batch slice by slice is numerically the decode of the batch (ref:…ControlNet.py:326-332)"""

    def disable_vae_slicing(self):
        pass

    def enable_vae_tiling(self):
        """encode / decode through overlapping VAE tiles blended at the seams (ref:…ControlNet.py:341-356): images
        above 1024 x 1024 pixels then fit, at the price of a result that differs from the untiled one at the seams"""
        self.vae.enable_tiling()

    def disable_vae_tiling(self):
        self.vae.disable_tiling()

    def prepare_mask_latents(self, mask, masked_image, batch_size, height, width, dtype, device, generator,
                             do_classifier_free_guidance):
        """nearest-resize the mask to latent resolution, VAE-encode the masked image (:671-710).
        Unlike the reference this returns ONE copy per image even under CFG: the duplication
        (`torch.cat([mask] * 2)`, :703-706) happens inside the fused step kernel."""
        if masked_image.dtype == torch.uint8:
            # uint8 fast path: `masked_image` is the raw image, the hole is zeroed inside the pre-processing kernel
            full_mask = mask.contiguous()
            masked_image_latents = (self.vae.config.scaling_factor *
                                    self.vae.encode_uint8(masked_image, full_mask).sample(generator).float())
            mask = (mask >= 128).to(dtype) if mask.dtype == torch.uint8 else (mask >= 0.5).to(dtype)
        else:
            masked_image_latents = None
        mask = torch.nn.functional.interpolate(mask, size=(height // self.vae_scale_factor,
                                                           width // self.vae_scale_factor))
        mask = mask.to(device=device, dtype=dtype)
        if masked_image_latents is None:
            masked_image = masked_image.to(device=device, dtype=dtype)
            masked_image_latents = vae_encode(self.vae, masked_image, generator)
        for name, t in (("masks", mask), ("images", masked_image_latents)):
            if t.shape[0] < batch_size and batch_size % t.shape[0] != 0:
                raise ValueError(f"The passed {name} and the required batch size don't match: {t.shape[0]} {name} "
                                 f"were passed for a total batch size of {batch_size}.")
        if mask.shape[0] < batch_size:
            mask = mask.repeat(batch_size // mask.shape[0], 1, 1, 1)
        if masked_image_latents.shape[0] < batch_size:
            masked_image_latents = masked_image_latents.repeat(batch_size // masked_image_latents.shape[0], 1, 1, 1)
        return mask, masked_image_latents.to(device=device, dtype=dtype)

    # ------------------------------------------------------------------ __call__ (:722-1071)
    @torch.no_grad()
    def __call__(self, *args, **kwargs):
        """`prepare_loop`'s arguments: prepares the call, runs the fused denoising loop and decodes"""
        return run_loop(self, self.prepare_loop(*args, **kwargs))

    @torch.no_grad()
    def prepare_loop(self, promptA: Union[str, List[str]] = None, promptB: Union[str, List[str]] = None, image=None,
                 mask=None, height: Optional[int] = None, width: Optional[int] = None, strength: float = 1.0,
                 tradoff: float = 1.0, tradoff_nag: float = 1.0, num_inference_steps: int = 50,
                 guidance_scale: float = 7.5, negative_promptA: Optional[Union[str, List[str]]] = None,
                 negative_promptB: Optional[Union[str, List[str]]] = None, num_images_per_prompt: Optional[int] = 1,
                 eta: float = 0.0, generator: Optional[Union[torch.Generator, List[torch.Generator]]] = None,
                 latents: Optional[torch.FloatTensor] = None, prompt_embeds: Optional[torch.FloatTensor] = None,
                 negative_prompt_embeds: Optional[torch.FloatTensor] = None, output_type: Optional[str] = "pil",
                 return_dict: bool = True, callback: Optional[Callable[[int, int, torch.FloatTensor], None]] = None,
                 callback_steps: int = 1, cross_attention_kwargs=None, task_class=None):
        height = height or self.unet.config.sample_size * self.vae_scale_factor
        width = width or self.unet.config.sample_size * self.vae_scale_factor
        prompt, negative_prompt = promptA, negative_promptA
        self.check_inputs(prompt, height, width, strength, callback_steps, negative_prompt, prompt_embeds,
                          negative_prompt_embeds)
        if cross_attention_kwargs:
            raise NotImplementedError("cross_attention_kwargs (LoRA scale) is outside the PowerPaint hot path")
        if task_class is not None:
            raise NotImplementedError("task_class needs the class-conditioned UNet, not part of the released models")
        if prompt is not None and isinstance(prompt, str):
            batch_size = 1
        elif prompt is not None and isinstance(prompt, list):
            batch_size = len(prompt)
        else:
            batch_size = prompt_embeds.shape[0]
        device = self._execution_device
        do_cfg = guidance_scale > 1.0
        prompt_embeds = self._encode_prompt(promptA, promptB, tradoff, device, num_images_per_prompt, do_cfg,
                                            negative_promptA, negative_promptB, tradoff_nag,
                                            prompt_embeds=prompt_embeds, negative_prompt_embeds=negative_prompt_embeds)
        self.scheduler.set_timesteps(num_inference_steps, device="cpu")
        timesteps, num_inference_steps = self.get_timesteps(num_inference_steps, strength, device)
        if num_inference_steps < 1:
            raise ValueError(f"After adjusting the num_inference_steps by strength parameter: {strength}, the number "
                             f"of pipelinesteps is {num_inference_steps} which is < 1 and not appropriate for this "
                             "pipeline.")
        if uint8_device_inputs(self.vae, image, mask):
            # device-resident uint8 request (< 1 MB per 512^2 image over PCIe): `image / 127.5 - 1`, the mask
            # threshold and `image * (mask < 0.5)` (:123-147) run inside the VAE encoder's input kernel
            if image.shape[-2:] != mask.shape[-2:] or image.shape[0] != mask.shape[0] or mask.shape[1] != 1:
                raise ValueError("uint8 image [B,3,H,W] and mask [B,1,H,W] must agree in batch and size")
            masked_image = init_image = image.contiguous()
        else:
            mask, masked_image, init_image = prepare_mask_and_masked_image(image, mask, height, width,
                                                                           return_image=True)
        num_channels_latents = self.vae.config.latent_channels
        num_channels_unet = self.unet.config.in_channels
        if num_channels_unet not in (4, 9):
            raise ValueError(f"The unet {self.unet.__class__} should have either 4 or 9 input channels, not "
                             f"{num_channels_unet}.")
        return_image_latents = num_channels_unet == 4
        total = batch_size * num_images_per_prompt
        # strength < 1 (ref:pipeline_PowerPaint.py:916-941): start part-way down the schedule from the encoded
        # image noised to the first kept timestep; the fused loop just sees a shorter timestep / coefficient table
        latent_timestep = timesteps[:1].repeat(total)
        is_strength_max = strength == 1.0
        outs = self.prepare_latents(total, num_channels_latents, height, width, torch.float32, device,
                                    generator, latents, image=init_image, timestep=latent_timestep,
                                    is_strength_max=is_strength_max, return_noise=True,
                                    return_image_latents=return_image_latents)
        latents, noise = outs[0], outs[1]
        image_latents = outs[2] if return_image_latents else None
        mask, masked_image_latents = self.prepare_mask_latents(mask, masked_image, total, height, width, torch.float32,
                                                               device, generator, do_cfg)
        if num_channels_unet == 9 and \
                num_channels_latents + mask.shape[1] + masked_image_latents.shape[1] != num_channels_unet:
            raise ValueError("Incorrect configuration settings! The config of `pipeline.unet` expects "
                             f"{num_channels_unet} input channels but received {num_channels_latents} + "
                             f"{mask.shape[1]} + {masked_image_latents.shape[1]}.")
        extra_step_kwargs = self.prepare_extra_step_kwargs(generator, eta)
        if not hasattr(self.scheduler, "step_coefficients"):
            raise TypeError("the fused loop needs powerpaint_b200.schedulers.DDIMScheduler (step_coefficients)")
        coef = self.scheduler.step_coefficients(timesteps, eta=extra_step_kwargs.get("eta", 0.0))
        ucoef = scoef = pcoef = None
        finish = None
        kind = getattr(self.scheduler, "kind", "ddim")
        if kind == "unipc":
            ucoef = self.scheduler.unipc_coefficients(first=len(self.scheduler.timesteps) - len(timesteps))
        if kind == "plms":
            pcoef = self.scheduler.plms_coefficients(first=len(self.scheduler.timesteps) - len(timesteps))
        blend = None
        if num_channels_unet == 4:
            # 4-channel UNet (:1025-1035): after every step the known region is reset to the original latents noised
            # to the NEXT timestep (un-noised after the last step); the reference indexes image_latents[:1] / mask[:1]
            ac = self.scheduler.alphas_cumprod
            sqrt_alpha = [float(ac[int(timesteps[i + 1])]) ** 0.5 if i < len(timesteps) - 1 else 1.0
                          for i in range(len(timesteps))]
            blend = dict(x0=image_latents, mask=mask, noise=noise, sqrt_alpha=sqrt_alpha)
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
        # `scoef` / `pcoef` are passed only when such a scheduler is set: a denoiser whose `run` predates those kinds
        # keeps serving DDIM and UniPC unchanged
        opt = {k: v for k, v in (("scoef", scoef), ("pcoef", pcoef), ("randn_draws", noise_kw.get("randn_draws")))
               if v is not None}
        run = dict(latents=latents, prompt_embeds=prompt_embeds, timesteps=timesteps, coef=coef,
                   guidance_scale=guidance_scale,
                   extra=torch.cat([mask, masked_image_latents], dim=1) if num_channels_unet == 9 else None,
                   noise_fn=noise_kw.get("noise_fn"), ucoef=ucoef, blend=blend, callback=cb, **opt)
        return LoopInputs(run, finish, output_type, return_dict)
