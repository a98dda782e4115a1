"""Drop-in `UNet2DConditionModel` / `BrushNetModel` / `ControlNetModel` for the PowerPaint hot path.

Same names, `forward` arguments, return types and `.config` attributes as the reference classes
(powerpaint/models/unet_2d_condition.py:1040-1058 forward signature, :166 config;
powerpaint/models/BrushNet_CA.py:690-704 forward, :456-464 from_unet; diffusers ControlNetModel as
called at powerpaint/pipelines/pipeline_PowerPaint_ControlNet.py:1686-1694), but `forward` runs the
recorded CUDA program of `powerpaint_b200.engine.NetEngine` instead of ~800 eager library kernels.

Parameters live in an `nn.Module` tree whose `state_dict()` keys equal the diffusers names, so
`safetensors.torch.load_model(unet, "unet/unet.safetensors")` (reference app.py:111) and
`load_state_dict` work unchanged; the packed bf16 copies are rebuilt lazily after any load.

API conventions kept from the reference (SURVEY.md §8b): inputs are caller-owned NCHW tensors and
are never mutated; the BrushNet add *lists* are consumed with `pop(0)` exactly like the
reference does (unet_2d_condition.py:1223); outputs are fresh tensors in `self.dtype`.
"""
from __future__ import annotations

from dataclasses import asdict, dataclass
from typing import Any, Dict, List, Optional, Tuple, Union

import torch
import torch.nn as nn

from .. import ops
from ..config import Config
from ..engine import NetConfig, NetEngine, guess_mode_alphas
from ..loading import net_config_from_diffusers, net_config_to_diffusers
from .base import DiffusersModel
from .spec import param_shapes, synthetic_state_dict


@dataclass
class UNet2DConditionOutput:
    sample: torch.Tensor = None


@dataclass
class BrushNetOutput:
    up_block_res_samples: Tuple[torch.Tensor]
    down_block_res_samples: Tuple[torch.Tensor]
    mid_block_res_sample: torch.Tensor


@dataclass
class ControlNetOutput:
    down_block_res_samples: Tuple[torch.Tensor]
    mid_block_res_sample: torch.Tensor


def _make_config(cfg: NetConfig, **extra) -> Config:
    d = asdict(cfg)
    d.update(dict(sample_size=extra.pop("sample_size", 64), time_cond_proj_dim=None, flip_sin_to_cos=True,
                  freq_shift=0, act_fn="silu", use_linear_projection=False, only_cross_attention=False,
                  num_attention_heads=None, class_embed_type=None, num_class_embeds=None,
                  upcast_attention=False, resnet_time_scale_shift="default", downsample_padding=1,
                  projection_class_embeddings_input_dim=None, mid_block_type="UNetMidBlock2DCrossAttn",
                  center_input_sample=False, addition_embed_type=None,
                  # the remaining constructor arguments of the reference class (unet_2d_condition.py:166-218) at the
                  # only values the hot path implements, so that `config.<name>` reads the same on both sides
                  addition_embed_type_num_heads=64, addition_time_embed_dim=None, attention_type="default",
                  class_embeddings_concat=False, conv_in_kernel=3, conv_out_kernel=3, cross_attention_norm=None,
                  dropout=0.0, dual_cross_attention=False, encoder_hid_dim=None, encoder_hid_dim_type=None,
                  mid_block_only_cross_attention=None, resnet_out_scale_factor=1.0, resnet_skip_time_act=False,
                  reverse_transformer_layers_per_block=None, time_embedding_act_fn=None, time_embedding_dim=None,
                  time_embedding_type="positional", timestep_post_act=None, transformer_layers_per_block=1))
    d.update(extra)
    return Config(**d)


class _HotPathModel(DiffusersModel):
    KIND = "unet"

    def __init__(self, cfg: Optional[NetConfig] = None, sample_size: int = 64, **cfg_kwargs):
        super().__init__()
        if cfg is None:
            cfg = NetConfig(**cfg_kwargs)
        self._cfg = cfg
        self.config = _make_config(cfg, sample_size=sample_size)
        for name, shape in param_shapes(cfg, self.KIND).items():
            self._register(name, torch.zeros(shape))

    @classmethod
    def from_state_dict(cls, cfg: NetConfig, state_dict: Dict[str, torch.Tensor], **kw):
        m = cls(cfg, **kw)
        m.load_state_dict(state_dict, strict=True)
        return m

    @classmethod
    def synthetic(cls, cfg: NetConfig, seed: int = 1234, **kw):
        return cls.from_state_dict(cfg, synthetic_state_dict(cfg, cls.KIND, seed), **kw)

    def _make_engine(self, state_dict, device) -> NetEngine:
        return NetEngine(self._cfg, state_dict, self.KIND, device)

    # ---- checkpoint directories in the diffusers layout (ref:app.py:121-123,141-147,165-171)
    @classmethod
    def from_config(cls, config, **kw):
        """a diffusers `config.json` dictionary (or another model's `.config`) -> an uninitialised model"""
        d = dict(vars(config)) if not isinstance(config, dict) else dict(config)
        m = cls(net_config_from_diffusers(d, cls.KIND), sample_size=d.get("sample_size") or 64, **kw)
        if cls.KIND != "unet":
            m.config.global_pool_conditions = bool(d.get("global_pool_conditions", False))
        return m

    def _diffusers_config(self) -> dict:
        return net_config_to_diffusers(self._cfg, self.KIND, self.config)

    # ---- shared helpers
    @staticmethod
    def _timesteps(timestep, nb: int, device) -> torch.Tensor:
        t = timestep
        if not torch.is_tensor(t):
            t = torch.tensor([float(t)], dtype=torch.float32, device=device)
        else:
            t = t.to(device=device, dtype=torch.float32).reshape(-1)
        if t.numel() == 1:
            t = t.expand(nb)
        if t.numel() != nb:
            raise ValueError(f"timestep has {t.numel()} entries for a batch of {nb}")
        return t.contiguous()

    def _load_inputs(self, plan, sample, timestep, encoder_hidden_states, extra_channels=None):
        nb, c, h, w = sample.shape
        x = sample if extra_channels is None else torch.cat([sample, extra_channels.to(sample.dtype)], dim=1)
        x_in = plan.inputs["x_in"]
        xn = ops.nchw_to_nhwc(x.float().contiguous(), x_in.shape[-1])
        x_in.copy_(xn.view_as(x_in))
        plan.inputs["timesteps"].copy_(self._timesteps(timestep, nb, sample.device))
        # the cross-attention K / V^T projections of the prompt are recomputed on every eager forward (32 tiny
        # GEMMs over [nb, 77, 768]): an address / version key is not a content identity — a new prompt tensor
        # commonly lands on the freed block of the previous one. The fused loop projects once per call.
        plan.inputs["ctx"].copy_(encoder_hidden_states.to(torch.bfloat16))
        plan.ctx_program.run()

    @staticmethod
    def _nhwc_like(src: torch.Tensor, dst: torch.Tensor) -> torch.Tensor:
        """a caller's NCHW residual as the NHWC buffer `dst`; a globally pooled [B, C, 1, 1] residual is broadcast
        over the pixels, as the reference's `sample + residual` does"""
        src = src.float()
        if src.shape[2:] == (1, 1) and dst.shape[1] != 1:
            return src.reshape(src.shape[0], 1, src.shape[1]).expand(-1, dst.shape[1], -1).to(dst.dtype)
        return ops.nchw_to_nhwc(src.contiguous()).view_as(dst)

    def _side_plan_options(self, guess_mode: bool, n_res: int):
        """(per-residual factors, pool) of a side net's forward: the logspace(-1, 0, n_res) factors in guess mode
        unless the net pools (the reference never applies them to a pooled net)"""
        pool = bool(self.config.global_pool_conditions)
        return (guess_mode_alphas(n_res) if guess_mode and not pool else None), pool

    @staticmethod
    def _pooled(t: torch.Tensor) -> torch.Tensor:
        """the [B, C, 1, 1] mean the reference returns for a pooled net (every pixel of `t` holds it)"""
        return t[:, :, :1, :1].contiguous()

    @staticmethod
    def _to_nchw(t: torch.Tensor, nb, h, w, dtype) -> torch.Tensor:
        c = t.shape[-1]
        return ops.nhwc_to_nchw(t.view(nb, h, w, c)).to(dtype)


class UNet2DConditionModel(_HotPathModel):
    KIND = "unet"

    @torch.no_grad()
    def forward(self, sample: torch.Tensor, timestep: Union[torch.Tensor, float, int],
                encoder_hidden_states: torch.Tensor, class_labels: Optional[torch.Tensor] = None,
                timestep_cond: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                cross_attention_kwargs: Optional[Dict[str, Any]] = None,
                added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                down_block_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
                mid_block_additional_residual: Optional[torch.Tensor] = None,
                down_intrablock_additional_residuals: Optional[Tuple[torch.Tensor]] = None,
                encoder_attention_mask: Optional[torch.Tensor] = None, return_dict: bool = True,
                down_block_add_samples: Optional[List[torch.Tensor]] = None,
                mid_block_add_sample: Optional[torch.Tensor] = None,
                up_block_add_samples: Optional[List[torch.Tensor]] = None):
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond),
                        ("attention_mask", attention_mask), ("added_cond_kwargs", added_cond_kwargs),
                        ("down_intrablock_additional_residuals", down_intrablock_additional_residuals),
                        ("encoder_attention_mask", encoder_attention_mask)):
            if v is not None:
                raise NotImplementedError(f"`{name}` is outside the PowerPaint SD-1.5 hot path")
        if cross_attention_kwargs:
            raise NotImplementedError("cross_attention_kwargs (LoRA scale / GLIGEN) are outside the hot path")
        if sample.dim() != 4 or sample.shape[1] != self._cfg.in_channels:
            raise ValueError(f"sample must be [B, {self._cfg.in_channels}, H, W], got {tuple(sample.shape)}")
        nb, _, h, w = sample.shape
        is_brushnet = (down_block_add_samples is not None and mid_block_add_sample is not None
                       and up_block_add_samples is not None)
        is_controlnet = mid_block_additional_residual is not None and down_block_additional_residuals is not None
        with torch.cuda.device(self.device):  # launches go to the stream of the model's device
            return self._forward(sample, timestep, encoder_hidden_states, is_brushnet, is_controlnet,
                                 down_block_add_samples, mid_block_add_sample, up_block_add_samples,
                                 down_block_additional_residuals, mid_block_additional_residual, return_dict)

    def _forward(self, sample, timestep, encoder_hidden_states, is_brushnet, is_controlnet, down_block_add_samples,
                 mid_block_add_sample, up_block_add_samples, down_block_additional_residuals,
                 mid_block_additional_residual, return_dict):
        nb, _, h, w = sample.shape
        eng = self.engine()
        plan = eng.plan(nb, h, w, encoder_hidden_states.shape[1], with_brushnet_adds=is_brushnet,
                        with_controlnet_res=is_controlnet)
        self._load_inputs(plan, sample, timestep, encoder_hidden_states)
        if is_brushnet:
            nd, nu = len(plan.inputs["adds_down"]), len(plan.inputs["adds_up"])
            if len(down_block_add_samples) != nd or len(up_block_add_samples) != nu:
                raise ValueError(f"expected {nd} down / {nu} up add samples, got "
                                 f"{len(down_block_add_samples)} / {len(up_block_add_samples)}")
            # the reference consumes the lists with pop(0) (unet_2d_condition.py:1223,:1232-1253,:1316-1339)
            for dst in plan.inputs["adds_down"]:
                src = down_block_add_samples.pop(0)
                dst.copy_(self._nhwc_like(src, dst))
            plan.inputs["add_mid"].copy_(self._nhwc_like(mid_block_add_sample, plan.inputs["add_mid"]))
            for dst in plan.inputs["adds_up"]:
                src = up_block_add_samples.pop(0)
                dst.copy_(self._nhwc_like(src, dst))
        if is_controlnet:
            if len(down_block_additional_residuals) != len(plan.inputs["cn_down"]):
                raise ValueError("wrong number of down_block_additional_residuals")
            for dst, src in zip(plan.inputs["cn_down"], down_block_additional_residuals):
                dst.copy_(self._nhwc_like(src, dst))
            plan.inputs["cn_mid"].copy_(self._nhwc_like(mid_block_additional_residual, plan.inputs["cn_mid"]))
        plan.program.launch()
        out = self._to_nchw(plan.outputs["eps"], nb, h, w, self.dtype)
        if not return_dict:
            return (out,)
        return UNet2DConditionOutput(sample=out)


class BrushNetModel(_HotPathModel):
    KIND = "brushnet"

    def __init__(self, cfg: Optional[NetConfig] = None, **kw):
        if cfg is None and "in_channels" not in kw:
            kw["in_channels"] = 4
        super().__init__(cfg, **kw)
        self.config.brushnet_conditioning_channel_order = "rgb"
        self.config.global_pool_conditions = False

    @classmethod
    def from_unet(cls, unet: UNet2DConditionModel, brushnet_conditioning_channel_order: str = "rgb",
                  conditioning_embedding_out_channels=(16, 32, 96, 256), load_weights_from_unet: bool = True,
                  conditioning_channels: int = 5):
        """reference BrushNet_CA.py:456-542: clone the trunk; conv_in weights go to input channels
        0:4 AND 4:8 of conv_in_condition, channel 8 (mask) stays zero; zero-convs stay zero."""
        cfg = NetConfig(**{**asdict(unet._cfg), "conditioning_channels": conditioning_channels})
        bn = cls(cfg, sample_size=unet.config.sample_size)
        if load_weights_from_unet:
            src = unet.state_dict()
            dst = bn.state_dict()
            new = {}
            for k, v in dst.items():
                if k == "conv_in_condition.weight":
                    w = torch.zeros_like(v)
                    w[:, :4] = src["conv_in.weight"]
                    w[:, 4:8] = src["conv_in.weight"]
                    new[k] = w
                elif k == "conv_in_condition.bias":
                    new[k] = src["conv_in.bias"].clone()
                elif k in src and src[k].shape == v.shape:
                    new[k] = src[k].clone()
                else:
                    new[k] = v  # zero-initialised 1x1 convs (zero_module, BrushNet_CA.py:955-958)
            bn.load_state_dict(new)
        bn.to(unet.device)
        bn._out_dtype = unet.dtype
        return bn

    @torch.no_grad()
    def forward(self, sample: torch.FloatTensor, timestep: Union[torch.Tensor, float, int],
                encoder_hidden_states: torch.Tensor, brushnet_cond: torch.FloatTensor,
                conditioning_scale: float = 1.0, class_labels: Optional[torch.Tensor] = None,
                timestep_cond: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                cross_attention_kwargs: Optional[Dict[str, Any]] = None, guess_mode: bool = False,
                return_dict: bool = True):
        """`guess_mode` and `config.global_pool_conditions` as BrushNet_CA.py:905-943: in guess mode residual k is
        scaled by logspace(-1, 0, 28)[k] x conditioning_scale; a pooled net skips those factors and returns the
        spatial mean of each residual, [B, C, 1, 1]."""
        for name, v in (("class_labels", class_labels), ("timestep_cond", timestep_cond),
                        ("attention_mask", attention_mask), ("added_cond_kwargs", added_cond_kwargs)):
            if v is not None:
                raise NotImplementedError(f"`{name}` is outside the PowerPaint SD-1.5 hot path")
        nb, _, h, w = sample.shape
        with torch.cuda.device(self.device):
            shapes_d, shape_m, shapes_u = self.engine()._state_shapes(nb, h, w)
            alphas, pool = self._side_plan_options(guess_mode, len(shapes_d) + 1 + len(shapes_u))
            # one recorded program for every conditioning_scale: the zero-conv epilogues read it from a device scalar
            plan = self.engine().plan(nb, h, w, encoder_hidden_states.shape[1], side_alphas=alphas, side_pool=pool)
            plan.scale_dev.fill_(float(conditioning_scale))
            self._load_inputs(plan, sample, timestep, encoder_hidden_states, extra_channels=brushnet_cond)
            plan.program.launch()
            down = [self._to_nchw(t, nb, s[1], s[2], self.dtype) for t, s in zip(plan.outputs["down"], shapes_d)]
            mid = self._to_nchw(plan.outputs["mid"], nb, shape_m[1], shape_m[2], self.dtype)
            up = [self._to_nchw(t, nb, s[1], s[2], self.dtype) for t, s in zip(plan.outputs["up"], shapes_u)]
            if pool:
                down, mid, up = [self._pooled(t) for t in down], self._pooled(mid), [self._pooled(t) for t in up]
        if not return_dict:
            return (down, mid, up)
        return BrushNetOutput(down_block_res_samples=down, mid_block_res_sample=mid, up_block_res_samples=up)


class ControlNetModel(_HotPathModel):
    KIND = "controlnet"

    def __init__(self, cfg: Optional[NetConfig] = None, **kw):
        if cfg is None and "in_channels" not in kw:
            kw["in_channels"] = 4
        super().__init__(cfg, **kw)
        self.config.global_pool_conditions = False

    @torch.no_grad()
    def forward(self, sample: torch.FloatTensor, timestep: Union[torch.Tensor, float, int],
                encoder_hidden_states: torch.Tensor, controlnet_cond: torch.FloatTensor,
                conditioning_scale: float = 1.0, class_labels: Optional[torch.Tensor] = None,
                timestep_cond: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                cross_attention_kwargs: Optional[Dict[str, Any]] = None, guess_mode: bool = False,
                return_dict: bool = True):
        """`guess_mode` and `config.global_pool_conditions` as diffusers 0.27.0 `ControlNetModel.forward` (restated
        as recalled, not copied): in guess mode residual k of the 12 down + mid residuals is scaled by
        logspace(-1, 0, 13)[k] x conditioning_scale; a pooled net skips those factors and returns the spatial mean
        of each residual, [B, C, 1, 1]."""
        nb, _, h, w = sample.shape
        if tuple(controlnet_cond.shape[2:]) != (8 * h, 8 * w):
            raise ValueError("controlnet_cond must be 8x the latent resolution")
        with torch.cuda.device(self.device):
            eng = self.engine()
            shapes_d, shape_m, _ = eng._state_shapes(nb, h, w)
            alphas, pool = self._side_plan_options(guess_mode, len(shapes_d) + 1)
            plan = eng.plan(nb, h, w, encoder_hidden_states.shape[1], side_alphas=alphas, side_pool=pool)
            # t-independent (SURVEY.md App. C (3)): the 8-conv embedding is re-run only when the staged control
            # image actually differs (content comparison on the device; an address is not an identity)
            ci = plan.inputs["cond_in"]
            new_ci = ops.nchw_to_nhwc(controlnet_cond.float().contiguous(), ci.shape[-1]).view_as(ci)
            if not plan.outputs.get("cond_valid") or not torch.equal(new_ci, ci):
                ci.copy_(new_ci)
                plan.cond_program.run()
                plan.outputs["cond_valid"] = True
            plan.scale_dev.fill_(float(conditioning_scale))
            self._load_inputs(plan, sample, timestep, encoder_hidden_states)
            plan.program.launch()
            down = [self._to_nchw(t, nb, sh[1], sh[2], self.dtype) for t, sh in zip(plan.outputs["down"], shapes_d)]
            mid = self._to_nchw(plan.outputs["mid"], nb, shape_m[1], shape_m[2], self.dtype)
            if pool:
                down, mid = [self._pooled(t) for t in down], self._pooled(mid)
        if not return_dict:
            return (down, mid)
        return ControlNetOutput(down_block_res_samples=down, mid_block_res_sample=mid)


class MultiControlNetModel(nn.Module):
    """Several ControlNets whose residuals are summed in net order: diffusers 0.27.0 `MultiControlNetModel` as the
    reference wraps a list of ControlNets (pipeline_PowerPaint_ControlNet.py:306; restated as recalled, not copied).
    `forward` runs each net eagerly on the kernel path; the fused loop (`FusedDenoiser`) records all nets into one
    step program instead."""

    def __init__(self, controlnets):
        super().__init__()
        self.nets = nn.ModuleList(controlnets)

    @property
    def dtype(self) -> torch.dtype:
        return self.nets[0].dtype

    @property
    def device(self) -> torch.device:
        return self.nets[0].device

    @torch.no_grad()
    def forward(self, sample: torch.FloatTensor, timestep: Union[torch.Tensor, float, int],
                encoder_hidden_states: torch.Tensor, controlnet_cond: List[torch.Tensor],
                conditioning_scale: List[float], class_labels: Optional[torch.Tensor] = None,
                timestep_cond: Optional[torch.Tensor] = None, attention_mask: Optional[torch.Tensor] = None,
                added_cond_kwargs: Optional[Dict[str, torch.Tensor]] = None,
                cross_attention_kwargs: Optional[Dict[str, Any]] = None, guess_mode: bool = False,
                return_dict: bool = True):
        """(down residuals, mid residual): the sum over nets, net 0 first. A tuple whatever `return_dict` says."""
        down = mid = None
        for i, (image, scale, net) in enumerate(zip(controlnet_cond, conditioning_scale, self.nets)):
            d, m = net(sample, timestep, encoder_hidden_states, image, scale, class_labels=class_labels,
                       timestep_cond=timestep_cond, attention_mask=attention_mask,
                       added_cond_kwargs=added_cond_kwargs, cross_attention_kwargs=cross_attention_kwargs,
                       guess_mode=guess_mode, return_dict=False)
            if i == 0:
                down, mid = d, m
            else:
                down = [a + b for a, b in zip(down, d)]
                mid = mid + m
        return down, mid
