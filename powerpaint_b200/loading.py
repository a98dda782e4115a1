"""Checkpoint directories in the diffusers layout — the data format on the caller's side of the hot path.

The reference assembles its models with `from_pretrained` (ref:app.py:91-93 pipeline, :121-123 ControlNet, :141-147 and
:165-171 UNet, :157-164 BrushNet pipeline) and then overwrites weights with `safetensors.torch.load_model`. The classes
here read the same directories:

    <root>/model_index.json                                   which component lives in which subfolder
    <root>/unet/config.json                                   diffusers config keys -> NetConfig (validated)
    <root>/unet/diffusion_pytorch_model[.<variant>].safetensors | .bin
    <root>/vae/config.json, <root>/vae/diffusion_pytorch_model...
    <root>/scheduler/scheduler_config.json
    <root>/text_encoder/, <root>/tokenizer/                   transformers' own format (loaded by transformers)

A name that is not a local directory is looked up in the local Hugging Face cache through `huggingface_hub` (the library
diffusers itself uses; it downloads only if the machine has network access and `local_files_only` is False). Host code
only: everything is loaded on the CPU, `.to("cuda")` moves it like upstream.
"""
from __future__ import annotations

import json
import os
from dataclasses import fields
from typing import Dict, Optional

import torch

from .engine import NetConfig

# diffusers config keys whose value must be the one the hot path implements (anything else: NotImplementedError)
_FIXED = {
    "act_fn": "silu", "use_linear_projection": False, "upcast_attention": False, "resnet_time_scale_shift": "default",
    "class_embed_type": None, "addition_embed_type": None, "time_embedding_type": "positional",
    "flip_sin_to_cos": True, "freq_shift": 0, "downsample_padding": 1, "dual_cross_attention": False,
    "num_class_embeds": None, "center_input_sample": False, "time_cond_proj_dim": None, "encoder_hid_dim": None,
    "encoder_hid_dim_type": None, "transformer_layers_per_block": 1, "attention_type": "default",
    "conv_in_kernel": 3, "conv_out_kernel": 3, "cross_attention_norm": None, "num_attention_heads": None,
    "resnet_skip_time_act": False, "resnet_out_scale_factor": 1.0, "time_embedding_act_fn": None,
    "timestep_post_act": None, "time_embedding_dim": None, "mid_block_only_cross_attention": None,
    "class_embeddings_concat": False, "reverse_transformer_layers_per_block": None, "dropout": 0.0,
    "global_pool_conditions": False, "mid_block_type": "UNetMidBlock2DCrossAttn",
}


def resolve_checkpoint_dir(name_or_path, subfolder: Optional[str] = None, revision: Optional[str] = None,
                           local_files_only: bool = False, cache_dir: Optional[str] = None) -> str:
    """local directory, or a snapshot of a hub repository in the local cache"""
    name_or_path = os.fspath(name_or_path)
    if os.path.isdir(name_or_path):
        root = name_or_path
    else:
        try:
            from huggingface_hub import snapshot_download

            root = snapshot_download(name_or_path, revision=revision, local_files_only=local_files_only,
                                     cache_dir=cache_dir)
        except Exception as e:  # noqa: BLE001  (whatever the hub client raises: say what was looked for)
            raise EnvironmentError(f"{name_or_path} is not a local directory and no snapshot of it could be obtained "
                                   f"from the Hugging Face cache / hub ({type(e).__name__}: {e})") from e
    d = os.path.join(root, subfolder) if subfolder else root
    if not os.path.isdir(d):
        raise EnvironmentError(f"{d} does not exist (subfolder {subfolder!r} of {name_or_path})")
    return d


def load_json(directory: str, name: str) -> dict:
    path = os.path.join(directory, name)
    if not os.path.isfile(path):
        raise EnvironmentError(f"{path} not found")
    with open(path) as f:
        return json.load(f)


def load_weights(directory: str, variant: Optional[str] = None, stem: str = "diffusion_pytorch_model"
                 ) -> Dict[str, torch.Tensor]:
    """`<stem>[.<variant>].safetensors`, else the pickled `.bin` (weights only)"""
    v = f".{variant}" if variant else ""
    st = os.path.join(directory, f"{stem}{v}.safetensors")
    if os.path.isfile(st):
        from safetensors.torch import load_file

        return load_file(st, device="cpu")
    pt = os.path.join(directory, f"{stem}{v}.bin")
    if os.path.isfile(pt):
        return torch.load(pt, map_location="cpu", weights_only=True)
    raise EnvironmentError(f"no {stem}{v}.safetensors or {stem}{v}.bin in {directory}")


def net_config_from_diffusers(cfg: dict, kind: str) -> NetConfig:
    """diffusers `config.json` -> NetConfig; options the hot path does not implement are refused by name"""
    for k, want in _FIXED.items():
        if k == "global_pool_conditions" and kind in ("controlnet", "brushnet"):
            continue  # side nets pool their residuals on the kernel path (pp_pool_broadcast)
        if k in cfg and cfg[k] != want and not (isinstance(want, float) and float(cfg[k]) == want):
            raise NotImplementedError(f"config.{k} = {cfg[k]!r}: the hot path implements {want!r} only (SD-1.5 family)")
    oca = cfg.get("only_cross_attention", False)
    if oca if isinstance(oca, bool) else any(oca):
        raise NotImplementedError("config.only_cross_attention: not implemented")
    heads = cfg.get("attention_head_dim", 8)
    if isinstance(heads, (list, tuple)):
        if len(set(heads)) != 1:
            raise NotImplementedError(f"config.attention_head_dim = {heads}: one value for all blocks only (SD-1.5)")
        heads = heads[0]
    known = {f.name for f in fields(NetConfig)}
    kw = {k: (tuple(v) if isinstance(v, list) else v) for k, v in cfg.items() if k in known}
    kw["attention_head_dim"] = int(heads)
    if kind == "controlnet":
        kw["controlnet_cond_channels"] = int(cfg.get("conditioning_channels", 3))
        kw.pop("conditioning_channels", None)
        kw.setdefault("in_channels", 4)
    elif kind == "brushnet":
        kw.setdefault("in_channels", 4)
    return NetConfig(**kw)


def net_config_to_diffusers(cfg: NetConfig, kind: str, config_surface) -> dict:
    """what `save_pretrained` writes: the model's `config` entries under the diffusers class name"""
    name = {"unet": "UNet2DConditionModel", "brushnet": "BrushNetModel", "controlnet": "ControlNetModel"}[kind]
    out = {"_class_name": name, "_diffusers_version": "0.27.0"}
    for k, v in vars(config_surface).items():
        if k.startswith("_") or callable(v):
            continue
        out[k] = list(v) if isinstance(v, tuple) else v
    if kind == "controlnet":
        out["conditioning_channels"] = cfg.controlnet_cond_channels
        out.pop("controlnet_cond_channels", None)
    return out


# deprecated attention parameter names of older VAE checkpoints (diffusers renames them on load)
_VAE_ATTN_RENAMES = {".query.": ".to_q.", ".key.": ".to_k.", ".value.": ".to_v.", ".proj_attn.": ".to_out.0."}


def rename_deprecated_vae_attention(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
    out = {}
    for k, v in state_dict.items():
        if ".attentions." in k:
            for old, new in _VAE_ATTN_RENAMES.items():
                k = k.replace(old, new)
            if v.dim() == 4 and v.shape[-2:] == (1, 1) and ".to_" in k:  # very old checkpoints: 1x1 convs
                v = v[:, :, 0, 0]
        out[k] = v
    return out


def save_weights(state_dict: Dict[str, torch.Tensor], directory: str, stem: str = "diffusion_pytorch_model",
                 variant: Optional[str] = None):
    from safetensors.torch import save_file

    os.makedirs(directory, exist_ok=True)
    v = f".{variant}" if variant else ""
    save_file({k: t.detach().cpu().contiguous() for k, t in state_dict.items()},
              os.path.join(directory, f"{stem}{v}.safetensors"))
