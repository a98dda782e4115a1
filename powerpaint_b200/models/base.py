"""What every kernel-backed module shares: parameters in an `nn.Module` tree under the upstream state-dict names, and
an engine that records CUDA programs from them, built on first use on the module's device and dropped whenever the
parameters change. The diffusers-layout checkpoint directory of the nets and the VAE is `DiffusersModel`'s."""
from __future__ import annotations

import json
import os
from typing import Dict, Optional

import torch
import torch.nn as nn

from ..engine import Recorder
from ..loading import load_json, load_weights, resolve_checkpoint_dir, save_weights


class KernelModule(nn.Module):
    """Subclasses register their parameters with `_register` and build their engine in `_make_engine`."""

    def __init__(self):
        super().__init__()
        self._engine: Optional[Recorder] = None
        self._out_dtype = torch.float32
        self._generation = 0  # bumped whenever the parameters change: recorded programs of older engines are stale
        self.register_load_state_dict_post_hook(lambda module, incompatible: module._invalidate())

    def _register(self, name: str, value: torch.Tensor):
        parts = name.split(".")
        mod = self
        for p in parts[:-1]:
            if not hasattr(mod, p):
                mod.add_module(p, nn.Module())
            mod = getattr(mod, p)
        mod.register_parameter(parts[-1], nn.Parameter(value, requires_grad=False))

    def _invalidate(self):
        self._engine = None
        self._generation += 1

    @property
    def generation(self) -> int:
        return self._generation

    def _apply(self, fn, *a, **k):  # .to() / .cuda() / .half() move parameters: repack lazily
        self._invalidate()
        return super()._apply(fn, *a, **k)

    @property
    def dtype(self) -> torch.dtype:
        return self._out_dtype

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def to(self, *args, **kwargs):
        # the reference app calls unet.to(dtype=fp16); compute is always bf16 x bf16 -> fp32 here,
        # the requested dtype only selects the dtype of returned tensors
        dtype = kwargs.pop("dtype", None)
        for a in args:
            if isinstance(a, torch.dtype):
                dtype = a
        if dtype is not None:
            self._out_dtype = dtype
        args = tuple(a for a in args if not isinstance(a, torch.dtype))
        return super().to(*args, **kwargs) if args or kwargs else self

    def engine(self) -> Recorder:
        if self._engine is None:
            dev = self.device
            if dev.type != "cuda":
                raise RuntimeError(f"{type(self).__name__} must be on a CUDA device (got {dev}): there is no CPU path")
            self._engine = self._make_engine(dict(self.state_dict()), dev)
        return self._engine

    def _make_engine(self, state_dict: Dict[str, torch.Tensor], device: torch.device) -> Recorder:
        raise NotImplementedError


class DiffusersModel(KernelModule):
    """A model stored as a diffusers directory: `config.json` + `diffusion_pytorch_model[.<variant>].safetensors | .bin`
    (ref:app.py:121-123,141-147,165-171). Subclasses convert the config (`from_config`, `_diffusers_config`) and may
    rename the keys a checkpoint file holds (`_checkpoint_state_dict`)."""

    def _diffusers_config(self) -> dict:
        raise NotImplementedError

    @staticmethod
    def _checkpoint_state_dict(state_dict: Dict[str, torch.Tensor]) -> Dict[str, torch.Tensor]:
        return state_dict

    @classmethod
    def from_pretrained(cls, pretrained_model_name_or_path, subfolder: Optional[str] = None, torch_dtype=None,
                        revision: Optional[str] = None, variant: Optional[str] = None, local_files_only: bool = False,
                        cache_dir: Optional[str] = None, **unused):
        """`ModelMixin.from_pretrained` for a local directory or a cached hub snapshot: strict load, on the CPU.
        `torch_dtype` selects the dtype of returned tensors (compute is bf16 x bf16 -> fp32 whatever it says)."""
        d = resolve_checkpoint_dir(pretrained_model_name_or_path, subfolder, revision, local_files_only, cache_dir)
        model = cls.from_config(load_json(d, "config.json"))
        model.load_state_dict(cls._checkpoint_state_dict(load_weights(d, variant)), strict=True)
        if torch_dtype is not None:
            model.to(dtype=torch_dtype)
        return model

    def save_pretrained(self, save_directory, variant: Optional[str] = None, **unused):
        os.makedirs(save_directory, exist_ok=True)
        with open(os.path.join(save_directory, "config.json"), "w") as f:
            json.dump(self._diffusers_config(), f, indent=2, sort_keys=True)
        save_weights(self.state_dict(), save_directory, variant=variant)
