"""diffusers-style model folders without diffusers: ``config.json`` + ``diffusion_pytorch_model.safetensors`` (or the
older ``.bin``), as written by ``save_pretrained`` of the reference's classes and of the diffusers models it loads
(/root/reference/inference.py:218-254, 337-376: ``X.from_pretrained(path, subfolder=..., low_cpu_mem_usage=False,
device_map=None)`` followed by ``.to(dtype).eval().cuda()``).

Only local folders are read (there is no hub access); unknown configuration keys are dropped the way diffusers'
``register_to_config`` / ``extract_init_dict`` does (private ``_*`` keys always, others when the constructor does not take
them), and the state dict must match the module's keys exactly -- which is the check that the class really is a drop-in
for the checkpoint.
"""
from __future__ import annotations

import inspect
import json
import os
from typing import Optional

import torch

CONFIG_NAME = "config.json"
WEIGHTS_SAFE = "diffusion_pytorch_model.safetensors"
WEIGHTS_BIN = "diffusion_pytorch_model.bin"


def _jsonable(v):
    if isinstance(v, (tuple, list)):
        return [_jsonable(x) for x in v]
    if isinstance(v, dict):
        return {k: _jsonable(x) for k, x in v.items()}
    if isinstance(v, (torch.dtype, torch.device)):
        return str(v)
    return v


class PretrainedMixin:
    """``save_pretrained`` / ``from_pretrained``, and diffusers' ``dtype`` / ``device`` properties, for an ``nn.Module``
    that keeps its constructor arguments in ``self.config`` (a dict)."""

    config_name = CONFIG_NAME

    @property
    def dtype(self) -> torch.dtype:
        return next(self.parameters()).dtype

    @property
    def device(self) -> torch.device:
        return next(self.parameters()).device

    def save_pretrained(self, path: str, safe_serialization: bool = True):
        os.makedirs(path, exist_ok=True)
        cfg = {"_class_name": type(self).__name__, **{k: _jsonable(v) for k, v in dict(self.config).items()}}
        with open(os.path.join(path, self.config_name), "w") as f:
            json.dump(cfg, f, indent=2, sort_keys=True)
        sd = {k: v.detach().contiguous().cpu() for k, v in self.state_dict().items()}
        if safe_serialization:
            from safetensors.torch import save_file
            save_file(sd, os.path.join(path, WEIGHTS_SAFE))
        else:
            torch.save(sd, os.path.join(path, WEIGHTS_BIN))

    @classmethod
    def from_config(cls, config: dict, **overrides):
        """Instantiate from a (diffusers-style) configuration dict: private ``_*`` keys are dropped, and so are keys the
        constructor does not take unless it accepts ``**kwargs``."""
        cfg = {k: v for k, v in dict(config).items() if not k.startswith("_")}
        cfg.update(overrides)
        params = inspect.signature(cls.__init__).parameters
        if not any(p.kind is inspect.Parameter.VAR_KEYWORD for p in params.values()):
            cfg = {k: v for k, v in cfg.items() if k in params}
        return cls(**cfg)

    @classmethod
    def from_pretrained(cls, path: str, subfolder: Optional[str] = None, low_cpu_mem_usage: bool = False,
                        device_map=None, torch_dtype=None, **overrides):
        folder = os.path.join(path, subfolder) if subfolder else path
        if not os.path.isdir(folder):
            raise FileNotFoundError(f"{folder}: only local model folders can be loaded (no hub access)")
        with open(os.path.join(folder, cls.config_name)) as f:
            model = cls.from_config(json.load(f), **overrides)
        safe, legacy = os.path.join(folder, WEIGHTS_SAFE), os.path.join(folder, WEIGHTS_BIN)
        if os.path.exists(safe):
            from safetensors.torch import load_file
            sd = load_file(safe)
        elif os.path.exists(legacy):
            sd = torch.load(legacy, map_location="cpu", weights_only=True)
        else:
            raise FileNotFoundError(f"{folder}: neither {WEIGHTS_SAFE} nor {WEIGHTS_BIN}")
        model.load_state_dict(sd)  # strict: the key set must be exactly the checkpoint's
        return model.to(torch_dtype) if torch_dtype is not None else model
