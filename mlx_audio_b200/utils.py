"""Model discovery + generic loader with the reference's flow and signatures (utils.py:108-416):
``config.json`` -> model_type -> ``mlx_audio_b200.<category>.models.<type>.{Model, ModelConfig}`` ->
``Model(config)`` -> ``sanitize`` -> ``load_weights`` -> ``eval`` -> ``post_load_hook``.
Local directories only (there is no network); weights are read with safetensors into torch tensors."""
from __future__ import annotations

import glob
import importlib
import json
from pathlib import Path
from typing import Optional

import numpy as np
import torch

from .dsp import STR_TO_WINDOW_FN, ISTFTCache, bartlett, blackman, hamming, hanning, istft, mel_filters, stft  # noqa: F401 (utils.py:31-40 re-exports)

MODEL_REMAPPING = {"tts": {"kokoro": "kokoro", "qwen3_tts": "qwen3_tts", "soprano": "soprano"}, "stt": {"whisper": "whisper"}}


def get_model_path(path_or_repo: str, **_) -> Path:
    p = Path(path_or_repo)
    if not p.exists():
        raise FileNotFoundError(f"Model path {path_or_repo} does not exist locally (no network in this build; utils.py:108-152)")
    return p


def load_config(model_path: Path) -> dict:
    cfg = Path(model_path) / "config.json"
    if not cfg.exists():
        raise FileNotFoundError(f"Config not found at {model_path}")
    with open(cfg) as f:
        return json.load(f)


def get_model_class(model_type: str, category: str, model_name=None):
    """utils.py:259-318: import <category>.models.<model_type> and return the module exposing Model / ModelConfig.  When the type does
    not resolve (a Soprano checkpoint says ``model_type: "qwen3"``), a part of the directory name ``model_name`` (its "-" separated
    pieces) that names a model of the category is used instead, as the reference's name hint does."""
    remap = MODEL_REMAPPING.get(category, {})
    mapped = remap.get(model_type, model_type)
    try:
        return importlib.import_module(f"mlx_audio_b200.{category}.models.{mapped}")
    except ImportError as e:
        if e.name != f"mlx_audio_b200.{category}.models.{mapped}":
            raise
        hint = next((remap[p] for p in (model_name or []) if p in remap), None)
        if hint is None:
            raise ValueError(f"Model type {model_type} not supported for {category} on the H100 path") from e
        return importlib.import_module(f"mlx_audio_b200.{category}.models.{hint}")


def load_weights(model_path: Path) -> dict:
    from safetensors.torch import load_file
    files = sorted(glob.glob(str(Path(model_path) / "*.safetensors")))
    if not files:
        raise FileNotFoundError(f"No safetensors found in {model_path}")
    out = {}
    for f in files:
        out.update(load_file(f))
    return out


def base_load_model(model_path, category: str, lazy: bool = False, strict: bool = True, model_type: Optional[str] = None,
                    device="cuda", **kwargs):
    path = get_model_path(str(model_path))
    config = load_config(path)
    mt = model_type or config.get("model_type") or config.get("architecture")
    if mt is None:
        parts = path.name.lower().replace("_", "-").split("-")
        known = MODEL_REMAPPING.get(category, {})
        mt = next((p for p in parts if p in known), None)
    if mt is None:
        raise ValueError(f"Could not determine model_type for {model_path}")
    mod = get_model_class(mt, category, path.name.lower().replace("_", "-").split("-"))
    cfg_cls = getattr(mod, "ModelConfig", None)
    if cfg_cls is not None and "model_path" in getattr(cfg_cls, "__dataclass_fields__", {}):
        config = {**config, "model_path": str(model_path)}              # utils.py:365 (Soprano picks its decoder from it)
    cfg = cfg_cls.from_dict(config) if cfg_cls is not None and hasattr(cfg_cls, "from_dict") else config
    model = mod.Model(cfg, device=device)
    weights = load_weights(path)
    if hasattr(model, "sanitize"):
        weights = model.sanitize(weights)
    model.load_weights(list(weights.items()), strict=strict)
    model.eval()
    if hasattr(mod.Model, "post_load_hook"):
        model = mod.Model.post_load_hook(model, path)
    return model


def load_model(model_path, lazy: bool = False, strict: bool = False, **kwargs):
    """utils.py:832: category inferred from the config's model_type."""
    cfg = load_config(get_model_path(str(model_path)))
    mt = kwargs.get("model_type") or cfg.get("model_type") or cfg.get("architecture")
    category = next((c for c, m in MODEL_REMAPPING.items() if mt in m), "tts")
    return base_load_model(model_path, category, lazy, strict, **kwargs)


def resample_audio(audio, orig_sr: int, target_sr: int, axis: int = -1):
    """utils.py:541-578: same type out as in -- NumPy through the reference's SciPy call, torch CUDA tensors through our
    polyphase kernel (same filter, same indexing)."""
    from .resample import resample_audio_array
    return resample_audio_array(audio, orig_sr, target_sr, axis=axis)
