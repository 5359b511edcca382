"""Soprano TTS (reference: mlx_audio/tts/models/soprano/__init__.py)."""
from .soprano import DecoderConfig, Model, ModelConfig, SopranoDecoder, SopranoModel
from .text import clean_text

__all__ = ["Model", "ModelConfig", "DecoderConfig", "SopranoModel", "SopranoDecoder", "clean_text"]
