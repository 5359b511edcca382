"""Qwen3-TTS (reference: mlx_audio/tts/models/qwen3_tts/__init__.py)."""
from .config import (ModelConfig, Qwen3TTSSpeakerEncoderConfig, Qwen3TTSTalkerCodePredictorConfig, Qwen3TTSTalkerConfig,
                     Qwen3TTSTokenizerConfig, Qwen3TTSTokenizerDecoderConfig, Qwen3TTSTokenizerEncoderConfig)
from .qwen3_tts import Model
from .speaker_encoder import Qwen3TTSSpeakerEncoder
from .speech_tokenizer import Qwen3TTSSpeechTokenizer, Qwen3TTSSpeechTokenizerDecoder, Qwen3TTSSpeechTokenizerEncoder
from .talker import Qwen3TTSTalkerForConditionalGeneration

__all__ = ["Model", "ModelConfig", "Qwen3TTSTalkerConfig", "Qwen3TTSTalkerCodePredictorConfig", "Qwen3TTSTokenizerConfig",
           "Qwen3TTSTokenizerDecoderConfig", "Qwen3TTSTokenizerEncoderConfig", "Qwen3TTSSpeakerEncoderConfig", "Qwen3TTSSpeakerEncoder", "Qwen3TTSSpeechTokenizer",
           "Qwen3TTSSpeechTokenizerDecoder", "Qwen3TTSSpeechTokenizerEncoder", "Qwen3TTSTalkerForConditionalGeneration"]
