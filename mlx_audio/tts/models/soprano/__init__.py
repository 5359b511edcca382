from mlx_audio_b200.tts.models.soprano import *  # noqa: F401,F403
from mlx_audio_b200.tts.models.soprano import DecoderConfig, Model, ModelConfig, clean_text  # noqa: F401
