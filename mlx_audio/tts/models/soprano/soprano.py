from mlx_audio_b200.tts.models.soprano.soprano import *  # noqa: F401,F403
from mlx_audio_b200.tts.models.soprano.soprano import DecoderConfig, Model, ModelConfig, SopranoDecoder, SopranoModel  # noqa: F401
