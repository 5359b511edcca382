from mlx_audio_b200.tts.models.qwen3_tts.continuous_batching import *  # noqa: F401,F403
from mlx_audio_b200.tts.models.qwen3_tts.continuous_batching import Qwen3TTSBatchSession  # noqa: F401
