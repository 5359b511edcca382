from mlx_audio_b200.tts.continuous import *  # noqa: F401,F403
from mlx_audio_b200.tts.continuous import TTSBatchEvent, TTSBatchItem, TTSBatchOptions, TTSBatchSession  # noqa: F401
