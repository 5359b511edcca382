from mlx_audio_b200.tts.models.qwen3_tts.speaker_encoder import *  # noqa: F401,F403
