from mlx_audio_b200.codec.models.vocos import Vocos, VocosBackbone  # noqa: F401
