from mlx_audio_b200.codec.models.dac import SUPPORTED_VERSIONS, DACFile  # noqa: F401
