from mlx_audio_b200.tts.models.soprano.decoder import ISTFTHead, SopranoDecoder  # noqa: F401
