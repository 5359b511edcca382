from mlx_audio_b200.codec.models.encodec import Encodec, EncodecConfig, preprocess_audio  # noqa: F401
