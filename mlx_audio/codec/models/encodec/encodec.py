from mlx_audio_b200.codec.models.encodec import Encodec, EncodecConfig, filter_dataclass_fields, preprocess_audio  # noqa: F401
