from mlx_audio_b200.codec.models.vocos import log_mel_spectrogram  # noqa: F401
