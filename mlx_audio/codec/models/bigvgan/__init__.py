from mlx_audio_b200.codec.models.bigvgan import BigVGAN, BigVGANConfig  # noqa: F401
