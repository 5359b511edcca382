from mlx_audio_b200.codec import DAC, DACFile, SNAC, Mimi, MimiConfig, MimiStreamingDecoder, mimi_202407, Vocos, Encodec  # noqa: F401
