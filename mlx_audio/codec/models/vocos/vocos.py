from mlx_audio_b200.codec.models.vocos import (EncodecFeatures, ISTFTHead, MelSpectrogramFeatures, Vocos, VocosBackbone,  # noqa: F401
                                               log_mel_spectrogram)
