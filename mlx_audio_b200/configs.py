"""Public configurations of the models on the hot path (data only), keyed the way this package's constructors take them.

Each dict restates the values the reference ships / tests with: Kokoro-82M (tts/tests/test_models.py:143-173), SNAC-24k
(codec/tests/test_snac.py:7-19), Mimi ``mimi_202407`` (codec/models/mimi/mimi.py:47-96), Whisper-small (the public
``openai/whisper-small`` geometry read through ``ModelDimensions.from_dict``, stt/models/whisper/whisper.py:292-322) and the
Qwen3-TTS-0.6B talker / speech-tokenizer decoder defaults (tts/models/qwen3_tts/config.py:32-133).  The benchmarks and tools
use these; ``tests/test_host_cpu.py`` asserts that the oracle's own copies say the same thing.
"""

KOKORO_82M = {
    "istftnet": {
        "upsample_kernel_sizes": [20, 12], "upsample_rates": [10, 6], "gen_istft_hop_size": 5,
        "gen_istft_n_fft": 20, "resblock_dilation_sizes": [[1, 3, 5], [1, 3, 5], [1, 3, 5]],
        "resblock_kernel_sizes": [3, 7, 11], "upsample_initial_channel": 512,
    },
    "dim_in": 64, "dropout": 0.2, "hidden_dim": 512, "max_conv_dim": 512, "max_dur": 50,
    "multispeaker": True, "n_layer": 3, "n_mels": 80, "n_token": 178, "style_dim": 128,
    "text_encoder_kernel_size": 5,
    "plbert": {"hidden_size": 768, "num_attention_heads": 12, "intermediate_size": 2048,
               "max_position_embeddings": 512, "num_hidden_layers": 12, "dropout": 0.1},
}

SNAC_24K = {
    "sampling_rate": 24000, "encoder_dim": 48, "encoder_rates": [2, 4, 8, 8], "decoder_dim": 1024,
    "decoder_rates": [8, 8, 4, 2], "attn_window_size": None, "codebook_size": 4096, "codebook_dim": 8,
    "vq_strides": [4, 2, 1], "noise": True, "depthwise": True,
}

MIMI_202407 = {
    "dimension": 512, "nfilters": 64, "ratios": [8, 6, 5, 4], "ksize": 7, "residual_ksize": 3, "last_ksize": 3,
    "compress": 2, "d_model": 512, "num_heads": 8, "num_layers": 8, "dim_feedforward": 2048, "context": 250,
    "max_period": 10000, "layer_scale": 0.01, "nq": 32, "bins": 2048, "qdim": 256, "upsample_stride": 2,
}

WHISPER_SMALL = {"n_mels": 80, "n_audio_ctx": 1500, "n_audio_state": 768, "n_audio_head": 12, "n_audio_layer": 12,
                 "n_vocab": 51865, "n_text_ctx": 448, "n_text_state": 768, "n_text_head": 12, "n_text_layer": 12}

QWEN3_TALKER = {
    "vocab_size": 3072, "hidden_size": 1024, "intermediate_size": 3072, "num_hidden_layers": 28, "num_attention_heads": 16,
    "num_key_value_heads": 8, "head_dim": 128, "rms_norm_eps": 1e-6, "rope_theta": 1000000.0, "mrope_section": [24, 20, 20],
    "num_code_groups": 16, "codec_eos_token_id": 2150, "text_hidden_size": 2048,
    "cp_vocab_size": 2048, "cp_hidden_size": 1024, "cp_intermediate_size": 3072, "cp_num_hidden_layers": 5,
    "cp_num_attention_heads": 16, "cp_num_key_value_heads": 8, "cp_head_dim": 128, "cp_rope_theta": 1000000.0,
}

QWEN3_TOKENIZER_DECODER = {
    "latent_dim": 1024, "codebook_dim": 512, "codebook_size": 2048, "decoder_dim": 1536, "hidden_size": 512,
    "intermediate_size": 1024, "layer_scale_initial_scale": 0.01, "head_dim": 64, "num_attention_heads": 16,
    "num_hidden_layers": 8, "num_key_value_heads": 16, "num_quantizers": 16, "num_semantic_quantizers": 1,
    "rms_norm_eps": 1e-5, "rope_theta": 10000.0, "upsample_rates": [8, 5, 4, 3], "upsampling_ratios": [2, 2],
}

QWEN3_TOKENIZER_ENCODER = {      # the speech-tokenizer encoder (ICL voice cloning) in Mimi's vocabulary: synth.qwen3_tokenizer_weights(encoder=)
    "dimension": 512, "nfilters": 64, "ratios": [8, 6, 5, 4], "ksize": 7, "residual_ksize": 3, "last_ksize": 3, "compress": 2, "d_model": 512,
    "num_heads": 8, "num_layers": 8, "dim_feedforward": 2048, "context": 250, "max_period": 10000, "layer_scale": 0.01, "nq": 32, "bins": 2048,
    "qdim": 256, "upsample_stride": 2, "valid_num_quantizers": 16,
}


# Vocos (codec/tests/test_vocos.py config_mel / config_encodec): the released 24 kHz mel checkpoint and the EnCodec-feature one, in the
# YAML shape Vocos.from_hparams takes.
VOCOS_MEL_24K = {
    "feature_extractor": {"class_path": "vocos.feature_extractors.MelSpectrogramFeatures",
                          "init_args": {"sample_rate": 24000, "n_fft": 1024, "hop_length": 256, "n_mels": 100}},
    "backbone": {"class_path": "vocos.models.VocosBackbone", "init_args": {"input_channels": 100, "dim": 512, "intermediate_dim": 1536, "num_layers": 8}},
    "head": {"class_path": "vocos.heads.ISTFTHead", "init_args": {"dim": 512, "n_fft": 1024, "hop_length": 256}},
}
VOCOS_ENCODEC_24K = {
    "feature_extractor": {"class_path": "vocos.feature_extractors.EncodecFeatures",
                          "init_args": {"encodec_model": "encodec_24khz", "bandwidths": [1.5, 3.0, 6.0, 12.0, 24.0]}},
    "backbone": {"class_path": "vocos.models.VocosBackbone",
                 "init_args": {"input_channels": 128, "dim": 384, "intermediate_dim": 1152, "num_layers": 8, "adanorm_num_embeddings": 4}},
    "head": {"class_path": "vocos.heads.ISTFTHead", "init_args": {"dim": 384, "n_fft": 1280, "hop_length": 320, "padding": "same"}},
}


# EnCodec (mlx-community/encodec-{24,48}khz-float32 config.json): 24 kHz mono, causal, weight norm; 48 kHz stereo, non-causal,
# time_group_norm, normalize, 1 s chunks with 1 % overlap.  Encodec(config) takes either dict.
ENCODEC_24K = dict(model_type="encodec", audio_channels=1, num_filters=32, kernel_size=7, num_residual_layers=1, dilation_growth_rate=2,
                   codebook_size=1024, codebook_dim=128, hidden_size=128, num_lstm_layers=2, residual_kernel_size=3, use_causal_conv=True,
                   normalize=False, pad_mode="reflect", norm_type="weight_norm", last_kernel_size=7, trim_right_ratio=1.0, compress=2,
                   upsampling_ratios=[8, 5, 4, 2], target_bandwidths=[1.5, 3.0, 6.0, 12.0, 24.0], sampling_rate=24000,
                   chunk_length_s=None, overlap=None)
ENCODEC_48K = dict(ENCODEC_24K, audio_channels=2, use_causal_conv=False, normalize=True, norm_type="time_group_norm",
                   target_bandwidths=[3.0, 6.0, 12.0, 24.0], sampling_rate=48000, chunk_length_s=1.0, overlap=0.01)
