"""Qwen3-TTS x-vector voice cloning on the GPU: the 24 kHz log-mel front end, the ECAPA-TDNN speaker encoder (csrc/speaker.cu + the
tensor-core conv) and ``generate(ref_audio=...)``, against the CPU oracle and the reference's own outputs (qwen3_golden.npz).

Tolerances: log-mel 2e-4 absolute; embeddings 2e-4 of the tensor's max (fp32 / bf16x2 tensor-core products vs float64); generated
codes bit-exact on the prompt built from the product's own embedding (fp32 near-ties of the sampler stay out of the comparison);
streamed audio 1e-3 of full scale, as in test_qwen3_stream_gpu.py."""
import json
import os
import sys

import numpy as np
import pytest
import torch

from oracle import dsp as D
from oracle import qwen3 as Q
from oracle import qwen3_stream as QS
from oracle import qwen3_xvector as QX

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
RELEASED = dict(Q.SPEAKER_ENCODER)


def _dev():
    return torch.device("cuda:0")


def rel_err(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _golden():
    return np.load(os.path.join(HERE, "golden", "qwen3_golden.npz"))


def _encoder(cfg, P, sanitize=True):
    """Product encoder loaded from a prefixed MLX-layout dict: through the reference's sanitize, or (``sanitize=False``: test-size
    channels, where its [out, in, K] shape heuristic does not apply) with the prefix stripped only."""
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeakerEncoderConfig
    from mlx_audio_b200.tts.models.qwen3_tts.speaker_encoder import Qwen3TTSSpeakerEncoder
    enc = Qwen3TTSSpeakerEncoder(Qwen3TTSSpeakerEncoderConfig(**cfg), _dev())
    if not sanitize:
        return enc.load_weights({k[len("speaker_encoder."):]: v for k, v in P.items()})
    return enc.load_weights(Qwen3TTSSpeakerEncoder.sanitize(P))


@pytest.fixture(scope="module")
def fixture_encoder():
    sys.path.insert(0, os.path.join(HERE, "golden"))
    import synth_params
    g = _golden()
    scfg = json.loads(str(g["spk_cfg"]))
    PS = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g["spk_params"]).items()}
    return _encoder(scfg, {k: v.float() for k, v in PS.items()}, sanitize=False), PS, scfg, g


@pytest.fixture(scope="module")
def released():
    from mlx_audio_b200 import synth
    P = synth.qwen3_speaker_encoder_weights(RELEASED)
    return _encoder(RELEASED, P), {k: v.double() for k, v in P.items()}


# ---------------------------------------------------------------------------------------------------------------- front end
@pytest.mark.parametrize("B", [1, 2])
def test_logmel_matches_oracle_10s(B):
    from mlx_audio_b200.tts.models.qwen3_tts.qwen3_tts import mel_spectrogram
    rng = np.random.default_rng(20 + B)
    t = np.arange(240000) / 24000
    audio = 0.2 * rng.standard_normal((B, 240000)) + 0.3 * np.sin(2 * np.pi * 220 * t)
    got = mel_spectrogram(audio.astype(np.float32), device=_dev())
    want = D.qwen3_mel_spectrogram(audio.astype(np.float32))
    assert tuple(got.shape) == want.shape == (B, 937, 128)
    assert float(np.abs(got.cpu().numpy() - want).max()) < 2e-4
    one = mel_spectrogram(audio[0].astype(np.float32), device=_dev())            # [n] -> [1, frames, 128]
    assert tuple(one.shape) == (1, 937, 128) and torch.equal(one[0], got[0])


def test_logmel_matches_reference_output(fixture_encoder):
    from mlx_audio_b200.tts.models.qwen3_tts.qwen3_tts import mel_spectrogram
    g = fixture_encoder[3]
    audio = 0.3 * np.random.default_rng(135).standard_normal((2, 9000))
    got = mel_spectrogram(audio, device=_dev())
    assert float(np.abs(got.cpu().numpy() - g["spk_mel"]).max()) < 2e-4
    with pytest.raises(ValueError, match="384"):
        mel_spectrogram(np.zeros(300), device=_dev())


# ---------------------------------------------------------------------------------------------------------------- encoder
def test_fixture_encoder_matches_reference(fixture_encoder):
    """Test-size config (32 channels, scale 4: 8-channel Res2Net chunks, CUDA-core fallbacks) on the reference's own mel and embedding,
    and the whole extract_speaker_embedding on the ICL seeds' audio (24 mel frames: below the tensor-core row minimum)."""
    from mlx_audio_b200.tts.models.qwen3_tts import Model, ModelConfig
    enc, PS, scfg, g = fixture_encoder
    emb = enc(torch.as_tensor(g["spk_mel"]).float().to(_dev()))
    assert emb.shape == (2, 64) and rel_err(emb, g["spk_embedding"]) < 2e-4
    model = Model(ModelConfig(speaker_encoder_config=scfg), _dev())
    model.speaker_encoder = enc
    for tag, seed in (("a", 46), ("b", 48)):
        ref_audio = 0.3 * np.random.default_rng(seed).standard_normal(3 * 1920 + 500)
        e = model.extract_speaker_embedding(ref_audio)
        assert e.shape == (1, 64) and rel_err(e, g[f"icl_{tag}_speaker_embed"]) < 2e-4, tag
    with pytest.raises(ValueError, match="24kHz"):
        model.extract_speaker_embedding(ref_audio, sr=16000)


@pytest.mark.parametrize("B,T", [(1, 281), (1, 937), (2, 203)], ids=["3s", "10s", "B2-odd-length"])
def test_released_size_encoder_matches_oracle(released, B, T):
    """512 / 1536 channels, scale 8 (64-channel chunks), enc_dim 1024, bf16-exact weights: float64 oracle within 2e-4 of max."""
    enc, P64 = released
    mel = torch.randn(B, T, 128, generator=torch.Generator().manual_seed(T)) * 2 - 4
    want = Q.speaker_encoder(P64, mel.double(), RELEASED)
    got = enc(mel.to(_dev()))
    assert got.shape == (B, 1024) and rel_err(got, want) < 2e-4


def test_encoder_rejects_too_short_mel(released):
    enc, _ = released
    with pytest.raises(ValueError, match="too few"):
        enc(torch.zeros(1, 4, 128, device=_dev()))
    assert enc.min_frames() == 5
    enc(torch.zeros(1, 5, 128, device=_dev()))                           # the shortest the reference's reflect pads accept


def _chain_oracle(y, w, b, scale, d):
    """Res2NetBlock (speaker_encoder.py:86-101) in float64: y [B, T, scale*C], w [scale-1, K, in, out]."""
    C = y.shape[2] // scale
    K = w.shape[1]
    pad = (K - 1) * d // 2
    outs, prev = [y[:, :, :C]], None
    for j in range(1, scale):
        x = y[:, :, j * C:(j + 1) * C] + (prev if j > 1 else 0)
        xp = torch.cat([x[:, 1:pad + 1].flip(1), x, x[:, -(pad + 1):-1].flip(1)], dim=1)
        acc = b[j - 1].expand(x.shape[0], x.shape[1], C).clone()
        for k in range(K):
            acc = acc + xp[:, k * d: k * d + x.shape[1]] @ w[j - 1, k]
        prev = torch.relu(acc)
        outs.append(prev)
    return torch.cat(outs, dim=2)


@pytest.mark.parametrize("C,scale", [(64, 8), (8, 4)])
@pytest.mark.parametrize("d", [2, 3, 4])
def test_res2net_chain_kernel(C, scale, d):
    """The one-launch Res2Net chain at every dilation of the released config, at the shortest T the reflect pads allow and at T spanning
    several 32-row tiles, on a channel-slice view input."""
    from mlx_audio_b200 import ops
    g = torch.Generator().manual_seed(C + d)
    w = torch.randn(scale - 1, 3, C, C, generator=g) / (3 * C) ** 0.5
    b = torch.randn(scale - 1, C, generator=g) * 0.1
    for T in (d + 1, 150):
        big = torch.randn(2, T, scale * C + 16, generator=g)
        y = big[:, :, 8:8 + scale * C]
        want = _chain_oracle(y.double(), w.double(), b.double(), scale, d)
        got = ops.spk_res2net(big.to(_dev())[:, :, 8:8 + scale * C], w.to(_dev()).contiguous(), b.to(_dev()).contiguous(), scale, d)
        assert rel_err(got, want) < 2e-5, (T, d)
    with pytest.raises(ValueError):
        ops.spk_res2net(torch.zeros(1, d, scale * C, device=_dev()), w.to(_dev()).contiguous(), b.to(_dev()).contiguous(), scale, d)


def test_pooling_kernel_is_safe_with_shifted_logits():
    """Softmax over 30 s of frames (2813) with every logit shifted by +80: max-subtracted, finite, equal to the unshifted float64 result."""
    from mlx_audio_b200 import ops
    g = torch.Generator().manual_seed(8)
    T, C = 2813, 1536
    x = torch.randn(1, T, C, generator=g)
    lg = torch.randn(1, T, C, generator=g) * 3
    a = torch.softmax(lg.double(), dim=1)
    mean = (a * x.double()).sum(1)
    std = torch.sqrt(torch.clamp((a * (x.double() - mean[:, None]) ** 2).sum(1), min=1e-12))
    got = ops.spk_asp_pool((lg + 80).to(_dev()), x.to(_dev()))
    assert bool(torch.isfinite(got).all())
    assert rel_err(got[:, :C], mean) < 2e-5 and rel_err(got[:, C:], std) < 2e-5


def test_embedding_is_deterministic(released):
    enc, _ = released
    mel = torch.randn(1, 700, 128, generator=torch.Generator().manual_seed(2)).to(_dev())
    assert torch.equal(enc(mel), enc(mel))


def test_launch_budget_and_no_torch_kernels_in_a_complete_trace(released):
    """One extract_speaker_embedding at B = 1 (3 s of audio): at most 40 launches, and no torch kernel (the samples' host -> device copy
    is a memcpy).  Every trace the profiler returns is checked for torch kernels.  In a long process it occasionally returns the
    activity records of earlier work instead of this call's, so a trace without the call's three Res2Net kernels is taken again
    (up to three times); a pass that stops launching them fails every attempt."""
    from mlx_audio_b200 import ops
    from mlx_audio_b200.tts.models.qwen3_tts import Model, ModelConfig
    enc, _ = released
    model = Model(ModelConfig(speaker_encoder_config=RELEASED), _dev())
    model.speaker_encoder = enc
    audio = (0.3 * np.random.default_rng(3).standard_normal(72000)).astype(np.float32)
    model.extract_speaker_embedding(audio)
    torch.cuda.synchronize()
    traces = []
    for _ in range(3):
        l0 = ops.LAUNCHES[0]
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            model.extract_speaker_embedding(audio)
            torch.cuda.synchronize()
        n = ops.LAUNCHES[0] - l0
        assert n <= 40, n
        kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
        assert not [k for k in kernels if "at::" in k], kernels
        traces.append(kernels)
        if sum("spk_res2net" in k for k in kernels) == 3:
            break
    assert sum("spk_res2net" in k for k in traces[-1]) == 3, traces


# ---------------------------------------------------------------------------------------------------------------- generation
def _tokenizer(seed=12):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeechTokenizer, Qwen3TTSTokenizerConfig
    flat = dict(Q.TOKENIZER_DECODER)
    P = synth.qwen3_tokenizer_weights(flat, seed=seed)
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), _dev()).load_weights(P)
    return st, {k: v.double() for k, v in P.items()}, flat


def _base_model(dtype=torch.float32, seed=11):
    """Base model: 2 + 1-layer talker at hidden 1024, released-size speaker encoder, test speech tokenizer."""
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Model, ModelConfig, Qwen3TTSTalkerConfig, Qwen3TTSTalkerCodePredictorConfig
    flat = dict(Q.TALKER, num_hidden_layers=2, cp_num_hidden_layers=1)
    P = synth.qwen3_talker_weights(flat, seed=seed)
    P.update(synth.qwen3_speaker_encoder_weights(RELEASED))
    cp = Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=1)
    tc = Qwen3TTSTalkerConfig(code_predictor_config=cp, num_hidden_layers=2, text_vocab_size=512, codec_eos_token_id=flat["codec_eos_token_id"],
                              spk_id={"amy": 2100})
    mc = ModelConfig(talker_config=tc, speaker_encoder_config=RELEASED, tts_pad_token_id=500, tts_bos_token_id=501, tts_eos_token_id=502)
    model = Model(mc, _dev()).load_weights({k: v.to(dtype) for k, v in P.items()})
    Pt = {k[len("talker."):]: v.double() for k, v in P.items() if k.startswith("talker.")}
    return model, Pt, flat


@pytest.fixture(scope="module")
def base():
    model, Pt, flat = _base_model()
    st, P64, tflat = _tokenizer()
    model.load_speech_tokenizer(st)
    return model, Pt, flat, P64, tflat


def _cfg_ids(model):
    tc = model.config.talker_config
    return {k: getattr(tc, k) for k in ("codec_nothink_id", "codec_think_id", "codec_think_bos_id", "codec_think_eos_id", "codec_pad_id", "codec_bos_id")}


def _ref_audio(seed=30, seconds=2.0):
    return (0.3 * np.random.default_rng(seed).standard_normal(int(24000 * seconds))).astype(np.float32)


def test_generate_from_ids_ref_audio_bit_exact(base):
    """generate_from_ids(ref_audio=a) == generate_from_ids(speaker_embed=<the product's embedding of a>), and both equal the oracle's codes
    on the oracle prompt built from that same embedding."""
    model, Pt, flat, P64, tflat = base
    a = _ref_audio()
    ids = torch.randint(0, 500, (12,), generator=torch.Generator().manual_seed(4)).tolist()
    u = torch.rand(8, 16, generator=torch.Generator().manual_seed(6))
    emb = model.extract_speaker_embedding(a)
    assert emb.shape == (1, 1024)
    r1 = list(model.generate_from_ids(ids, ref_audio=a, u=u[:, :, None], max_tokens=8))
    r2 = list(model.generate_from_ids(ids, speaker_embed=emb, u=u[:, :, None], max_tokens=8))
    assert len(r1) == len(r2) == 1 and r1[0].token_count == r2[0].token_count and torch.equal(r1[0].audio, r2[0].audio)
    got_in = model.prepare_generation_inputs_from_ids(ids, speaker_embed=emb)
    ref_in = QX.prepare_generation_inputs_from_embed(Pt, ids, (501, 502, 500), _cfg_ids(model), speaker_embed=emb.cpu())
    for x, y in zip(got_in, ref_in):
        assert x.shape == y.shape and rel_err(x, y) < 2e-5
    codes = model.generate_codes(*got_in, max_tokens=8, u=u[:, :, None])[0].cpu()
    want = Q.generate_codes(Pt, *ref_in, u.double(), 8, cfg=flat)
    assert torch.equal(codes, want) and codes.shape[0] == r1[0].token_count


def test_bf16_talker_rounds_the_embedding():
    """With a bf16 talker checkpoint the x-vector enters the prefix as bf16(embedding) (qwen3_tts.py:429-432)."""
    model, _, _ = _base_model(torch.bfloat16)
    assert model.talker_dtype == torch.bfloat16
    emb = model.extract_speaker_embedding(_ref_audio(31))
    ids = list(range(20, 34))
    got = model.prepare_generation_inputs_from_ids(ids, speaker_embed=emb)[0]
    bf = model.prepare_generation_inputs_from_ids(ids, speaker_embed=emb.to(torch.bfloat16).float())[0]
    assert torch.equal(got, bf)
    model.talker_dtype = torch.float32
    raw = model.prepare_generation_inputs_from_ids(ids, speaker_embed=emb)[0]
    assert not torch.equal(raw, bf)
    # speaker row = combined row 3 (nothink, think_bos, think_eos, SPEAKER): tts_pad + embedding
    pad = model.prepare_generation_inputs_from_ids(ids)[2]
    assert float((got[0, 6] - pad[0, 0] - emb[0].to(torch.bfloat16).float()).abs().max()) < 1e-5


@pytest.mark.parametrize("max_tokens,interval", [(7, 0.24)])
def test_stream_with_ref_audio_matches_oracle(base, max_tokens, interval):
    model, Pt, flat, P64, tflat = base
    a = _ref_audio(32)
    ids = torch.randint(0, 500, (12,), generator=torch.Generator().manual_seed(5)).tolist()
    u = torch.rand(max_tokens, 16, generator=torch.Generator().manual_seed(7))
    events = list(model.generate_from_ids(ids, ref_audio=a, max_tokens=max_tokens, u=u[:, :, None], stream=True, streaming_interval=interval))
    emb = model.extract_speaker_embedding(a)
    ref_in = QX.prepare_generation_inputs_from_embed(Pt, ids, (501, 502, 500), _cfg_ids(model), speaker_embed=emb.cpu())
    want = QS.generate_stream(Pt, P64, *ref_in, u.double(), max_tokens, interval, cfg=flat, tcfg=tflat)
    assert [e.token_count for e in events] == [e["token_count"] for e in want]
    assert [e.is_final_chunk for e in events] == [e["is_final_chunk"] for e in want]
    got = torch.cat([e.audio for e in events]).cpu().double()
    assert float((got - QS.concat_audio(want)).abs().max()) < 1e-3


class _CharTokenizer:
    MARK = {"<|im_start|>": 1, "<|im_end|>": 2, "assistant": 3, "user": 4, "\n": 5}

    def encode(self, text):
        ids, i = [], 0
        while i < len(text):
            for mk, v in self.MARK.items():
                if text.startswith(mk, i):
                    ids.append(v)
                    i += len(mk)
                    break
            else:
                ids.append(10 + (ord(text[i]) % 100))
                i += 1
        return ids


def test_generate_routing(base):
    """ref_audio on a base model: x-vector route on every segment (it wins over a preset voice); ref_audio + ref_text: x-vector when the
    speech tokenizer has no encoder, NotImplementedError (ICL) when it has one."""
    model, Pt, flat, P64, tflat = base
    model.tokenizer = _CharTokenizer()
    a = _ref_audio(33)
    emb = model.extract_speaker_embedding(a)
    kw = dict(max_tokens=4, seed=3)
    xv = list(model.generate("Hi there.\nSecond.", ref_audio=a, **kw))
    assert [r.segment_idx for r in xv] == [0, 1]
    with_voice = list(model.generate("Hi there.\nSecond.", ref_audio=a, voice="amy", **kw))
    assert all(torch.equal(p.audio, q.audio) for p, q in zip(xv, with_voice))
    model.speech_tokenizer_has_encoder = False
    with_text = list(model.generate("Hi there.\nSecond.", ref_audio=a, ref_text="words", **kw))
    assert all(torch.equal(p.audio, q.audio) for p, q in zip(xv, with_text))
    # segment 0 equals generate_from_ids on the same ids with the embedding pinned (seed + segment index)
    ids0 = QX.segment_ids(_CharTokenizer().encode, "Hi there.\nSecond.")[0]
    pinned = list(model.generate_from_ids(ids0, speaker_embed=emb, **kw))
    assert torch.equal(pinned[0].audio, xv[0].audio)
    plain = list(model.generate("Hi there.\nSecond.", **kw))
    assert not torch.equal(plain[0].audio, xv[0].audio) or plain[0].token_count != xv[0].token_count
    model.speech_tokenizer_has_encoder = True
    try:
        with pytest.raises(NotImplementedError, match="ICL"):
            next(model.generate("Hi.", ref_audio=a, ref_text="words"))
    finally:
        model.speech_tokenizer_has_encoder = False
    with pytest.raises(ValueError, match="24kHz"):
        model.extract_speaker_embedding(a, sr=16000)
