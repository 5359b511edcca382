"""Qwen3-TTS in-context voice cloning on the GPU: the speech-tokenizer encoder (Mimi's encode chain with a full causal mask and half-split
RoPE), the in-context prompt, ``generate(text, ref_audio=..., ref_text=...)`` and the tensor-core causal GQA prefill attention, against the
float64 oracle at released sizes.

Tolerances: attention 2e-5 of the output's scale (fp16 hi / lo, 3 products, fp32 accumulate vs float64); encoder latent 2e-4 of max;
code streams identical except at fp32 near-ties of the nearest-code search (the rule of test_mimi_encode_matches_the_oracle); prompt
embeddings 2e-5 of max; talker logits 2e-4 of max; generated codes bit-exact on injected uniforms; audio 1e-3 of full scale."""
import os

import numpy as np
import pytest
import torch

from oracle import qwen3 as Q
from oracle import qwen3_stream as QS

pytestmark = pytest.mark.gpu

CFG_IDS = ("codec_nothink_id", "codec_think_id", "codec_think_bos_id", "codec_think_eos_id", "codec_pad_id", "codec_bos_id")


def _dev():
    return torch.device("cuda:0")


def rel_err(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


# ---------------------------------------------------------------------------------------------------------- prefill attention
def _attn_ref(q, kc, vc, Hq, Hkv, base, kv_start, scale):
    """float64 causal GQA attention of q [B,S,Hq*128] against cache rows [kv_start[b], base + s]."""
    B, S, _ = q.shape
    D, G = 128, Hq // Hkv
    out = torch.zeros(B, S, Hq * D, dtype=torch.float64)
    pos = base + torch.arange(S)
    for b in range(B):
        k0 = int(kv_start[b]) if kv_start is not None else 0
        keys = torch.arange(base + S)
        mask = (keys[None, :] <= pos[:, None]) & (keys[None, :] >= k0)
        for h in range(Hq):
            qh = q[b, :, h * D:(h + 1) * D].double()
            kh = kc[b, :base + S, (h // G) * D:(h // G + 1) * D].double()
            vh = vc[b, :base + S, (h // G) * D:(h // G + 1) * D].double()
            s = (qh @ kh.T) * scale
            s = s.masked_fill(~mask, float("-inf"))
            out[b, :, h * D:(h + 1) * D] = torch.softmax(s, dim=-1) @ vh
    return out.nan_to_num(0.0)            # a row before kv_start[b] sees no key: 0, as attn_decode returns


@pytest.mark.parametrize("B,S,base,kv_start,dev_base", [(1, 64, 0, None, False), (2, 200, 0, [0, 37], True), (1, 511, 130, None, True),
                                                         (2, 1000, 0, [5, 0], False), (1, 300, 77, [100], True)],
                         ids=["S64", "S200-B2-kvstart", "S511-base130", "S1000-B2", "S300-base77-kvstart"])
def test_prefill_attention_matches_float64(B, S, base, kv_start, dev_base):
    """Released talker shapes (Hq 16, Hkv 8, head_dim 128) against the fp32 cache; two runs bit-identical."""
    from mlx_audio_b200 import ops
    Hq, Hkv, D = 16, 8, 128
    g = torch.Generator().manual_seed(S + base)
    rows = -(-(base + S) // 256) * 256
    q = torch.randn(B, S, Hq * D, generator=g) * 1.5
    kc = torch.randn(B, rows, Hkv * D, generator=g)
    vc = torch.randn(B, rows, Hkv * D, generator=g)
    ks = None if kv_start is None else torch.tensor(kv_start, dtype=torch.int32)
    want = _attn_ref(q, kc, vc, Hq, Hkv, base, ks, D ** -0.5)
    dev = _dev()
    kw = dict(scale=D ** -0.5, kv_start=None if ks is None else ks.to(dev))
    if dev_base:
        kw.update(base_dev=torch.tensor([base], dtype=torch.int32, device=dev))
    else:
        kw.update(base=base)
    args = (q.to(dev), kc.to(dev), vc.to(dev), Hq, Hkv, D)
    got = ops.attn_prefill(*args, **kw)
    again = ops.attn_prefill(*args, **kw)
    assert torch.equal(got, again)
    assert float((got.cpu().double() - want).abs().max()) < 2e-5 * float(want.abs().max())


# ---------------------------------------------------------------------------------------------------------------- encoder
@pytest.fixture(scope="module")
def released_tokenizer():
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeechTokenizer, Qwen3TTSTokenizerConfig, Qwen3TTSTokenizerEncoderConfig
    P = synth.qwen3_tokenizer_weights(dict(Q.TOKENIZER_DECODER), seed=12, encoder=dict(Q.TOKENIZER_ENCODER))
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(encoder_config=Qwen3TTSTokenizerEncoderConfig()), _dev()).load_weights(P)
    assert st.has_encoder
    return st, {k: v.double() for k, v in P.items()}


@pytest.mark.parametrize("seconds", [3, 10])
def test_released_encoder_matches_oracle(released_tokenizer, seconds):
    st, P64 = released_tokenizer
    n = seconds * 24000
    audio = torch.as_tensor(0.3 * np.random.default_rng(seconds).standard_normal((1, 1, n)))
    from oracle import codec as OC
    cfg = dict(Q.TOKENIZER_ENCODER)
    root = "encoder_model."
    x = OC.mimi_seanet_encoder(P64, audio, cfg, root)
    x = OC.mimi_transformer(P64, root + "encoder_transformer", x, cfg, rope_traditional=False, full_causal=True)
    latent = OC.mimi_causal_conv(P64, root + "downsample.conv", x, 4, stride=2, pad_mode="edge")          # [B, C, T]
    want = OC.mimi_quantizer_encode(P64, latent, cfg, root)[:, :16]
    got_latent = st.encoder_model.encode_latent(audio.float())
    assert got_latent.shape[1] == -(-n // 1920) and rel_err(got_latent.transpose(1, 2), latent) < 2e-4
    got = st.encode(audio.float()).cpu()
    assert got.shape == want.shape == (1, 16, -(-n // 1920))
    # fp32 differences of the latent move some deep arg-mins (test_mimi_encode_matches_the_oracle's rule): the first books agree almost everywhere
    same = (got == want).float()
    assert float(same[:, :4].mean()) >= 0.9 and float(same.mean()) >= 0.6, (float(same[:, :4].mean()), float(same.mean()))


# ---------------------------------------------------------------------------------------------------------------- talker + ICL
def _model(n_layers, cp_layers, st):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Model, ModelConfig, Qwen3TTSTalkerCodePredictorConfig, Qwen3TTSTalkerConfig
    flat = dict(Q.TALKER, num_hidden_layers=n_layers, cp_num_hidden_layers=cp_layers)
    P = synth.qwen3_talker_weights(flat, seed=11)
    P.update(synth.qwen3_speaker_encoder_weights(dict(Q.SPEAKER_ENCODER)))        # the x-vector row of generate(ref_audio=..., ref_text=...)
    cp = Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=cp_layers)
    tc = Qwen3TTSTalkerConfig(code_predictor_config=cp, num_hidden_layers=n_layers, text_vocab_size=512, codec_eos_token_id=flat["codec_eos_token_id"])
    model = Model(ModelConfig(talker_config=tc, tts_model_type="base", tts_pad_token_id=500, tts_bos_token_id=501, tts_eos_token_id=502),
                  _dev()).load_weights(P)
    model.load_speech_tokenizer(st)
    return model, {k[len("talker."):]: v.double() for k, v in P.items() if k.startswith("talker.")}, flat


def _icl_case(model, Pt, seed, n_ref_frames, n_ref_text=20, n_text=30):
    g = torch.Generator().manual_seed(seed)
    target = [1, 3, 5] + torch.randint(10, 500, (n_text,), generator=g).tolist() + [2, 5, 1, 3, 5]
    ref = [1, 3, 5] + torch.randint(10, 500, (n_ref_text,), generator=g).tolist() + [2, 5]
    ref_codes = torch.randint(1, 2048, (1, 16, n_ref_frames), generator=g)
    spk = torch.randn(1, 1024, generator=g) * 0.05
    tc = model.config.talker_config
    want = Q.prepare_icl_generation_inputs_from_ids(Pt, target, ref, ref_codes, (501, 502, 500), {k: getattr(tc, k) for k in CFG_IDS},
                                                    language_id=2050, speaker_embed=spk.double())
    got = model.prepare_icl_generation_inputs_from_ids(target, ref, ref_codes, 2050, spk.to(_dev()))
    return target, ref, ref_codes, spk, want, got


@pytest.fixture(scope="module")
def small(released_tokenizer):
    return _model(3, 2, released_tokenizer[0])


def test_icl_prompt_matches_oracle(small):
    model, Pt, flat = small
    for seed, n_ref in ((1, 25), (2, 125)):
        _, _, _, _, want, got = _icl_case(model, Pt, seed, n_ref)
        # role 3, codec prefix 6 (language + speaker), transcript + target + eos 51, codec bos 1, one row per reference frame
        assert got[0].shape == want[0].shape == (1, 3 + 6 + 20 + 30 + 1 + 1 + n_ref, 1024)
        for a, b in zip(got, want):
            assert rel_err(a, b) < 2e-5


def test_icl_generate_and_stream_match_oracle(small, released_tokenizer):
    """ICL frame loop (repetition penalty 1.5, trailing text = pad) on a 3+2-layer talker with a 160-row prompt (the tensor-core prefill),
    joint [ref | generated] decode with the reference's share cut off, and the streamed events on the generated codes only."""
    model, Pt, flat = small
    _, PT = released_tokenizer
    target, ref, ref_codes, spk, want_in, got_in = _icl_case(model, Pt, 3, 100)
    u = torch.rand(6, 16, generator=torch.Generator().manual_seed(4))
    want = Q.generate_codes(Pt, *want_in, u.double(), 6, repetition_penalty=1.5, cfg=flat)
    res = list(model.generate_icl_from_ids(target, ref, ref_codes=ref_codes, speaker_embed=spk.to(_dev()), language_id=2050, max_tokens=6,
                                           u=u[:, :, None]))
    assert len(res) == 1 and res[0].token_count == want.shape[0] == 6 and res[0].segment_idx == 0
    wav = Q.decode_icl_generated_codes(PT, want, ref_codes)
    assert res[0].audio.shape == wav.shape and float((res[0].audio.cpu().double() - wav).abs().max()) < 1e-3
    events = list(model.generate_icl_from_ids(target, ref, ref_codes=ref_codes, speaker_embed=spk.to(_dev()), language_id=2050, max_tokens=6,
                                              u=u[:, :, None], stream=True, streaming_interval=0.32))
    ref_events = QS.stream_events(PT, want, 0.32)
    assert [e.token_count for e in events] == [e["token_count"] for e in ref_events]
    assert all(e.segment_idx == 0 for e in events) and events[-1].is_final_chunk
    got = torch.cat([e.audio for e in events]).cpu().double()
    assert float((got - QS.concat_audio(ref_events)).abs().max()) < 1e-3


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


def test_generate_icl_routing_and_cache(small):
    """generate(text, ref_audio, ref_text): one segment whatever the newlines; a repeated reference runs no encoder launch."""
    from mlx_audio_b200 import ops
    model, Pt, flat = small
    model.tokenizer = _CharTokenizer()
    model._icl_cache.clear()
    a = 0.3 * np.random.default_rng(7).standard_normal(2 * 24000).astype(np.float32)
    kw = dict(ref_audio=a, ref_text="the words of the reference", max_tokens=3, seed=5)
    l0 = ops.LAUNCHES[0]
    first = list(model.generate("Hello there.\nSecond line.", **kw))
    l1 = ops.LAUNCHES[0]
    second = list(model.generate("Hello there.\nSecond line.", **kw))
    l2 = ops.LAUNCHES[0]
    model.encode_reference(a)
    enc = ops.LAUNCHES[0] - l2
    assert [r.segment_idx for r in first] == [0] and len(second) == 1 and enc > 0
    assert (l1 - l0) - (l2 - l1) == enc and torch.equal(first[0].audio, second[0].audio)
    assert len(model._icl_cache) == 1
    streamed = list(model.generate("Hello there.\nSecond line.", stream=True, streaming_interval=0.08, **kw))
    assert all(e.segment_idx == 0 for e in streamed) and sum(e.token_count for e in streamed) == first[0].token_count


def test_full_size_talker_icl_prefill():
    """Full Qwen3-TTS-0.6B talker (28 + 5 layers) on a ~300-row ICL prompt: prefill logits within 2e-4 of the oracle, 3 frames of codes
    bit-exact on injected uniforms."""
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeechTokenizer, Qwen3TTSTokenizerConfig
    model, Pt, flat = _model(28, 5, Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), _dev()))
    _, _, _, _, want_in, got_in = _icl_case(model, Pt, 9, 240, n_ref_text=25, n_text=25)
    assert got_in[0].shape[1] >= 290 and rel_err(got_in[0], want_in[0]) < 2e-5
    u = torch.rand(3, 16, generator=torch.Generator().manual_seed(2))
    trace = []
    want = Q.generate_codes(Pt, *want_in, u.double(), 3, repetition_penalty=1.5, cfg=flat, trace=trace)
    codes = model.generate_codes(*got_in, max_tokens=3, u=u[:, :, None], repetition_penalty=1.5)
    assert torch.equal(codes[0].cpu(), want)
    model.talker.reset_cache(1, 512)
    lg, _ = model.talker(got_in[0])
    assert rel_err(lg[0, -1], trace[0]["logits"]) < 2e-4
