"""Qwen3-TTS hot path on the GPU vs the CPU oracle (SURVEY.md section 8 rows a15-a18).

Tolerances: logits / hidden states 2e-4 of the tensor's max (fp32 GEMV / bf16x2 tensor-core products vs float64); sampled
codes and token ids bit-exact (integer work, same injected uniforms); vocoder waveform 1e-3 of full scale (north_star)."""
import math

import pytest
import torch

from oracle import nn as ON
from oracle import qwen3 as Q

pytestmark = pytest.mark.gpu


def rel_err(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _dev():
    return torch.device("cuda:0")


def _bf(x):
    return x.to(torch.bfloat16).float()


@pytest.mark.parametrize("M,K,N,norm,swiglu,res", [(1, 1024, 4096, True, False, False), (2, 1024, 6144, True, True, False),
                                                    (3, 2048, 1024, False, False, True), (8, 3072, 1024, False, False, True),
                                                    (11, 1024, 3072, True, False, False), (5, 64, 36, False, True, True)])
def test_gemv(M, K, N, norm, swiglu, res):
    from mlx_audio_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(0)
    x = torch.randn(M, K, generator=g)
    w = _bf(torch.randn(N, K, generator=g) / math.sqrt(K))
    nw = 1 + 0.1 * torch.randn(K, generator=g)
    r = torch.randn(M, N // 2 if swiglu else N, generator=g)
    xd = x.double()
    if norm:
        xd = ON.rms_norm(xd, nw.double(), 1e-6)
    y = xd @ w.double().T
    if swiglu:
        y = torch.nn.functional.silu(y[:, 0::2]) * y[:, 1::2]
    if res:
        y = y + r.double()
    if N % 32:
        cw = ops.ConvW(w.t().contiguous().to(dev)[None], None, 1, K, N, 1)
        cw.w_tc, cw.cin_pad = w.to(torch.bfloat16).to(dev).contiguous()[None], K
    else:
        cw = ops.pack_linear(w, None, dev)
    out = ops.gemv(x.to(dev), cw, norm_w=nw.to(dev) if norm else None, norm_eps=1e-6, swiglu=swiglu, res=r.to(dev) if res else None)
    assert rel_err(out, y) < 2e-5


@pytest.mark.parametrize("temperature,top_k,top_p,min_p,rep", [(0.9, 50, 1.0, 0.0, 1.05), (0.7, 20, 0.8, 0.0, 1.3), (1.0, 0, 0.9, 0.05, 1.0),
                                                                (0.0, 50, 1.0, 0.0, 1.05), (1.2, 3000, 1.0, 0.1, 1.1)])
def test_sampler_matches_oracle(temperature, top_k, top_p, min_p, rep):
    """b2a_sample_token vs Model._sample_token restated (oracle/qwen3.py:sample_token): same token, same filtered logits."""
    from mlx_audio_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(3)
    B, V = 6, 3072
    logits = torch.randn(B, V, generator=g) * 2.5
    u = torch.rand(B, generator=g)
    suppress = [i for i in range(V - 1024, V) if i != 2150]
    mask = torch.zeros(V)
    mask[suppress] = float("-inf")
    seen_lists = [torch.randint(0, 2048, (40,), generator=g).tolist() for _ in range(B)]
    seen = torch.zeros(B, V, dtype=torch.uint8)
    for b, l in enumerate(seen_lists):
        seen[b, l] = 1
    tok, filt = ops.sample_token(logits.to(dev), temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p, u=u.to(dev),
                                 suppress_mask=mask.to(dev), seen=seen.to(dev), repetition_penalty=rep, return_filtered=True)
    for b in range(B):
        t_ref, f_ref = Q.sample_token(logits[b], float(u[b]), temperature, top_k, top_p, rep, seen_lists[b], suppress, min_p, return_filtered=True)
        assert int(tok[b]) == t_ref
        if temperature > 0:
            assert torch.equal(filt[b].cpu(), f_ref)                     # the scaled logits (logits / temperature) or -inf


def _talker(cfg_over, seed=11):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Model, ModelConfig, Qwen3TTSTalkerConfig, Qwen3TTSTalkerCodePredictorConfig
    flat = dict(Q.TALKER)
    flat.update(cfg_over)
    P = synth.qwen3_talker_weights(flat, seed=seed)
    cp = Qwen3TTSTalkerCodePredictorConfig(num_hidden_layers=flat["cp_num_hidden_layers"])
    tc = Qwen3TTSTalkerConfig(code_predictor_config=cp, num_hidden_layers=flat["num_hidden_layers"], text_vocab_size=512,
                              codec_eos_token_id=flat["codec_eos_token_id"])
    mc = ModelConfig(talker_config=tc, tts_pad_token_id=500, tts_bos_token_id=501, tts_eos_token_id=502)
    model = Model(mc, _dev()).load_weights(P)
    Pt = {k[len("talker."):]: v.double() for k, v in P.items()}
    return model, Pt, flat


def test_talker_prefill_and_steps_match_oracle():
    """Talker stack: prefill of 21 rows (tensor-core path), then 3 single-row steps (GEMV path) against the concat-cache oracle;
    also an explicit 3-axis MRoPE position tensor (talker.py:186-226)."""
    model, Pt, flat = _talker({"num_hidden_layers": 3, "cp_num_hidden_layers": 1})
    t = model.talker
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 21, 1024, generator=g)
    cache = Q.make_cache(3)
    lo, ho = Q.talker_forward(Pt, x.double(), cache, cfg=flat)
    t.reset_cache(2, 64)
    lg, hg = t(x.to(_dev()))
    assert rel_err(lg, lo) < 2e-4 and rel_err(hg, ho) < 2e-4
    for s in range(3):
        xs = torch.randn(2, 1, 1024, generator=g)
        lo, ho = Q.talker_forward(Pt, xs.double(), cache, cfg=flat)
        lg, hg = t(xs.to(_dev()), use_device_offset=bool(s % 2))
        assert rel_err(lg, lo) < 2e-4 and rel_err(hg, ho) < 2e-4
    pos3 = torch.stack([torch.arange(5), torch.arange(5) * 2 + 1, torch.arange(5) * 3 + 2])[:, None, :].expand(3, 2, 5).contiguous()
    x5 = torch.randn(2, 5, 1024, generator=g)
    lo, _ = Q.talker_forward(Pt, x5.double(), Q.make_cache(3), position_ids=pos3, cfg=flat)
    t.reset_cache(2, 16)
    lg, _ = t(x5.to(_dev()), position_ids=pos3)
    assert rel_err(lg, lo) < 2e-4


def _prompt(model, Pt, seed=5, n_text=14):
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, 500, (n_text,), generator=g).tolist()
    tc = model.config.talker_config
    cfg_ids = {k: getattr(tc, k) for k in ("codec_nothink_id", "codec_think_id", "codec_think_bos_id", "codec_think_eos_id", "codec_pad_id", "codec_bos_id")}
    ref = Q.prepare_generation_inputs_from_ids(Pt, ids, (501, 502, 500), cfg_ids, language_id=2050, speaker_id=2100)
    got = model.prepare_generation_inputs_from_ids(ids, language_id=2050, speaker_id=2100)
    return ids, ref, got


@pytest.mark.parametrize("use_graph", [True, False])
def test_generate_codes_small_model_bit_exact(use_graph):
    """Frame loop (qwen3_tts.py:1323-1404) on a 3+2-layer model: prompt assembly, 8 frames x 16 codebooks, injected uniforms:
    every sampled code equals the oracle's; then EOS handling with the EOS id set to frame 4's first code."""
    model, Pt, flat = _talker({"num_hidden_layers": 3, "cp_num_hidden_layers": 2})
    ids, ref, got = _prompt(model, Pt)
    for a, b in zip(got, ref):
        assert a.shape == b.shape and rel_err(a, b) < 2e-5
    g = torch.Generator().manual_seed(9)
    u = torch.rand(8, 16, generator=g)
    want = Q.generate_codes(Pt, *ref, u.double(), 8, cfg=flat)
    codes = model.generate_codes(*got, max_tokens=8, u=u[:, :, None], use_graph=use_graph)
    assert codes.shape == (1, 8, 16) and torch.equal(codes[0].cpu(), want)
    eos = int(want[4, 0])
    flat2 = dict(flat, codec_eos_token_id=eos)
    model.config.talker_config.codec_eos_token_id = eos
    want2 = Q.generate_codes(Pt, *ref, u.double(), 8, cfg=flat2)
    codes2 = model.generate_codes(*got, max_tokens=8, u=u[:, :, None], use_graph=use_graph)
    assert want2.shape[0] < 8 and torch.equal(codes2[0].cpu(), want2)


def test_generate_codes_full_size_talker():
    """Full Qwen3-TTS-0.6B shapes (28 + 5 layers): 3 frames, codes bit-exact, talker logits within 2e-4."""
    model, Pt, flat = _talker({})
    ids, ref, got = _prompt(model, Pt, n_text=12)
    u = torch.rand(3, 16, generator=torch.Generator().manual_seed(2))
    trace = []
    want = Q.generate_codes(Pt, *ref, u.double(), 3, cfg=flat, trace=trace)
    codes = model.generate_codes(*got, max_tokens=3, u=u[:, :, None])
    assert torch.equal(codes[0].cpu(), want)
    model.talker.reset_cache(1, 64)
    lg, _ = model.talker(got[0])
    assert rel_err(lg[0, -1], trace[0]["logits"]) < 2e-4


def _tokenizer(seed=12):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeechTokenizer, Qwen3TTSTokenizerConfig
    flat = dict(Q.TOKENIZER_DECODER)
    P = synth.qwen3_tokenizer_weights(flat, seed=seed)
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), _dev()).load_weights(P)
    return st, {k: v.double() for k, v in P.items()}, flat


def test_speech_tokenizer_decoder_matches_oracle():
    """Qwen3TTSSpeechTokenizerDecoder.__call__ (speech_tokenizer.py:843-880): 1920 samples per frame, waveform within 1e-3."""
    from mlx_audio_b200 import synth
    st, P64, flat = _tokenizer()
    codes = synth.qwen3_codes(flat, 40, batch=2)
    taps_o, taps_g = {}, {}
    want = Q.tokenizer_decode(P64, codes, flat, taps_o)
    got = st.decoder(codes, taps_g)
    assert got.shape == (2, 1, 40 * 1920)
    for k in taps_o:
        assert rel_err(taps_g[k], taps_o[k]) < 5e-4, k
    assert float((got.cpu().double() - want).abs().max()) < 1e-3
    with pytest.raises(ValueError, match="Expected 16 layers of codes"):
        st.decoder(codes[:, :8])


def test_speech_tokenizer_chunked_and_public_decode():
    """chunked_decode / decode / batch_decode / streaming_decode (speech_tokenizer.py:932-954,1099-1217) vs the oracle's
    sequential chunk loop (batched equal-length chunks must give the same samples)."""
    from mlx_audio_b200 import synth
    st, P64, flat = _tokenizer()
    codes = synth.qwen3_codes(flat, 37, batch=1)
    want = Q.chunked_decode(P64, codes, chunk_size=12, left_context_size=4, cfg=flat)
    got = st.decoder.chunked_decode(codes, chunk_size=12, left_context_size=4)
    assert got.shape == want.shape == (1, 1, 37 * 1920)
    assert float((got.cpu().double() - want).abs().max()) < 1e-3
    ac = codes.transpose(1, 2).clone()
    ac[0, -3:, 0] = 0                                                   # three padded frames -> valid length 34 frames
    wav, lengths = st.decode(ac)
    assert wav.shape == (1, 37 * 1920) and int(lengths[0]) == 34 * 1920
    audios, lens = st.batch_decode([ac[0, :20], ac[0, :9]])
    assert [a.shape[0] for a in audios] == [20 * 1920, 9 * 1920] and lens == [20 * 1920, 9 * 1920]
    w20 = Q.tokenizer_decode(P64, ac[:, :20].transpose(1, 2), flat)[0, 0]
    assert float((audios[0].cpu().double() - w20).abs().max()) < 1e-3
    chunks = list(st.streaming_decode(ac[:, :20], chunk_tokens=8))
    assert [c.shape[-1] for c in chunks] == [8 * 1920, 8 * 1920, 4 * 1920]


def test_generate_from_ids_end_to_end():
    """Model.generate contract (tts/models/base.py:71-87): one GenerationResult with 1920 samples per generated frame."""
    model, Pt, flat = _talker({"num_hidden_layers": 2, "cp_num_hidden_layers": 1})
    st, _, _ = _tokenizer()
    model.load_speech_tokenizer(st)
    ids = torch.randint(0, 500, (12,), generator=torch.Generator().manual_seed(4)).tolist()
    res = list(model.generate_from_ids(ids, max_tokens=5, seed=1))
    assert len(res) == 1
    r = res[0]
    assert r.sample_rate == 24000 and r.token_count == 5 and r.samples == r.audio.shape[0] == 5 * 1920
    assert float(r.audio.abs().max()) <= 1.0
    with pytest.raises(ValueError, match="Tokenizer not loaded"):
        next(model.generate("hello"))


@pytest.mark.parametrize("use_graph", [True, False])
def test_batch_generate_codes_left_padded_bit_exact(use_graph):
    """batch_generate's loop (qwen3_tts.py:1861-1935) with prompts of different lengths: left padding + key masking + cumsum positions,
    right-padded trailing text with the clamp-pad rule, a row that hits EOS early is frozen at EOS and stops advancing its text."""
    model, Pt, flat = _talker({"num_hidden_layers": 3, "cp_num_hidden_layers": 2})
    tc = model.config.talker_config
    cfg_ids = {k: getattr(tc, k) for k in ("codec_nothink_id", "codec_think_id", "codec_think_bos_id", "codec_think_eos_id", "codec_pad_id", "codec_bos_id")}
    g = torch.Generator().manual_seed(21)
    ids_list = [torch.randint(0, 500, (n,), generator=g).tolist() for n in (15, 11, 13)]
    spk, ins = [2100, None, None], [None, None, [7, 8, 9, 10, 11]]          # a speaker row (+1) and an instruct row (+5): three prefill lengths
    refs = [Q.prepare_generation_inputs_from_ids(Pt, ids, (501, 502, 500), cfg_ids, language_id=2050, speaker_id=spk[i], instruct_ids=ins[i])
            for i, ids in enumerate(ids_list)]
    x, trailing, pad, left = model.prepare_batch_inputs_from_ids(ids_list, language_id=2050, speaker_ids=spk, instruct_ids=ins)
    assert left == [4, 5, 0] and x.shape[0] == 3 and float(x[1, :5].abs().max()) == 0.0
    u = torch.rand(9, 16, 3, generator=g)
    want = Q.generate_codes_batch(Pt, [r[0] for r in refs], [r[1] for r in refs], refs[0][2], u.double(), 9, cfg=flat)
    codes, lengths = model.generate_codes(x, trailing, pad, max_tokens=9, u=u, left_padding=left, batch_mode=True, use_graph=use_graph)
    assert lengths.tolist() == [w.shape[0] for w in want] == [9, 9, 9]
    for b in range(3):
        assert torch.equal(codes[b, : int(lengths[b])].cpu(), want[b]), b
    # EOS for row 1 at its 4th frame: it stops there, the others run on
    eos = int(want[1][3, 0])
    flat2 = dict(flat, codec_eos_token_id=eos)
    tc.codec_eos_token_id = eos
    want2 = Q.generate_codes_batch(Pt, [r[0] for r in refs], [r[1] for r in refs], refs[0][2], u.double(), 9, cfg=flat2)
    codes2, lengths2 = model.generate_codes(x, trailing, pad, max_tokens=9, u=u, left_padding=left, batch_mode=True, use_graph=use_graph)
    assert lengths2.tolist() == [w.shape[0] for w in want2] and want2[1].shape[0] <= 3
    for b in range(3):
        assert torch.equal(codes2[b, : int(lengths2[b])].cpu(), want2[b]), b
        assert int(codes2[b, int(lengths2[b]):].abs().sum()) == 0


def test_batch_generate_from_ids_results():
    """BatchGenerationResult contract (tts/models/base.py:89-99): one result per sequence, 1920 samples per generated frame."""
    model, Pt, flat = _talker({"num_hidden_layers": 2, "cp_num_hidden_layers": 1})
    st, _, _ = _tokenizer()
    model.load_speech_tokenizer(st)
    g = torch.Generator().manual_seed(8)
    ids_list = [torch.randint(0, 500, (n,), generator=g).tolist() for n in (12, 16)]
    res = list(model.batch_generate_from_ids(ids_list, max_tokens=4, seed=3))
    assert [r.sequence_idx for r in res] == [0, 1]
    for r in res:
        assert r.sample_rate == 24000 and r.token_count == 4 and r.samples == r.audio.shape[0] == 4 * 1920
        assert not r.is_streaming_chunk and not r.is_final_chunk         # the default path's events carry neither flag (continuous_batching.py:326-344)
    res = list(model.batch_generate_from_ids(ids_list, max_tokens=4, seed=3, stream=True))
    assert [r.sequence_idx for r in res] == [0, 1] and all(r.is_streaming_chunk and r.is_final_chunk and r.samples == 4 * 1920 for r in res)
