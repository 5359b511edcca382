"""Incremental (streaming) Qwen3-TTS speech-tokenizer decoder and generate(stream=True) on the GPU, against the CPU oracle.

The oracle of a stream is ``oracle.qwen3.tokenizer_decode(..., stream_boundaries=...)``: the one-shot decode plus the reference's
overlap-add quirk (the transposed conv's bias counted twice over ``stride`` samples after every boundary), pinned to the reference's own
streaming code by tests/test_oracle_pins.py and tests/test_qwen3_stream_pins.py.  Waveform tolerance 1e-3 of full scale, as in
test_qwen3_gpu.py."""
import itertools

import pytest
import torch

from oracle import qwen3 as Q
from oracle import qwen3_stream as QS

pytestmark = pytest.mark.gpu

WTOL = 1e-3


def _dev():
    return torch.device("cuda:0")


def _tokenizer(seed=12):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeechTokenizer, Qwen3TTSTokenizerConfig
    flat = dict(Q.TOKENIZER_DECODER)
    P = synth.qwen3_tokenizer_weights(flat, seed=seed)
    st = Qwen3TTSSpeechTokenizer(Qwen3TTSTokenizerConfig(), _dev()).load_weights(P)
    return st, {k: v.double() for k, v in P.items()}, flat


@pytest.fixture(scope="module")
def tok():
    return _tokenizer()


def _stream(dec, codes, sizes):
    dec.reset_streaming_state()
    outs, s = [], 0
    for n in sizes:
        outs.append(dec.streaming_step(codes[:, :, s:s + n]))
        s += n
    return outs


def _boundaries(sizes):
    return tuple(itertools.accumulate(sizes))[:-1]


@pytest.mark.parametrize("B,sizes", [(1, [1] * 12), (1, [25, 25, 7]), (1, [3, 10, 1, 6]), (2, [4, 7])],
                         ids=["1-frame-chunks", "25+25+7", "3-10-1-6", "batch2"])
def test_streaming_step_matches_oracle(tok, B, sizes):
    """streaming_step over the chunks equals the oracle's incremental decode; 1-frame chunks keep more history than a call brings
    (block 0's dilation-9 unit: 54 rows of history, 32 new rows per frame)."""
    from mlx_audio_b200 import synth
    st, P64, flat = tok
    T = sum(sizes)
    codes = synth.qwen3_codes(flat, T, batch=B, seed=T + B)
    outs = _stream(st.decoder, codes.to(_dev()), sizes)
    assert [tuple(o.shape) for o in outs] == [(B, 1, 1920 * n) for n in sizes]
    got = torch.cat(outs, dim=-1)
    want = Q.tokenizer_decode(P64, codes, flat, stream_boundaries=_boundaries(sizes))
    assert float((got.cpu().double() - want).abs().max()) < WTOL
    assert float(got.abs().max()) <= 1.0


def test_single_chunk_equals_one_shot_and_quirk_is_visible(tok):
    """One streaming_step over a whole sequence is the one-shot decode; with 1-frame chunks the stream differs from it near every boundary
    by far more than the tolerance (the reproduced overlap-add quirk, not an absent one)."""
    from mlx_audio_b200 import synth
    st, _, flat = tok
    codes = synth.qwen3_codes(flat, 40, batch=1, seed=3).to(_dev())
    one = st.decoder(codes)
    (whole,) = _stream(st.decoder, codes, [40])
    assert float((whole - one).abs().max()) < 2e-6
    c12 = codes[:, :, :12]
    streamed = torch.cat(_stream(st.decoder, c12, [1] * 12), dim=-1)
    assert float((streamed - st.decoder(c12)).abs().max()) > 50 * WTOL


def test_kv_growth_is_exact(tok):
    """KV capacity grown in steps of 8 frames (device copies of the cached rows) gives the same bits as the default 256-frame step."""
    from mlx_audio_b200 import synth
    st, _, flat = tok
    dec = st.decoder
    codes = synth.qwen3_codes(flat, 20, batch=1, seed=5).to(_dev())
    sizes = [3] * 6 + [2]
    ref = _stream(dec, codes, sizes)
    dec.kv_step = 8
    try:
        got = _stream(dec, codes, sizes)
        assert dec._st["kv_cap"] == 24
    finally:
        del dec.kv_step
    for a, b in zip(got, ref):
        assert torch.equal(a, b)


def test_state_isolation(tok):
    """reset + replay repeats the chunks bit for bit; a one-shot decode between two steps leaves the stream untouched; a batch-size change
    within a stream and a wrong quantizer count raise."""
    from mlx_audio_b200 import synth
    st, _, flat = tok
    dec = st.decoder
    codes = synth.qwen3_codes(flat, 14, batch=1, seed=7).to(_dev())
    sizes = [5, 2, 7]
    first = _stream(dec, codes, sizes)
    second = _stream(dec, codes, sizes)
    assert all(torch.equal(a, b) for a, b in zip(first, second))
    dec.reset_streaming_state()
    a = dec.streaming_step(codes[:, :, :5])
    dec(synth.qwen3_codes(flat, 9, batch=2, seed=8).to(_dev()))
    dec.chunked_decode(codes, chunk_size=4, left_context_size=2)
    b = dec.streaming_step(codes[:, :, 5:7])
    c = dec.streaming_step(codes[:, :, 7:])
    assert torch.equal(a, first[0]) and torch.equal(b, first[1]) and torch.equal(c, first[2])
    with pytest.raises(ValueError, match="batch size"):
        dec.streaming_step(codes.expand(2, -1, -1)[:, :, :3])
    with pytest.raises(ValueError, match="Expected 16 layers of codes"):
        dec.streaming_step(codes[:, :8, :3])
    dec.reset_streaming_state()


def test_step_launches_and_no_torch_kernels(tok):
    """A step that does not grow the KV cache launches at most 5 kernels more than the one-shot decode of the same length (one carry,
    four overlap-adds), and runs no torch kernel except the int64 layout copy of a strided code slice."""
    from mlx_audio_b200 import ops, synth
    st, _, flat = tok
    dec = st.decoder
    codes = synth.qwen3_codes(flat, 75, batch=1, seed=9).to(_dev())
    ct = codes.transpose(1, 2).contiguous().transpose(1, 2)          # [1, 16, T] with the frame axis strided, as generate() passes it
    dec(codes[:, :, :25])
    l0 = ops.LAUNCHES[0]
    dec(codes[:, :, :25])
    one_shot = ops.LAUNCHES[0] - l0
    dec.reset_streaming_state()
    dec.streaming_step(ct[:, :, :25])
    l0 = ops.LAUNCHES[0]
    dec.streaming_step(ct[:, :, 25:50])
    step = ops.LAUNCHES[0] - l0
    assert one_shot < step <= one_shot + 5, (one_shot, step)
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        dec.streaming_step(ct[:, :, 50:75])
        torch.cuda.synchronize()
    dec.reset_streaming_state()
    kernels = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and not e.name.startswith(("Memcpy", "Memset"))]
    assert any("stream_rows" in k for k in kernels), kernels
    torch_kernels = [k for k in kernels if "at::" in k]
    assert len(torch_kernels) <= 1 and all("copy" in k for k in torch_kernels), torch_kernels


# ---------------------------------------------------------------------------------------------------------------- generate(stream=True)
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


@pytest.fixture(scope="module")
def model(tok):
    m, Pt, flat = _talker({"num_hidden_layers": 2, "cp_num_hidden_layers": 1})
    m.load_speech_tokenizer(tok[0])
    return m, Pt, flat


@pytest.mark.parametrize("max_tokens,interval,sizes", [(8, 0.32, [4, 4]), (7, 0.24, [3, 3, 1])], ids=["exact-multiple", "remainder"])
def test_generate_from_ids_stream_matches_oracle(model, tok, max_tokens, interval, sizes):
    """generate_from_ids(stream=True): the chunks' frames are generate_codes' frames (same uniforms); the events (sizes, token counts,
    flags) and their audio are the oracle's -- no final event when the frame count is a multiple of the chunk size."""
    m, Pt, flat = model
    _, P64, tflat = tok
    ids = torch.randint(0, 500, (12,), generator=torch.Generator().manual_seed(4)).tolist()
    u = torch.rand(max_tokens, 16, generator=torch.Generator().manual_seed(6))
    events = list(m.generate_from_ids(ids, max_tokens=max_tokens, u=u[:, :, None], stream=True, streaming_interval=interval))
    codes = m.generate_codes(*m.prepare_generation_inputs_from_ids(ids), max_tokens=max_tokens, u=u[:, :, None])[0].cpu()
    tc = m.config.talker_config
    cfg_ids = {k: getattr(tc, k) for k in ("codec_nothink_id", "codec_think_id", "codec_think_bos_id", "codec_think_eos_id", "codec_pad_id", "codec_bos_id")}
    ref_in = Q.prepare_generation_inputs_from_ids(Pt, ids, (501, 502, 500), cfg_ids)
    want = QS.generate_stream(Pt, P64, *ref_in, u.double(), max_tokens, interval, cfg=flat, tcfg=tflat)
    assert codes.shape[0] == max_tokens and torch.equal(torch.cat([e["codes"] for e in want]), codes)
    assert [e.token_count for e in events] == [e["token_count"] for e in want] == sizes
    assert [e.samples for e in events] == [e["samples"] for e in want] == [1920 * n for n in sizes]
    assert [e.is_final_chunk for e in events] == [e["is_final_chunk"] for e in want]
    assert all(e.is_streaming_chunk and e.segment_idx == 0 and e.audio.shape[0] == e.samples for e in events)
    assert [e.audio_samples.get("tokens") for e in events] == [s if not e["is_final_chunk"] else None
                                                              for s, e in zip(itertools.accumulate(sizes), want)]
    got = torch.cat([e.audio for e in events]).cpu().double()
    assert float((got - QS.concat_audio(want)).abs().max()) < WTOL


class _CharTokenizer:
    """Stands in for the HF tokenizer (as tests/golden/make_qwen3_golden.py's CharTokenizer): chat markers are single ids, every other
    character one id."""
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


def test_generate_stream_two_segments_reset_between(model):
    """Base generate(text, stream=True, seed=...) over two '\\n' segments: segment_idx 0 then 1, each segment's audio equal to a fresh
    stream of that segment's frames (the decoder state is reset between segments)."""
    m, _, _ = model
    m.tokenizer = _CharTokenizer()
    try:
        events = list(m.generate("Hello there.\nSecond line", stream=True, streaming_interval=0.16, max_tokens=5, seed=3))
        assert sorted({e.segment_idx for e in events}) == [0, 1] and [e.segment_idx for e in events] == sorted(e.segment_idx for e in events)
        dec = m.speech_tokenizer.decoder
        for idx, seg in enumerate(["Hello there.", "Second line"]):
            evs = [e for e in events if e.segment_idx == idx]
            assert [e.token_count for e in evs] == [2, 2, 1] and [e.is_final_chunk for e in evs] == [False, False, True]
            codes = m.generate_codes(*m._prepare_generation_inputs(seg), max_tokens=5, seed=3 + idx)
            fresh = _stream(dec, codes.transpose(1, 2), [2, 2, 1])
            for e, f in zip(evs, fresh):
                assert torch.equal(e.audio, f[0, 0])
    finally:
        m.tokenizer = None
