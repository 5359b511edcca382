"""Qwen3-TTS ``batch_generate`` on the GPU: in-context (ICL) cloning of several texts from one shared reference with per-row frame caps,
the batch stream (a chunk per row every interval), and the request routes -- against the float64 oracle with the cap and stream rules
of test_qwen3_batch_pins.py (which pins them to the reference's own batch_generate).

Tolerances: sampled codes bit-exact on injected uniforms; audio 1e-3 relative RMS against float64 (the rule of test_qwen3_session_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import qwen3 as Q
from test_qwen3_batch_pins import capped, stream_audio, stream_schedule       # tests/ is on sys.path (rootdir-relative "prepend" import mode)
from test_qwen3_icl_gpu import CFG_IDS, _CharTokenizer, _dev, _model, released_tokenizer   # noqa: F401  (module fixture)

pytestmark = pytest.mark.gpu


def rel_rms(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float(((a - b) ** 2).mean().sqrt() / ((b ** 2).mean().sqrt() + 1e-30))


@pytest.fixture(scope="module")
def small(released_tokenizer):
    return _model(3, 2, released_tokenizer[0])


def _case(model, Pt, seed=41, n_ref=30, n_texts=(24, 9, 16)):
    g = torch.Generator().manual_seed(seed)
    targets = [[1, 3, 5] + torch.randint(10, 500, (n,), generator=g).tolist() + [2, 5, 1, 3, 5] for n in n_texts]
    ref = [1, 3, 5] + torch.randint(10, 500, (12,), generator=g).tolist() + [2, 5]
    ref_codes = torch.randint(1, 2048, (1, 16, n_ref), generator=g)
    spk = torch.randn(1, 1024, generator=g) * 0.05
    tc = model.config.talker_config
    want_in = [Q.prepare_icl_generation_inputs_from_ids(Pt, t, ref, ref_codes, (501, 502, 500), {k: getattr(tc, k) for k in CFG_IDS},
                                                        language_id=2050, speaker_embed=spk.double()) for t in targets]
    return targets, ref, ref_codes, spk, want_in


class _Spy:
    """Records the generated codes handed to the joint decode and counts CUDA-graph captures."""
    def __init__(self, model, monkeypatch):
        self.codes, self.captures = [], 0
        real_decode, real_graph = model._decode_icl_batch, torch.cuda.CUDAGraph
        spy = self

        def decode(gen_list, ref_codes):
            spy.codes.append([c.cpu() for c in gen_list])
            return real_decode(gen_list, ref_codes)

        class Graph(real_graph):
            def __init__(self, *a, **k):
                spy.captures += 1
                super().__init__(*a, **k)
        monkeypatch.setattr(model, "_decode_icl_batch", decode)
        monkeypatch.setattr(torch.cuda, "CUDAGraph", Graph)


def test_icl_batch_matches_oracle_rows_alone_and_the_row_by_row_decode(small, released_tokenizer, monkeypatch):
    """Three texts, one reference: rows capped at 6 / 9 / 7 frames (max_tokens 9), the EOS id set so that one row stops on it.  Codes equal
    the oracle's batch loop with the cap rule and, row by row, generate_icl_from_ids run alone with that row's uniforms and max_tokens =
    its cap; audio is the oracle's joint decode; the batched joint decode equals the per-row one; one graph capture per call."""
    model, Pt, flat = small
    _, PT = released_tokenizer
    targets, ref, ref_codes, spk, want_in = _case(model, Pt)
    caps, max_tokens = [6, 9, 7], 9
    u = torch.rand(max_tokens, 16, 3, generator=torch.Generator().manual_seed(42))
    batch = lambda cfg: capped(Q.generate_codes_batch(Pt, [w[0] for w in want_in], [w[1] for w in want_in], want_in[0][2], u.double(),
                                                      max_tokens, repetition_penalty=1.5, cfg=cfg), caps)
    eos = int(batch(flat)[0][4, 0])                                  # row 0 samples this first code in its 5th frame
    tc = model.config.talker_config
    eos0, tc.codec_eos_token_id = tc.codec_eos_token_id, eos
    try:
        want = batch(dict(flat, codec_eos_token_id=eos))
        lengths = [int(w.shape[0]) for w in want]
        assert lengths[0] < caps[0] and any(n == c for n, c in zip(lengths, caps)), lengths
        spy = _Spy(model, monkeypatch)
        kw = dict(ref_codes=ref_codes, speaker_embed=spk.to(_dev()), language_id=2050, max_tokens=max_tokens)
        res = list(model.batch_generate_icl_from_ids(targets, ref, row_max_tokens=caps, u=u, **kw))
        assert spy.captures == 1
        assert [r.sequence_idx for r in res] == [b for b in range(3) if lengths[b] > 0]
        assert [r.token_count for r in res] == [n for n in lengths if n > 0]
        got = dict(zip([r.sequence_idx for r in res], spy.codes[0]))
        for r in res:
            b = r.sequence_idx
            assert torch.equal(got[b], want[b]), b
            wav = Q.decode_icl_generated_codes(PT, want[b], ref_codes)
            assert r.audio.shape == wav.shape and r.samples == wav.shape[0] and rel_rms(r.audio, wav) < 1e-3, b
        identical = True
        for r in res:
            b = r.sequence_idx
            alone = list(model.generate_icl_from_ids(targets[b], ref, u=u[:, :, b:b + 1].contiguous(), **dict(kw, max_tokens=caps[b])))
            assert torch.equal(spy.codes[-1][0], got[b]), b                       # the row alone generates the same codes, bit for bit
            per_row = alone[0].audio
            assert per_row.shape == r.audio.shape
            assert float((per_row - r.audio).abs().max()) < 1e-4, b               # batched joint decode = row-by-row decode
            identical &= torch.equal(per_row, r.audio)
        print("batched joint decode bit-identical to the row-by-row decode:", identical)
    finally:
        tc.codec_eos_token_id = eos0


def test_icl_batch_stream_follows_the_chunk_rule(small, released_tokenizer, monkeypatch):
    """stream=True with 3-frame chunks: the events (row order, token_count, flags) are the reference's emission rule on the oracle's codes,
    each chunk's audio the oracle's chunked decode behind its context; one graph capture."""
    model, Pt, flat = small
    _, PT = released_tokenizer
    targets, ref, ref_codes, spk, want_in = _case(model, Pt, seed=43)
    caps, max_tokens, interval = [8, 11, 5], 11, 0.24
    u = torch.rand(max_tokens, 16, 3, generator=torch.Generator().manual_seed(44))
    want = capped(Q.generate_codes_batch(Pt, [w[0] for w in want_in], [w[1] for w in want_in], want_in[0][2], u.double(), max_tokens,
                                         repetition_penalty=1.5, cfg=flat), caps)
    spy = _Spy(model, monkeypatch)
    events = list(model.batch_generate_icl_from_ids(targets, ref, ref_codes=ref_codes, speaker_embed=spk.to(_dev()), language_id=2050,
                                                    row_max_tokens=caps, max_tokens=max_tokens, u=u, stream=True, streaming_interval=interval))
    assert spy.captures == 1
    sched = stream_schedule([int(w.shape[0]) for w in want], caps, max_tokens, 3)
    assert [(e.sequence_idx, e.token_count, e.is_final_chunk) for e in events] == [(b, end - dec, f) for b, dec, end, f in sched]
    assert any(not f for *_, f in sched) and all(e.is_streaming_chunk for e in events)
    for e, a in zip(events, stream_audio(PT, want, sched, Q.TOKENIZER_DECODER)):
        assert e.audio.shape == a.shape and e.samples == a.shape[0] and rel_rms(e.audio, a) < 1e-3


def test_batch_generate_from_ids_streams_per_interval(small, released_tokenizer):
    """batch_generate_from_ids(stream=True) without a reference: 4-frame chunks of a 10-frame batch (clamp-pad trailing rule), the last
    chunk completed on the final frame emitted in the loop, as the reference does without caps."""
    model, Pt, flat = small
    _, PT = released_tokenizer
    tc = model.config.talker_config
    g = torch.Generator().manual_seed(45)
    ids_list = [torch.randint(0, 500, (n,), generator=g).tolist() for n in (12, 20)]
    rows = [Q.prepare_generation_inputs_from_ids(Pt, ids, (501, 502, 500), {k: getattr(tc, k) for k in CFG_IDS}, language_id=2050) for ids in ids_list]
    u = torch.rand(8, 16, 2, generator=g)
    want = Q.generate_codes_batch(Pt, [r[0] for r in rows], [r[1] for r in rows], rows[0][2], u.double(), 8, cfg=flat)
    events = list(model.batch_generate_from_ids(ids_list, language_id=2050, max_tokens=8, u=u, stream=True, streaming_interval=0.32))
    sched = stream_schedule([int(w.shape[0]) for w in want], None, 8, 4)
    assert [(e.sequence_idx, e.token_count, e.is_final_chunk) for e in events] == [(b, end - dec, f) for b, dec, end, f in sched]
    for e, a in zip(events, stream_audio(PT, want, sched, Q.TOKENIZER_DECODER)):
        assert e.audio.shape == a.shape and rel_rms(e.audio, a) < 1e-3


def test_batch_generate_routes(small, monkeypatch):
    """What supports_tts_batch accepts, batch_generate runs: a shared-reference ICL request (and its per-text list form) and a plain one;
    the text-level stream=False route without a reference is the continuous-batching session's output."""
    from mlx_audio_b200.tts.continuous import TTSBatchItem, TTSBatchOptions
    from mlx_audio_b200.tts.models.qwen3_tts import continuous_batching as CB
    model, Pt, flat = small
    model.tokenizer = _CharTokenizer()
    model._icl_cache.clear()
    a = torch.as_tensor(0.3 * np.random.default_rng(9).standard_normal(24000).astype(np.float32))
    texts = ["first text", "the second, longer text"]
    req = dict(ref_audio=a, ref_text="reference words")
    assert model.supports_tts_batch(**req) is True
    res = list(model.batch_generate(texts, max_tokens=2, **req))
    assert sorted(r.sequence_idx for r in res) == [0, 1] and all(0 < r.token_count <= 2 for r in res)
    res = list(model.batch_generate(texts, ref_audios=[a, a], ref_texts=[req["ref_text"]] * 2, max_tokens=2, stream=True, streaming_interval=0.08))
    assert res and all(r.is_streaming_chunk and r.token_count == 1 for r in res)
    assert len(model._icl_cache) == 1                                            # one encoder run for both calls
    with pytest.raises(ValueError, match="does not support voices"):
        next(model.batch_generate(texts, voices=["amy", None], max_tokens=2, **req))
    assert model.supports_tts_batch() is True
    init = CB.Qwen3TTSBatchSession.__init__

    def seeded(self, *a_, **k_):
        init(self, *a_, **k_)
        self._rng.manual_seed(7)
    monkeypatch.setattr(CB.Qwen3TTSBatchSession, "__init__", seeded)
    got = list(model.batch_generate(texts, max_tokens=5))
    session = model.create_tts_batch_session(TTSBatchOptions(max_tokens=5, max_batch_size=2))
    session.add([TTSBatchItem(sequence_id=i, text=t) for i, t in enumerate(texts)])
    want = []
    while not session.idle:
        want += [ev for ev in session.step() if ev.audio is not None and ev.samples > 0]
    assert [(r.sequence_idx, r.token_count, r.samples) for r in got] == [(e.sequence_id, e.token_count, e.samples) for e in want]
    assert all(torch.equal(r.audio, e.audio) for r, e in zip(got, want))
