"""Qwen3-TTS continuous batching on the GPU: the attention / cache kernels with per-row cache positions and a slot map, and the batch
session (``Model.create_tts_batch_session``) against the single-sequence oracle on a staggered schedule.

Tolerances: attention 2e-5 of the output's scale against float64 (fp32 CUDA-core kernels; fp16 hi / lo 3-product tensor-core prefill);
the per-row paths bit-identical to the scalar-base paths when every row shares one base; sampled codes bit-exact on injected uniforms;
audio 1e-3 relative RMS; full-size talker logits 2e-4 of max (the rule of test_qwen3_gpu.py)."""
import pytest
import torch

from oracle import qwen3 as Q
from oracle import qwen3_session as QS

pytestmark = pytest.mark.gpu

CFG_IDS = ("codec_nothink_id", "codec_think_id", "codec_think_bos_id", "codec_think_eos_id", "codec_pad_id", "codec_bos_id")


def _dev():
    return torch.device("cuda:0")


def rel_err(a, b):
    a, b = torch.as_tensor(a).detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


# ------------------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("D,Hq,Hkv,S", [(128, 16, 8, 1), (64, 4, 2, 1), (128, 4, 2, 5), (128, 4, 2, 96)], ids=["decode-d128", "decode-d64", "S5", "prefill-S96"])
def test_ragged_cache_kernels(D, Hq, Hkv, S):
    """qknorm_rope_cache + attn_decode / attn_prefill with ragged ``base_rows`` (one of them negative: a
    left-padding row) and a slot map with gaps, against float64 attention; padding positions write nothing and read zero; each
    kernel's output is bit-identical to the scalar-base path run on the same rows one at a time."""
    from mlx_audio_b200 import ops
    from test_lm_decode_matrix_gpu import cache_attn_ref   # tests/ is on sys.path (rootdir-relative "prepend" import mode)
    dev = _dev()
    g = torch.Generator().manual_seed(D + S)
    nslots, rows = 5, 320
    base_rows = torch.tensor([37, -3 if S > 1 else -1, 130], dtype=torch.int32) if S < 64 else torch.tensor([10, -40, 0], dtype=torch.int32)
    slot = torch.tensor([4, 0, 2], dtype=torch.int32)
    B = 3
    qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g)
    qn, kn = 1 + 0.1 * torch.randn(D, generator=g), 1 + 0.1 * torch.randn(D, generator=g)
    kc0 = torch.randn(nslots, rows, Hkv * D, generator=g)
    vc0 = torch.randn(nslots, rows, Hkv * D, generator=g)
    kc, vc = kc0.to(dev), vc0.to(dev)
    kw = dict(q_norm=qn.to(dev), k_norm=kn.to(dev), eps=1e-6, theta=1e6, mrope=(3 * D // 16, 3 * D // 16))
    br, sl = base_rows.to(dev), slot.to(dev)
    q = ops.qknorm_rope_cache(qkv.to(dev), Hq, Hkv, D, kc, vc, base_rows=br, slot=sl, **kw)
    # the same rows one at a time through the scalar-base path, on a copy of the cache
    kr, vr = kc0.clone().to(dev), vc0.clone().to(dev)
    for b in range(B):
        first = max(0, -int(base_rows[b]))                  # padding queries are dropped: the scalar path has no such rows
        if first >= S:
            continue
        qb = ops.qknorm_rope_cache(qkv[b:b + 1, first:].contiguous().to(dev), Hq, Hkv, D, kr[int(slot[b])][None], vr[int(slot[b])][None],
                                   base=int(base_rows[b]) + first, **kw)
        assert torch.equal(qb[0], q[b, first:]), b
    assert torch.equal(kr, kc) and torch.equal(vr, vc)         # identical rows written, nothing for padding, other slots untouched
    scale = D ** -0.5
    want = cache_attn_ref(q.cpu(), kc.cpu(), vc.cpu(), Hq, Hkv, D, base_rows, slot, None, rows, scale)
    attn = ops.attn_prefill if S >= 64 else ops.attn_decode
    if S >= 64 and (D != 128 or Hq != 2 * Hkv):
        pytest.skip("prefill kernel shape")
    got = attn(q, kc, vc, Hq, Hkv, D, scale=scale, base_rows=br, slot=sl)
    assert float((got.cpu().double() - want).abs().max()) < 2e-5 * float(want.abs().max())
    for b in range(B):                                         # padding rows read zero; live rows match the scalar-base path bit for bit
        first = max(0, -int(base_rows[b]))
        assert float(got[b, :first].abs().max()) == 0.0 if first else True
        if first >= S:
            continue
        one = attn(q[b:b + 1, first:].contiguous(), kc[int(slot[b])][None], vc[int(slot[b])][None], Hq, Hkv, D, scale=scale,
                   base=int(base_rows[b]) + first, max_k=rows)
        if attn is ops.attn_decode:
            assert torch.equal(one[0], got[b, first:]), b
        else:                                                  # other 64-row tiling of the queries: same math, same key order per row
            assert float((one[0] - got[b, first:]).abs().max()) < 2e-5 * float(want.abs().max()), b


@pytest.mark.parametrize("S", [1, 4, 70])
def test_shared_base_rows_match_the_scalar_base_bit_for_bit(S):
    """Every row at one base and an identity slot map: the per-row paths equal the device-scalar paths bit for bit."""
    from mlx_audio_b200 import ops
    dev = _dev()
    D, Hq, Hkv, B, base, rows = 128, 4, 2, 3, 45, 256
    g = torch.Generator().manual_seed(S)
    qkv = torch.randn(B, S, (Hq + 2 * Hkv) * D, generator=g).to(dev)
    kc0, vc0 = torch.randn(B, rows, Hkv * D, generator=g).to(dev), torch.randn(B, rows, Hkv * D, generator=g).to(dev)
    kw = dict(eps=1e-6, theta=1e6, mrope=(24, 20))
    base_dev = torch.tensor([base], dtype=torch.int32, device=dev)
    br = torch.full((B,), base, dtype=torch.int32, device=dev)
    sl = torch.arange(B, dtype=torch.int32, device=dev)
    outs = []
    for rows_kw in (dict(base_dev=base_dev), dict(base_rows=br, slot=sl)):
        kc, vc = kc0.clone(), vc0.clone()
        q = ops.qknorm_rope_cache(qkv, Hq, Hkv, D, kc, vc, **kw, **rows_kw)
        a = ops.attn_decode(q, kc, vc, Hq, Hkv, D, scale=D ** -0.5, **rows_kw)
        p = ops.attn_prefill(q, kc, vc, Hq, Hkv, D, scale=D ** -0.5, **rows_kw)
        outs.append((q, kc, vc, a, p))
    (q0, k0, v0, a0, p0), (q1, k1, v1, a1, p1) = outs
    assert torch.equal(q0, q1) and torch.equal(k0, k1) and torch.equal(v0, v1) and torch.equal(a0, a1) and torch.equal(p0, p1)


def test_slot_advance():
    """Live slots record their codes, advance length and frame count, finish at their cap and load the next uniforms; finished and
    empty slots are unchanged."""
    from mlx_audio_b200 import ops
    dev = _dev()
    B, G, F = 4, 3, 5
    lengths = torch.tensor([10, 20, 30, 40], dtype=torch.int32, device=dev)
    frames = torch.tensor([0, 3, 4, 2], dtype=torch.int32, device=dev)
    finished = torch.tensor([0, 0, 0, 1], dtype=torch.uint8, device=dev)
    cap = torch.tensor([5, 4, 5, 5], dtype=torch.int32, device=dev)
    codes = torch.arange(B * G, dtype=torch.int64, device=dev).view(B, G) + 1
    out = torch.zeros(B, F, G, dtype=torch.int64, device=dev)
    utab = torch.rand(B, F, G, device=dev)
    u = torch.full((G, B), -1.0, device=dev)
    ops.slot_advance(lengths, frames, finished, cap, codes, out, utab, u)
    assert lengths.tolist() == [11, 21, 31, 40] and frames.tolist() == [1, 4, 5, 2] and finished.tolist() == [0, 1, 1, 1]
    assert torch.equal(out[0, 0], codes[0]) and torch.equal(out[1, 3], codes[1]) and torch.equal(out[2, 4], codes[2])
    assert int(out[3].abs().sum()) == 0
    assert torch.equal(u[:, 0], utab[0, 1]) and float(u[:, 1:].max()) == -1.0


# ------------------------------------------------------------------------------------------------------------------- session
class _Tok:
    """Stands in for the HF tokenizer: the chat-template markers are single ids, every other character one id below 500."""
    MARK = {"<|im_start|>": 1, "<|im_end|>": 2, "assistant": 3, "user": 4, "\n": 5}

    def encode(self, text):
        ids, i = [], 0
        while i < len(text):
            for m, v in self.MARK.items():
                if text.startswith(m, i):
                    ids.append(v)
                    i += len(m)
                    break
            else:
                ids.append(10 + (ord(text[i]) * 7) % 480)
                i += 1
        return ids


def _model(over, with_tokenizer=True):
    from test_qwen3_gpu import _talker, _tokenizer          # tests/ is on sys.path (rootdir-relative "prepend" import mode)
    model, Pt, flat = _talker(over)
    if with_tokenizer:
        st, P64, tflat = _tokenizer()
        model.load_speech_tokenizer(st)
    else:
        P64 = tflat = None
    model.tokenizer = _Tok()
    return model, Pt, flat, P64, tflat


def _oracle_codes(model, Pt, flat, item, u, max_tokens):
    tc, tok = model.config.talker_config, model.tokenizer
    ids = tok.encode(f"<|im_start|>assistant\n{item.text}<|im_end|>\n<|im_start|>assistant\n")
    iid = tok.encode(f"<|im_start|>user\n{item.instruct}<|im_end|>\n") if item.instruct else None
    ie, tr, pad = Q.prepare_generation_inputs_from_ids(Pt, ids, (501, 502, 500), {k: getattr(tc, k) for k in CFG_IDS}, instruct_ids=iid)
    return Q.generate_codes(Pt, ie, tr, pad, u.double(), max_tokens, cfg=flat), ie.shape[1]


def _spy_decode(model):
    seen = []
    real = model._decode_generated_codes

    def spy(codes, **k):
        seen.append(codes.cpu().clone())
        return real(codes, **k)
    model._decode_generated_codes = spy
    return seen


def _run(session, script, n_steps=200):
    from mlx_audio_b200.tts.continuous import TTSBatchEvent
    events = []
    for step in range(n_steps):
        for kind, arg in script.get(step, []):
            session.add(arg) if kind == "add" else session.cancel(arg)
        if session.idle and step > max(script):
            break
        for e in session.step():
            assert isinstance(e, TTSBatchEvent) and e.done
            events.append((step, e))
    return events


def _items(texts, instructs, us, max_tokens=None):
    from mlx_audio_b200.tts.continuous import TTSBatchItem
    return [TTSBatchItem(sequence_id=i, text=t, instruct=ins, extra={"u": us[i]}) for i, (t, ins) in enumerate(zip(texts, instructs))]


TEXTS = ["Good morning, this is the first request.", "Short.", "A third sentence of middling size.", "Fourth.", "Fifth arrives late."]
INSTRUCTS = ["Speak slowly and warmly, like a radio host at night, calm.", None, "Bright and fast.", None, "Whisper it."]


@pytest.mark.parametrize("use_graph", [True, False])
def test_staggered_session_matches_the_oracle(use_graph):
    """max_batch_size 2, five requests of different prompt lengths (one of >= 64 rows: the tensor-core prefill), one added after the
    third step, one active row cancelled, rows ending on EOS and on max_tokens: events (step, id, token count) identical to the oracle's
    schedule, every finished row's codes bit-exact against the single-sequence loop, its audio within 1e-3 relative RMS."""
    from mlx_audio_b200.tts.continuous import TTSBatchOptions
    model, Pt, flat, P64, tflat = _model({"num_hidden_layers": 2, "cp_num_hidden_layers": 1})
    max_tokens = 12
    g = torch.Generator().manual_seed(41)
    us = [torch.rand(max_tokens, 16, generator=g) for _ in TEXTS]
    items = _items(TEXTS, INSTRUCTS, us)
    first, _ = _oracle_codes(model, Pt, flat, items[1], us[1], max_tokens)
    eos = int(first[6, 0])                                     # request 1 ends on EOS at its 7th frame
    flat = dict(flat, codec_eos_token_id=eos)
    model.config.talker_config.codec_eos_token_id = eos
    codes, plen = {}, {}
    for it in items:
        codes[it.sequence_id], plen[it.sequence_id] = _oracle_codes(model, Pt, flat, it, us[it.sequence_id], max_tokens)
    assert max(plen.values()) >= 64 and len(set(plen.values())) >= 3
    assert codes[1].shape[0] <= 6 and any(c.shape[0] == max_tokens for k, c in codes.items() if k != 0)
    script = {0: [("add", [0, 1, 2, 3])], 3: [("add", [4])], 5: [("cancel", 0)]}
    want, cancelled = QS.run_schedule(codes, {k: [(kd, a if kd == "cancel" else list(a)) for kd, a in v] for k, v in script.items()}, 2, max_tokens)
    assert cancelled == {0: 5}
    session = model.create_tts_batch_session(TTSBatchOptions(max_tokens=max_tokens, max_batch_size=2))
    session._use_graph = use_graph
    seen = _spy_decode(model)
    by_id = {it.sequence_id: it for it in items}
    got = _run(session, {k: [(kd, [by_id[i] for i in a] if kd == "add" else a) for kd, a in v] for k, v in script.items()})
    assert [(s, e.sequence_id, e.token_count) for s, e in got] == want
    assert session.idle and session.captures == (1 if use_graph else 0)
    for (s, e), c in zip(got, seen):
        assert torch.equal(c, codes[e.sequence_id]), e.sequence_id
        ref = Q.decode_generated_codes(P64, codes[e.sequence_id], tflat)
        assert e.samples == e.audio.shape[0] == c.shape[0] * 1920 and e.sample_rate == 24000
        assert float(((e.audio.cpu().double() - ref) ** 2).mean().sqrt() / (ref ** 2).mean().sqrt()) < 1e-3


def test_session_all_up_front_equals_batch_generate():
    """Every item added before the first step: the same codes as batch_generate_from_ids(stream=False) with the same uniforms."""
    from mlx_audio_b200.tts.continuous import TTSBatchItem, TTSBatchOptions
    model, Pt, flat, _, _ = _model({"num_hidden_layers": 2, "cp_num_hidden_layers": 1})
    g = torch.Generator().manual_seed(5)
    ids_list = [torch.randint(10, 500, (n,), generator=g).tolist() for n in (12, 30, 17)]
    n_frames = 9
    u = torch.rand(n_frames, 16, 3, generator=g)
    x, trailing, pad, left = model.prepare_batch_inputs_from_ids(ids_list)        # batch_generate_from_ids(stream=False)'s loop
    codes, lengths = model.generate_codes(x, trailing, pad, max_tokens=n_frames, u=u, left_padding=left, batch_mode=True, trailing_rule="standard")
    want = {b: codes[b, : int(lengths[b])].cpu() for b in range(3)}
    seen = _spy_decode(model)

    class _Ids:                                                # the item's text is a key into the prepared ids
        def encode(self, text):
            key = text.split("\n")[1].split("<|im_end|>")[0]
            return ids_list[int(key)]
    model.tokenizer = _Ids()
    session = model.create_tts_batch_session(TTSBatchOptions(max_tokens=n_frames, max_batch_size=3))
    session.add([TTSBatchItem(sequence_id=b, text=str(b), extra={"u": u[:, :, b]}) for b in range(3)])
    events = _run(session, {0: []})
    assert sorted(e.sequence_id for _, e in events) == [0, 1, 2]
    for (_, e), c in zip(events, seen):
        assert torch.equal(c, want[e.sequence_id]), e.sequence_id


def test_session_graph_is_captured_once_and_cache_grows():
    """One capture for a session whose rows come and go; a prompt longer than the cache grows it mid-session (re-allocate, copy the
    live rows, capture again) and every row stays bit-exact against the oracle."""
    from mlx_audio_b200.tts.continuous import TTSBatchItem, TTSBatchOptions
    model, Pt, flat, _, _ = _model({"num_hidden_layers": 2, "cp_num_hidden_layers": 1})
    max_tokens = 8
    g = torch.Generator().manual_seed(77)
    texts = ["one", "two two", "three three three", "a long prompt"]
    instructs = [None, None, None, "x" * 250]                   # ~262 prompt rows: past the first cache (9 + 8 + 1 -> 256 rows)
    us = [torch.rand(max_tokens, 16, generator=g) for _ in texts]
    items = [TTSBatchItem(sequence_id=i, text=t, instruct=ins, extra={"u": us[i]}) for i, (t, ins) in enumerate(zip(texts, instructs))]
    codes = {it.sequence_id: _oracle_codes(model, Pt, flat, it, us[it.sequence_id], max_tokens)[0] for it in items}
    session = model.create_tts_batch_session(TTSBatchOptions(max_tokens=max_tokens, max_batch_size=3))
    seen = _spy_decode(model)
    script = {0: [("add", items[:2])], 2: [("add", [items[2]])], 4: [("add", [items[3]])]}
    got = _run(session, script)
    assert sorted(e.sequence_id for _, e in got) == [0, 1, 2, 3]
    for (_, e), c in zip(got, seen):
        assert torch.equal(c, codes[e.sequence_id]), e.sequence_id
    assert session._rows == 512 and session.captures == 2


def test_full_size_talker_eight_slots():
    """Released 28 + 5-layer talker, 8 slots of different prompt lengths, 3 frames: the talker logits of frame 1 at the ragged cache
    lengths within 2e-4 of the oracle's, and the codes bit-exact (first and last slot)."""
    from mlx_audio_b200.tts.continuous import TTSBatchItem, TTSBatchOptions
    model, Pt, flat, _, _ = _model({})
    max_tokens = 3
    g = torch.Generator().manual_seed(3)
    items = [TTSBatchItem(sequence_id=i, text="w" * (3 + 5 * i), instruct="calm " * i if i % 2 else None,
                          extra={"u": torch.rand(max_tokens, 16, generator=g)}) for i in range(8)]
    session = model.create_tts_batch_session(TTSBatchOptions(max_tokens=max_tokens, max_batch_size=8))
    seen = _spy_decode(model)
    session.add(items)
    assert session.step() == []
    st = session._st
    with session._use_caches():
        lg, _ = model.talker(st._x_in, base_rows=st._base_rows.clone())
    events = _run(session, {0: []})
    assert [e.sequence_id for _, e in events] == list(range(8))
    for i in (0, 7):
        trace = []
        tc = model.config.talker_config
        tok = model.tokenizer
        ids = tok.encode(f"<|im_start|>assistant\n{items[i].text}<|im_end|>\n<|im_start|>assistant\n")
        iid = tok.encode(f"<|im_start|>user\n{items[i].instruct}<|im_end|>\n") if items[i].instruct else None
        ie, tr, pad = Q.prepare_generation_inputs_from_ids(Pt, ids, (501, 502, 500), {k: getattr(tc, k) for k in CFG_IDS}, instruct_ids=iid)
        want = Q.generate_codes(Pt, ie, tr, pad, items[i].extra["u"].double(), max_tokens, cfg=flat, trace=trace)
        assert torch.equal(seen[i], want), i
        assert rel_err(lg[i, -1], trace[1]["logits"]) < 2e-4, i


def test_hooks_and_empty_sessions():
    """supports_tts_batch / supports_tts_continuous_batch follow the reference's truth table; max_tokens <= 0 gives empty events."""
    from mlx_audio_b200.tts.continuous import TTSBatchItem, TTSBatchOptions
    model, _, _, _, _ = _model({"num_hidden_layers": 1, "cp_num_hidden_layers": 1})
    assert model.supports_tts_batch() and model.supports_tts_continuous_batch()
    assert not model.supports_tts_batch(stream=True) and not model.supports_tts_batch(speed=1.5) and not model.supports_tts_batch(instruct="x")
    assert not model.supports_tts_continuous_batch(ref_audio=[0.0], ref_text="hi")
    session = model.create_tts_batch_session(TTSBatchOptions(max_tokens=0, max_batch_size=2))
    session.add([TTSBatchItem(sequence_id=i, text="hi") for i in range(3)])
    ev = session.step()
    assert [(e.sequence_id, e.samples, e.token_count, e.done) for e in ev] == [(0, 0, 0, True), (1, 0, 0, True)]
    assert [e.sequence_id for e in session.step()] == [2] and session.idle
