"""Mimi's incremental decode_step / encode_step on the GPU (mimi_stream.cu) at the released size with synthetic weights: the streams
against the float64 oracle's one-shot slices (oracle/mimi_stream.py, pinned to the reference's own step functions) and against the
product's one-shot decode / encode.  The kernels themselves are tested in test_stream_kernels_matrix_gpu.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import ops, synth
from oracle import codec as OC
from oracle import mimi_stream as MS

DEV = "cuda:0"


def rel_rms(a, b):
    a, b = torch.as_tensor(a).double().cpu().reshape(-1), torch.as_tensor(b).double().cpu().reshape(-1)
    return float(torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean()))


@pytest.fixture(scope="module")
def mimi():
    from mlx_audio_b200.codec import Mimi, mimi_202407
    P = synth.mimi_weights(OC.MIMI_202407, encoder=True)
    return Mimi(mimi_202407(32), device=DEV).load_weights(P), {k: v.double() for k, v in P.items()}


# ------------------------------------------------------------------------------------------------------------------------- decode
def _run(model, codes, chunks):
    model.reset_state()
    a, outs, mem = 0, [], {}
    for c in chunks:
        outs.append(model.decode_step(codes[:, :, a:a + c]).cpu())
        a += c
        mem[a] = torch.cuda.memory_allocated()
    return outs, mem


def _uneven(T):
    base, out = [1, 3, 7, 1, 25, 2, 12, 1, 40], []
    while sum(out) < T:
        out.append(min(base[len(out) % len(base)], T - sum(out)))
    return out


@pytest.fixture(scope="module")
def stream200(mimi):
    model, P64 = mimi
    codes = synth.mimi_codes(OC.MIMI_202407, 200, 2)
    return codes, OC.mimi_decode(P64, codes), model.decode(codes).cpu()


@pytest.mark.parametrize("kind", ["frames", "uneven"])
def test_decode_step_stream_matches_the_oracle_and_decode(mimi, stream200, kind):
    """200 frames at B = 2 = 400 transformer positions: the ring wraps.  Every chunk within 1e-3 of the float64 one-shot slice; the stream
    within 1e-4 of the product's one-shot decode; memory flat once the stream is running."""
    model, _ = mimi
    codes, ref, one_shot = stream200
    chunks = [1] * 200 if kind == "frames" else _uneven(200)
    outs, mem = _run(model, codes, chunks)
    a = 0
    for c, o in zip(chunks, outs):
        assert o.shape == (2, 1, 1920 * c)
        assert rel_rms(o, ref[..., a * 1920:(a + c) * 1920]) < 1e-3, (a, c)
        a += c
    assert rel_rms(torch.cat(outs, -1), one_shot) < 1e-4
    if kind == "frames":
        assert mem[10] == mem[200], (mem[10], mem[200])


def test_graph_replay_is_bit_identical_to_eager(mimi):
    from mlx_audio_b200.codec.models import mimi as MM
    model, _ = mimi
    codes = synth.mimi_codes(OC.MIMI_202407, 30, 2)
    try:
        MM.GRAPH_SINGLE_FRAME[0] = False
        eager, _ = _run(model, codes, [1] * 30)
    finally:
        MM.GRAPH_SINGLE_FRAME[0] = True
    graph, _ = _run(model, codes, [1] * 30)
    assert model._dec_state.graphs, "single-frame steps did not replay a graph"
    assert torch.equal(torch.cat(eager, -1), torch.cat(graph, -1))


def test_reset_decode_restart_and_batch_change(mimi):
    model, _ = mimi
    codes = synth.mimi_codes(OC.MIMI_202407, 8, 2)
    first, _ = _run(model, codes, [3, 5])
    model.decode_step(codes[:, :, :2])
    with pytest.raises(ValueError):
        model.decode_step(codes[:1, :, :1])
    model.decode(codes)                                                 # decode() restarts the stream, B may change
    again = [model.decode_step(codes[:, :, :3]).cpu(), model.decode_step(codes[:, :, 3:]).cpu()]
    assert torch.equal(torch.cat(first, -1), torch.cat(again, -1))
    model.reset_state()
    y1 = model.decode_step(codes[:1, :, :4]).cpu()                      # a new stream at B = 1
    assert rel_rms(y1, model.decode(codes[:1, :, :4]).cpu()) < 1e-4


def test_streaming_decoder_wrapper_is_unchanged(mimi, stream200):
    from mlx_audio_b200.codec.models.mimi import MimiStreamingDecoder
    model, _ = mimi
    codes, _, one_shot = stream200
    dec = MimiStreamingDecoder(model)
    outs = [dec.decode_frames(codes[:, :, a:a + c]) for a, c in ((0, 4), (4, 1), (5, 11))]
    assert rel_rms(torch.cat([o.cpu() for o in outs], -1), one_shot[..., :16 * 1920]) < 1e-4
    dec.reset()
    y = dec.decode_frames(codes[0, :, :4])                              # [C, T] form: a new stream at B = 1
    assert y.shape == (1, 1, 4 * 1920) and rel_rms(y, model.decode(codes[:1, :, :4])) < 1e-4


# ------------------------------------------------------------------------------------------------------------------------- encode
@pytest.mark.parametrize("chunks", [[1920] * 6, [2500, 2500, 4600, 3400, 6200, 300], [700, 1920, 1220, 5000, 3180]])
def test_encode_step_matches_encode(mimi, chunks):
    """Concatenated encode_step codes = encode() of the whole audio (frame-aligned), with the near-tie allowance of the one-shot encode test
    (fp32 latents from different kernels move some deep arg-mins); per call, the frames the oracle says it completes."""
    model, P64 = mimi
    g = torch.Generator().manual_seed(sum(chunks) + len(chunks))
    n = sum(chunks) // 1920 * 1920
    pcm = torch.randn(2, 1, sum(chunks), generator=g) * 0.3
    want_counts = [p.shape[-1] for p in MS.encode_stream(P64, pcm.double(), chunks)] if len(chunks) < 4 else None
    model.reset_state()
    a, parts = 0, []
    for c in chunks:
        parts.append(model.encode_step(pcm[:, :, a:a + c]).cpu())
        a += c
    counts = [p.shape[-1] for p in parts]
    seen, done, exp = 0, 0, []
    for c in chunks:
        seen += c
        exp.append(seen // 1920 - done)
        done = seen // 1920
    assert counts == exp and (want_counts is None or counts == want_counts)
    assert all(p.shape[:2] == (2, 32) and p.dtype == torch.int64 for p in parts)
    got = torch.cat(parts, -1)
    want = model.encode(pcm[..., :n]).cpu()
    same = (got == want).float()
    assert float(same[:, :4].mean()) >= 0.9 and float(same.mean()) >= 0.6, (float(same[:, :4].mean()), float(same.mean()))


def test_encode_step_sub_frame_chunk_returns_no_frames(mimi):
    model, _ = mimi
    model.reset_state()
    pcm = torch.randn(2, 1, 700) * 0.3
    c = model.encode_step(pcm)
    assert c.shape == (2, 32, 0) and c.dtype == torch.int64
    with pytest.raises(ValueError):
        model.encode_step(pcm[:1])
