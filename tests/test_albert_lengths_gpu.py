"""Kokoro's ALBERT encoder across utterance lengths, against the float64 oracle (oracle/kokoro.py:albert).

T decides how the text side runs: below 64 tokens as separate ops, from 64 as the plane-emitting launch chain; the row-tile count
(1 to 4) and its ragged tail; the zero keys that pad the transposed V plane to a multiple of 8; and the qkv GEMM's N tile (32-wide
while its grid covers under half the SMs, 128-wide from T = 385 on 132 SMs).  The lengths below sit on each side of those edges."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import _lib, ops, synth
from oracle import kokoro as OK

LENGTHS = [31, 32, 63, 64, 65, 127, 128, 129, 192, 255, 256, 257, 384, 385, 511, 512]
# Relative RMS.  Measured on an H100 80GB HBM3: 7.1e-6 to 7.5e-6 from T = 32 to 512 in x2 (5e-7 at T = 31, where the GEMMs have too
# few rows for the tensor cores and run in fp32 on the CUDA cores); 1.5e-3 at T = 257 in x1, where every GEMM rounds its input to
# 8 significant bits.  test_kokoro_gpu.py bounds the whole text side at 1e-4.
TOL_BERT = 2e-5
TOL_BERT_X1 = 5e-3
STATE = ("X", "t_en", "pred", "idx", "total")


def rel_rms(a, b):
    a, b = a.double().cpu().reshape(-1), b.double().cpu().reshape(-1)
    return float(torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean()))


@pytest.fixture(scope="module")
def kokoro():
    from mlx_audio_b200.configs import KOKORO_82M
    from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig
    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    model = Model(ModelConfig.from_dict(KOKORO_82M), device="cuda:0").load_weights(list(P.items()))
    P64 = {k: v.double() for k, v in P.items() if k.startswith("bert.")}
    return model, P64, KOKORO_82M["plbert"]


def _inputs(T):
    ids, ref_s = synth.kokoro_inputs(T - 2, seed=T)
    assert ids.shape[1] == T
    return ids, ref_s


def _text(model, ids, ref_s):
    model.tap = {}
    st = model._text_side(ids[0].cuda(), ref_s.cuda())
    torch.cuda.synchronize()
    bert, model.tap = model.tap["bert"], None
    return bert, st


def _separate_ops(model, ids, ref_s):
    model._albert_planes = lambda T_: False
    try:
        return _text(model, ids, ref_s)
    finally:
        del model._albert_planes


def _oracle(P64, ids, pb):
    return OK.albert(P64, ids, torch.ones_like(ids), pb)[0]


@pytest.mark.parametrize("T", LENGTHS)
def test_albert_vs_float64(kokoro, T):
    """tap["bert"] against float64; from T = 64 the launch chain, which must equal the separate-op path bit for bit."""
    model, P64, pb = kokoro
    ids, ref_s = _inputs(T)
    assert model._albert_planes(T) == (T >= 64)
    bert, st = _text(model, ids, ref_s)
    e = rel_rms(bert, _oracle(P64, ids, pb))
    print(f"\n[albert] T {T}: bert rel RMS {e:.2e}")
    assert e < TOL_BERT, e
    if T >= 64:
        bert0, st0 = _separate_ops(model, ids, ref_s)
        assert torch.equal(bert, bert0)
        for k in STATE:
            assert torch.equal(st[k], st0[k]), k


def test_albert_x1_vs_float64(kokoro):
    """The chain with one bf16 activation plane per GEMM (TC_MODE x1): within bf16 rounding of the oracle, and still equal to the
    separate-op path."""
    model, P64, pb = kokoro
    T = 257
    ids, ref_s = _inputs(T)
    old, ops.TC_MODE[0] = ops.TC_MODE[0], "x1"
    try:
        assert model._albert_planes(T)
        bert, st = _text(model, ids, ref_s)
        bert0, st0 = _separate_ops(model, ids, ref_s)
    finally:
        ops.TC_MODE[0] = old
    e = rel_rms(bert, _oracle(P64, ids, pb))
    print(f"\n[albert x1] T {T}: bert rel RMS {e:.2e}")
    assert TOL_BERT < e < TOL_BERT_X1, e               # also shows the x1 mode really ran
    assert torch.equal(bert, bert0)
    for k in STATE:
        assert torch.equal(st[k], st0[k]), k


@pytest.mark.parametrize("T", [64, 257, 512])
def test_qkv_attention_planes_equal_prep(T):
    """The qkv GEMM's epilogue writes the attention's fp16 planes exactly as the attention's own prep kernels do: one row tile and
    no V padding (64), a ragged tile with 7 zero keys (257), and 4 full row tiles at the 128-wide N tile (512)."""
    import ctypes as C
    H, hs = 12, 768
    g = torch.Generator().manual_seed(9)
    w = (torch.randn(3 * hs, hs, generator=g) / hs ** 0.5).to(torch.bfloat16).float()
    cw = ops.pack_linear(w, torch.randn(3 * hs, generator=g) * 0.1, device="cuda")
    x = torch.randn(1, T, hs, generator=g).cuda()
    scale = 1.0 / 8.0
    qkv = ops.linear(x, cw)
    y, ap = ops.linear(x, cw, qkv_heads=H, qkv_scale=scale)
    bn = ops.conv1d_tc_last_config()["BN"]
    print(f"\n[qkv planes] T {T}: N tile {bn}")
    if T == 512:
        assert bn == 128
    assert torch.equal(y, qkv)
    ws = torch.empty_like(ap.ws)
    p = _lib.AttnParams()
    q, k, v = qkv[:, :, :hs], qkv[:, :, hs:2 * hs], qkv[:, :, 2 * hs:]
    o = torch.empty(1, T, hs, device="cuda")
    p.q, p.k, p.v, p.o = q.data_ptr(), k.data_ptr(), v.data_ptr(), o.data_ptr()
    p.q_bs, p.q_ld, p.k_bs, p.k_ld, p.v_bs, p.v_ld, p.o_bs, p.o_ld = q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1), o.stride(0), o.stride(1)
    p.B, p.Tq, p.Tk, p.H, p.Hkv, p.D, p.scale = 1, T, T, H, H, 64, scale
    _lib.check(_lib.lib().b2a_attention_tc(C.byref(p), ws.data_ptr(), torch.cuda.current_stream().cuda_stream))
    tkp = (T + 7) // 8 * 8
    n = 2 * 2 * H * 64 * (2 * T + tkp)                # bytes of the q / k / v^T hi and lo planes
    off = (-ap.ws.data_ptr()) % 256
    assert (-ws.data_ptr()) % 256 == off
    assert torch.equal(ap.ws[off:off + n], ws[off:off + n])
    ctx, cp = ops.attention_planes(ap, planes=True)
    assert torch.equal(ctx, o)
    hi, lo = ops.prep_bf16(ctx, None, hs)
    assert torch.equal(cp.hi.view(torch.int16), hi.view(torch.int16)) and torch.equal(cp.lo.view(torch.int16), lo.view(torch.int16))


@pytest.mark.parametrize("T", [64, 257, 512])
def test_text_graph_replays_eager(kokoro, T):
    model = kokoro[0]
    ids, ref_s = _inputs(T)
    _, st = _text(model, ids, ref_s)
    ent = model._text_graph(T, 1.0, False)
    ent["ids"].copy_(ids[0].cuda())
    ent["ref_s"].copy_(ref_s.cuda())
    ent["graph"].replay()
    torch.cuda.synchronize()
    for k in STATE:
        assert torch.equal(ent["st"][k], st[k]), k
