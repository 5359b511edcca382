"""Kokoro's text side as a plane-emitting launch chain: every producer writes the 16-bit operand planes its tensor-core consumer reads.

Each emitted plane must be bit for bit what the stand-alone prep kernel makes of the fp32 value it replaces, the N tile the small-M
GEMMs now take must not change a single output bit, and the chain must reproduce the separate-op ALBERT exactly."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import _lib, ops, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
T = 130                                             # cfg2: 128 phonemes + BOS / EOS
ALBERT_SHAPES = [(768, 2304), (768, 768), (768, 2048), (2048, 768)]     # qkv, attn_out, ffn, ffn_out


def _bf16_linear(cin, cout, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(cout, cin, generator=g) / cin ** 0.5).to(torch.bfloat16).float()
    b = torch.randn(cout, generator=g) * 0.1
    return ops.pack_linear(w, b, device="cuda")


def _x(*shape, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g).cuda()


def _same_planes(pl, ref_hi, ref_lo):
    assert torch.equal(pl.hi.view(torch.int16), ref_hi.view(torch.int16))
    assert torch.equal(pl.lo.view(torch.int16), ref_lo.view(torch.int16))


@pytest.mark.parametrize("C_", [128, 768])
def test_layernorm_planes_equal_prep(C_):
    x, r = _x(T, C_, seed=1) * 3, _x(T, C_, seed=2)
    w, b = _x(C_, seed=3), _x(C_, seed=4)
    ref = ops.layernorm(x, w, b, eps=1e-12, res=r)
    y, pl = ops.layernorm(x, w, b, eps=1e-12, res=r, planes=True)
    assert torch.equal(y, ref)
    _same_planes(pl, *ops.prep_bf16(y[None], None, C_))


@pytest.mark.parametrize("act,res", [(0, False), (ops.ACT["gelu"], False), (0, True), (ops.ACT["gelu"], True)])
def test_gemm_epilogue_planes_equal_prep(act, res):
    cw = _bf16_linear(768, 2048, seed=5)
    x = _x(1, T, 768, seed=6)
    r = _x(1, T, 2048, seed=7) if res else None
    ref = ops.linear(x, cw, post_act=act, res=r)
    y, pl = ops.linear(x, cw, post_act=act, res=r, planes=True)
    assert torch.equal(y, ref)
    _same_planes(pl, *ops.prep_bf16(y, None, 2048))
    # a Planes operand feeds the next GEMM exactly like the fp32 tensor it stands for
    cw2 = _bf16_linear(2048, 768, seed=8)
    assert torch.equal(ops.linear(pl, cw2), ops.linear(y, cw2))


def test_qkv_attention_planes_equal_prep():
    H, hs = 12, 768
    cw = _bf16_linear(hs, 3 * hs, seed=9)
    x = _x(1, T, hs, seed=10)
    scale = 1.0 / 8.0
    qkv = ops.linear(x, cw)
    y, ap = ops.linear(x, cw, qkv_heads=H, qkv_scale=scale)
    assert torch.equal(y, qkv)
    # the stand-alone entry point's own prologue into a workspace of the same layout
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
    assert torch.equal(ctx, ops.attention(q, k, v, n_heads=H, scale=scale))
    _same_planes(cp, *ops.prep_bf16(ctx, None, hs))


@pytest.mark.parametrize("cin,cout", ALBERT_SHAPES)
def test_conv_tc_bit_identical_across_n_tiles(cin, cout):
    """At B = 1 the 2 row tiles leave the GPU mostly idle and the GEMM runs 32-wide N tiles; at B = 12 (24 row tiles) it keeps the
    128-wide ones.  Every batch row of the wide-tile run must equal the narrow-tile result bit for bit."""
    cw = _bf16_linear(cin, cout, seed=11)
    x = _x(1, T, cin, seed=12)
    r = _x(1, T, cout, seed=13)
    narrow = ops.linear(x, cw, res=r, post_act=ops.ACT["gelu"])
    wide = ops.linear(x.expand(12, T, cin).contiguous(), cw, res=r.expand(12, T, cout).contiguous(), post_act=ops.ACT["gelu"])
    for b in range(12):
        assert torch.equal(wide[b], narrow[0])


@pytest.fixture(scope="module")
def kokoro():
    from mlx_audio_b200.configs import KOKORO_82M
    from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig
    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    model = Model(ModelConfig.from_dict(KOKORO_82M), device="cuda:0").load_weights(list(P.items()))
    ids, ref_s = synth.kokoro_inputs(128, seed=1)
    assert ids.shape[1] == T
    return model, ids[0].cuda(), ref_s.cuda()


def _text(model, ids, ref_s):
    model.tap = {}
    st = model._text_side(ids, ref_s)
    torch.cuda.synchronize()
    bert, model.tap = model.tap["bert"], None
    return bert, st


def test_albert_chain_matches_separate_ops(kokoro):
    model, ids, ref_s = kokoro
    assert model._albert_planes(T)
    bert, st = _text(model, ids, ref_s)
    model._albert_planes = lambda T_: False
    try:
        bert0, st0 = _text(model, ids, ref_s)
    finally:
        del model._albert_planes
    assert torch.equal(bert, bert0)
    for k in ("X", "t_en", "pred", "idx", "total"):
        assert torch.equal(st[k], st0[k]), k


def test_albert_launches_per_layer(kokoro):
    model, ids, ref_s = kokoro
    pb = model.config.plbert
    n_layers = pb["num_hidden_layers"]
    counts = []
    try:
        for n in (n_layers, n_layers - 1):
            pb["num_hidden_layers"] = n
            n0 = ops.LAUNCHES[0]
            model._text_side(ids, ref_s)
            counts.append(ops.LAUNCHES[0] - n0)
    finally:
        pb["num_hidden_layers"] = n_layers
    torch.cuda.synchronize()
    assert counts[0] - counts[1] <= 7, counts


def test_text_graph_replays_eager(kokoro):
    model, ids, ref_s = kokoro
    _, st = _text(model, ids, ref_s)
    ent = model._text_graph(T, 1.0, False)
    ent["ids"].copy_(ids)
    ent["ref_s"].copy_(ref_s)
    ent["graph"].replay()
    torch.cuda.synchronize()
    for k in ("X", "t_en", "pred", "idx", "total"):
        assert torch.equal(ent["st"][k], st[k]), k


_PDL_OFF = """
import sys, numpy as np, torch
sys.path.insert(0, {root!r})
from mlx_audio_b200 import synth
from mlx_audio_b200.configs import KOKORO_82M
from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig
m = Model(ModelConfig.from_dict(KOKORO_82M), device="cuda:0").load_weights(list(synth.kokoro_weights(KOKORO_82M, seed=0).items()))
ids, ref_s = synth.kokoro_inputs(128, seed=1)
st = m._text_side(ids[0].cuda(), ref_s.cuda())
np.savez({out!r}, X=st["X"].cpu().numpy(), pred=st["pred"].cpu().numpy())
"""


def test_pdl_off_identical(kokoro, tmp_path):
    model, ids, ref_s = kokoro
    _, st = _text(model, ids, ref_s)
    out = str(tmp_path / "pdl_off.npz")
    env = dict(os.environ, B2A_PDL="0")
    subprocess.run([sys.executable, "-c", _PDL_OFF.format(root=ROOT, out=out)], env=env, check=True, timeout=600)
    r = np.load(out)
    assert np.array_equal(r["X"], st["X"].cpu().numpy())
    assert np.array_equal(r["pred"], st["pred"].cpu().numpy())
