"""Kokoro's harmonic-source convs (csrc/conv.cu: b2a_kokoro_source_conv) against the CUDA-core dense tile and float64.

The kernel replaces b2a_conv1d_cl's generic dense tile for the two noise convs on the 22-channel source (K = 12 / stride 6 into 256
channels, K = 1 into 128) and promises the same bytes: the tile's fmaf sequence per output, including what its zero-padded channels
do to a -0 accumulator.  Each case compares the two bit for bit (as int32 words, so -0 and +0 differ) and checks both against
oracle/nn.py's conv1d in float64.  Lengths are the source of F frames, 120 F + 1 rows: F = 1, 2, 3 (one partial CTA tile), 37, 390
(the benchmark's utterance) and 391, so the last tile is ragged and the zero padding is read at both ends.  The source is a slice of
a NaN-filled buffer, so a read outside its rows poisons the result."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nn as ON

DEV = "cuda:0"
TOL = 2e-5
CONVS = {"k12s6": (256, 12, 6, 3), "k1": (128, 1, 1, 0)}      # Cout, K, stride, pad_left (kokoro.py: noise_convs[0], [1])


def _source(L, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    guard = 64
    buf = torch.full(((L + 2 * guard) * 22,), float("nan"), device=DEV)
    buf[guard * 22:(guard + L) * 22] = (torch.randn(L * 22, generator=g) * scale).to(DEV)
    return buf[guard * 22:(guard + L) * 22].view(1, L, 22)


def _layer(conv, seed, bias=True, wscale=0.2, negative=False):
    from mlx_audio_b200 import ops
    cout, K, _, _ = CONVS[conv]
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(cout, K, 22, generator=g) * wscale               # MLX layout [Cout, K, Cin]
    if negative:
        w = -w.abs()
    b = torch.randn(cout, generator=g) if bias else None             # negative entries included
    return ops.pack_conv(w, b, 1, DEV), w, b


def _cuda_core(x, cw, stride, pad):
    from mlx_audio_b200 import ops
    y = ops.conv1d(x, cw, stride=stride, pad_left=pad)
    path = ops.conv1d_cl_last_path()
    assert path["kernel"] == "dense" and path["variant"] == (64, 32 if cw.K == 1 else 16, 0), path
    return y


def _bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("conv", sorted(CONVS))
@pytest.mark.parametrize("F", [1, 2, 3, 37, 390, 391])
def test_source_conv_matches_dense_tile_and_float64(conv, F):
    from mlx_audio_b200 import ops
    _, K, stride, pad = CONVS[conv]
    L = 120 * F + 1
    x = _source(L, seed=F)
    cw, w, b = _layer(conv, seed=100 + F)
    y = ops.kokoro_source_conv(x, cw, stride=stride, pad_left=pad)
    ref = _cuda_core(x, cw, stride, pad)
    torch.cuda.synchronize()
    assert y.shape == ref.shape == (1, (L + 2 * pad - K) // stride + 1, cw.cout)
    assert torch.isfinite(y).all()
    assert _bits_equal(y, ref), f"{(y != ref).sum().item()} outputs differ from the dense tile"
    want = ON.conv1d(x.double().cpu(), w.double(), stride=stride, padding=pad, bias=b.double())
    err = float((y.double().cpu() - want).abs().max() / want.abs().max())
    assert err <= TOL, err


@pytest.mark.parametrize("conv", sorted(CONVS))
def test_source_conv_signed_zero(conv):
    """Products that underflow to -0 (a positive source of ~1e-30 times negative weights of ~1e-17, no bias): the dense tile's padded
    channels turn the -0 accumulator into +0 after every tap of its last chunk; the new kernel must do the same."""
    from mlx_audio_b200 import ops
    _, K, stride, pad = CONVS[conv]
    x = _source(120 * 3 + 1, seed=7, scale=1e-30).abs()
    cw, _, _ = _layer(conv, seed=8, bias=False, wscale=1e-17, negative=True)
    y = ops.kokoro_source_conv(x, cw, stride=stride, pad_left=pad)
    ref = _cuda_core(x, cw, stride, pad)
    torch.cuda.synchronize()
    assert (ref == 0).all() and not torch.signbit(ref).any()
    assert _bits_equal(y, ref)


def test_source_conv_rejects_other_shapes():
    from mlx_audio_b200 import ops
    cw, _, _ = _layer("k12s6", seed=1)
    with pytest.raises(NotImplementedError):
        ops.kokoro_source_conv(_source(361, seed=1), cw, stride=4, pad_left=2)
    with pytest.raises(ValueError):
        ops.kokoro_source_conv(torch.zeros(1, 361, 24, device=DEV), cw, stride=6, pad_left=3)
