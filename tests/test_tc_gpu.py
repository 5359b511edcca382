"""Tensor-core path (csrc/gemm_tc.cu) vs the float64 oracle and vs the CUDA-core kernel.
x2 mode (hi+lo bf16 activation planes, bf16-exact weights) must be fp32-grade: <= 2e-5 of the output scale.
x1 mode (single bf16 plane) carries bf16 activation rounding: <= 4e-3."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nn as ON


def _rand(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


@pytest.fixture(params=["gemm_tc", "fused"])
def path(request):
    """Every dense-conv case runs through both tensor-core kernels: round 1's prologue pass + conv_tc_kernel (csrc/gemm_tc.cu) and
    the fused kernel that converts the activations on the fly (csrc/conv_fused.cu)."""
    from mlx_audio_b200 import ops
    old, oldd = ops.FUSED[0], ops.FUSED_DISPATCH[0]
    ops.FUSED[0] = ops.FUSED_DISPATCH[0] = request.param == "fused"
    yield request.param
    ops.FUSED[0], ops.FUSED_DISPATCH[0] = old, oldd


CASES = [
    # B, L, Cin, Cout, K, dil, pad
    (1, 300, 128, 128, 7, 3, 9),
    (1, 1000, 256, 256, 11, 5, 25),
    (1, 130, 768, 2304, 1, 1, 0),
    (1, 390, 1090, 1024, 3, 1, 1),
    (2, 257, 64, 64, 3, 1, 1),
    (1, 129, 96, 32, 5, 2, 4),
    (1, 5000, 128, 128, 3, 1, 1),
    (1, 3000, 64, 64, 1, 1, 0),
    (2, 700, 96, 96, 7, 9, 54),          # Qwen3 vocoder block 4, taps spanning 54 rows; 12 row tiles: 32-wide N tiles on conv_tc
    (1, 40000, 192, 192, 7, 3, 18),      # 96-wide N tiles, several waves of CTAs (every N tile: test_gemm_tc_matrix_gpu.py)
    (1, 600, 384, 384, 1, 1, 0),
    (1, 5000, 32, 64, 1, 1, 0),          # Mimi's last residual 1x1 (hidden 32): half of the 64-wide K chunk is zero padding
]


@pytest.mark.parametrize("mode,tol", [("x2", 2e-5), ("x1", 4e-3)])
@pytest.mark.parametrize("case", CASES)
def test_conv1d_tc(case, mode, tol, path):
    from mlx_audio_b200 import ops
    B, L, Cin, Cout, K, dil, pad = case
    dev = torch.device("cuda:0")
    x = _rand(B, L, Cin, seed=1)
    w = (_rand(Cout, K, Cin, seed=2, scale=0.05)).to(torch.bfloat16).float()
    bias = _rand(Cout, seed=3, scale=0.1)
    sc, sh = 1 + 0.3 * _rand(B, Cin, seed=4), 0.2 * _rand(B, Cin, seed=5)
    a = (1 + 0.2 * _rand(Cin, seed=6)).abs() + 0.1
    v = x.double() * sc.double()[:, None] + sh.double()[:, None]
    v = v + (1.0 / a.double()) * torch.sin(a.double() * v) ** 2
    ref = ON.conv1d(v, w.double(), 1, pad, dil, 1, bias.double())
    res = _rand(*ref.shape, seed=7)
    ref = (ref + res.double()) * 0.5
    cw = ops.pack_conv(w, bias, 1, dev)
    assert cw.w_tc is not None
    pre = ops.Pre(sc.to(dev).contiguous(), sh.to(dev).contiguous(), ops.ACT["snake"], 0.0, a.to(dev), (1.0 / a).to(dev))
    old = ops.TC_MODE[0]
    try:
        ops.TC_MODE[0] = mode
        assert ops._tc_eligible(cw, L, 1, False, 0)
        y = ops.conv1d(x.to(dev), cw, dilation=dil, pad_left=pad, pre=pre, res=res.to(dev), out_scale=0.5)
        torch.cuda.synchronize()
    finally:
        ops.TC_MODE[0] = old
    assert y.shape == ref.shape
    e = rel_err(y, ref)
    assert e < tol, e
    if mode == "x2":
        y_cc = ops.conv1d(x.to(dev), cw, dilation=dil, pad_left=pad, pre=pre, res=res.to(dev), out_scale=0.5)
        assert rel_err(y, y_cc.double()) < 2e-5


def test_conv1d_tc_epilogue_variants(path):
    from mlx_audio_b200 import ops
    dev = torch.device("cuda:0")
    x = _rand(2, 200, 128, seed=1)
    w = _rand(64, 3, 128, seed=2, scale=0.05).to(torch.bfloat16).float()
    cs = _rand(2, 64, seed=3)
    y0 = _rand(2, 200, 64, seed=4)
    ref = ON.gelu(ON.conv1d(x.double(), w.double(), 1, 1, 1, 1)) * cs.double()[:, None] + y0.double()
    cw = ops.pack_conv(w, None, 1, dev)
    old = ops.TC_MODE[0]
    try:
        ops.TC_MODE[0] = "x2"
        out = y0.to(dev).clone()
        big = torch.zeros(2, 200, 100, device=dev)
        y = ops.conv1d(x.to(dev), cw, pad_left=1, post_act=ops.ACT["gelu"], cscale=cs.to(dev), out=out, accumulate=True)
        ops.conv1d(x.to(dev), cw, pad_left=1, post_act=ops.ACT["gelu"], cscale=cs.to(dev), res=y0.to(dev), out=big[:, :, 8:72])
    finally:
        ops.TC_MODE[0] = old
    assert rel_err(y, ref) < 2e-5 and rel_err(big[:, :, 8:72], ref) < 2e-5
    assert float(big[:, :, :8].abs().max()) == 0 and float(big[:, :, 72:].abs().max()) == 0


@pytest.mark.parametrize("B,L,Cin,Cout,K,stride,pad,opad", [(1, 780, 512, 256, 20, 10, 5, 0), (1, 500, 256, 128, 12, 6, 3, 0),
                                                             (2, 300, 128, 64, 16, 8, 4, 1), (1, 257, 64, 32, 4, 2, 1, 1), (1, 100, 256, 128, 8, 4, 0, 0)])
def test_convtr1d_tc_polyphase(B, L, Cin, Cout, K, stride, pad, opad, path):
    """Transposed conv on the tensor-core path (K = 2*stride, polyphase: the GEMM output is the up-sampled signal)."""
    from mlx_audio_b200 import ops
    dev = torch.device("cuda:0")
    x = _rand(B, L, Cin, seed=1)
    w = _rand(Cout, K, Cin, seed=2, scale=0.05).to(torch.bfloat16).float()
    bias = _rand(Cout, seed=3, scale=0.1)
    ref = ON.conv_transpose1d(ON.leaky_relu(x.double(), 0.1), w.double(), stride, pad, 1, opad, 1, bias.double())
    res = _rand(*ref.shape, seed=5)
    ref = ref + res.double()
    cw = ops.pack_conv(w, bias, 1, dev)
    old = ops.TC_MODE[0]
    try:
        ops.TC_MODE[0] = "x2"
        assert ops._tc_eligible(cw, L, stride, True, 0)
        y = ops.conv1d(x.to(dev), cw, stride=stride, pad_left=pad, lout=ref.shape[1], pre=ops.Pre(act=ops.ACT["lrelu"], p0=0.1),
                       res=res.to(dev), transpose=True)
        torch.cuda.synchronize()
    finally:
        ops.TC_MODE[0] = old
    assert y.shape == ref.shape and rel_err(y, ref) < 2e-5
