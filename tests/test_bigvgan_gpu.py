"""BigVGAN on the GPU against the float64 oracle (oracle/bigvgan.py, itself pinned to the reference's code by tests/test_bigvgan_pins.py):
the anti-aliased SnakeBeta kernel on its own, and the whole vocoder at the released widths with synthetic weights."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import ops, synth
from oracle import bigvgan as OB

DEV = "cuda:0"


def rel_rms(a, b):
    a, b = torch.as_tensor(a).double().cpu().reshape(-1), torch.as_tensor(b).double().cpu().reshape(-1)
    return float(torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean()))


def _act_case(B, L, C, seed, asym=False):
    g = torch.Generator().manual_seed(seed)
    x = 2.0 * torch.randn(B, L, C, generator=g, dtype=torch.float64)
    alpha, beta = 0.3 * torch.randn(C, generator=g, dtype=torch.float64), 0.3 * torch.randn(C, generator=g, dtype=torch.float64)
    if asym:
        fu, fd = torch.randn(12, generator=g, dtype=torch.float64) / 3, torch.randn(12, generator=g, dtype=torch.float64) / 3
    else:
        fu = fd = OB.kaiser_sinc_filter1d(0.25, 0.3, 12)
    x, alpha, beta, fu, fd = (t.float().double() for t in (x, alpha, beta, fu, fd))          # the oracle sees exactly the fp32 inputs
    P = {"x.act.alpha": alpha, "x.act.beta": beta, "x.upsample.filter": fu, "x.downsample.lowpass.filter": fd}
    want = OB.activation1d(P, "x", x, True)
    args = [t.float().to(DEV).contiguous() for t in (torch.exp(alpha), 1.0 / (torch.exp(beta) + 1e-9), fu, fd)]
    return x.float().to(DEV), args, want


# fp32 products and sums over 6 + 12 taps and the SFU sine against float64: measured at most 2.7e-7 of max|y| over these cases on an
# NVIDIA H100 80GB HBM3 (700 W)
ACT_TOL = 2e-6


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("C", [24, 48, 96, 768])
@pytest.mark.parametrize("L", [1, 2, 3, 129, 4096, 777])
def test_aa_snakebeta_against_oracle(B, C, L):
    x, args, want = _act_case(B, L, C, seed=L * 1000 + C + B)
    y = ops.aa_snakebeta(x, *args)
    assert y.shape == want.shape
    err = float((y.double().cpu() - want).abs().max() / want.abs().max())
    print("aa_snakebeta rel err", B, C, L, err)
    assert err < ACT_TOL, err


class _TC:
    """Stand-in for a tensor-core conv's packing: only the channel count and the planes' width matter to aa_snakebeta."""
    def __init__(self, C):
        self.cin, self.cin_pad, self.w_tc, self.f16 = C, -(-C // 64) * 64, torch.empty(0), False


@pytest.mark.parametrize("C,L", [(96, 129), (768, 4096), (48, 3), (384, 777)])
def test_aa_snakebeta_planes(C, L):
    """bf16 hi / lo planes for the next tensor-core conv: hi + lo is the fp32 result to ~2^-17, pad channels are zero."""
    x, args, _ = _act_case(2, L, C, seed=7 + C)
    y = ops.aa_snakebeta(x, *args)
    pl = ops.aa_snakebeta(x, *args, planes_for=_TC(C))
    assert isinstance(pl, ops.Planes) and pl.hi.shape == (2, L, -(-C // 64) * 64) and pl.C == C
    if ops.TC_MODE[0] == "x2":
        rec = pl.hi.float() + pl.lo.float()
        assert float((rec[..., :C] - y).abs().max()) <= 2 ** -16 * float(y.abs().max())
        assert not bool(pl.lo[..., C:].any())
    assert torch.equal(pl.hi[..., :C], y.to(torch.bfloat16)) and not bool(pl.hi[..., C:].any())


def test_aa_snakebeta_non_symmetric_filters_and_strided_input():
    x, args, want = _act_case(2, 300, 96, seed=3, asym=True)
    y = ops.aa_snakebeta(x, *args)
    assert float((y.double().cpu() - want).abs().max() / want.abs().max()) < ACT_TOL
    flipped = ops.aa_snakebeta(x, args[0], args[1], args[2].flip(0).contiguous(), args[3].flip(0).contiguous())
    assert float((flipped - y).abs().max()) > 1e-2 * float(y.abs().max())                  # the filters' orientation shows
    wide = torch.zeros(2, 300, 160, device=DEV)                                             # channel slice of a wider buffer
    wide[:, :, 32:128] = x
    batched = torch.zeros(5, 300, 96, device=DEV)                                            # every other item of a batch
    batched[::2][:2] = x
    for xv in (wide[:, :, 32:128], batched[::2][:2]):
        assert not xv.is_contiguous()
        assert torch.equal(ops.aa_snakebeta(xv, *args), y)


def test_aa_snakebeta_rejects_other_shapes():
    x, args, _ = _act_case(1, 16, 24, seed=1)
    with pytest.raises(NotImplementedError):
        ops.aa_snakebeta(x, args[0], args[1], torch.ones(8, device=DEV), torch.ones(8, device=DEV))
    with pytest.raises(ValueError):
        ops.aa_snakebeta(x, args[0][:10].contiguous(), *args[1:])


# ---- the whole vocoder --------------------------------------------------------------------------------------------------------
def _model(base, **over):
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    cfg = dict(base, **over)
    P = synth.bigvgan_weights(BigVGANConfig(**cfg))
    return BigVGAN(BigVGANConfig(**cfg), device=DEV).load_weights(P), P, cfg


@pytest.fixture(scope="module", params=["22k", "44k"])
def released(request):
    return _model(OB.BIGVGAN_22K if request.param == "22k" else OB.BIGVGAN_44K)


def test_vocoder_against_oracle(released):
    model, P, cfg = released
    mel = torch.randn(1, cfg["num_mels"], 64, generator=torch.Generator().manual_seed(5))
    want = OB.forward({k: v.double() for k, v in P.items()}, mel.double(), cfg)
    y = model(mel.to(DEV))
    assert y.shape == want.shape == (1, 1, 64 * OB.output_length(cfg, 1))
    # 44 convs in sequence at up to 1536 channels, unit-gain weights through bf16 hi / lo operand planes (~2^-16 per product): measured
    # 2.6e-4 (22 kHz) and 3.1e-4 (44 kHz) on an NVIDIA H100 80GB HBM3 (700 W); the bound is the DAC decoder's
    err = rel_rms(y, want)
    print("vocoder rel RMS", cfg["num_mels"], err)
    assert err < 2e-3, err


def test_batch_rows_equal_single_calls(released):
    """Dispatch depends on the sequence length only, never on B, and every kernel's summation order is fixed: a batched call returns
    the same bits as each row on its own."""
    model, _, cfg = released
    mel = torch.randn(2, cfg["num_mels"], 50, generator=torch.Generator().manual_seed(6)).to(DEV)
    both = model(mel)
    for b in range(2):
        assert torch.equal(both[b:b + 1], model(mel[b:b + 1])), b


@pytest.mark.parametrize("which", ["22k", "44k"])
def test_reference_shape_pins(which):
    """codec/tests/test_bigvgan.py through the shim path: 800 frames -> 800 * 256 / 800 * 512 samples, finite and within [-1, 1]."""
    from mlx_audio.codec.models.bigvgan.bigvgan import BigVGAN, BigVGANConfig
    cfg = OB.BIGVGAN_22K if which == "22k" else OB.BIGVGAN_44K
    model = BigVGAN(BigVGANConfig(**cfg))
    y = model(torch.zeros(1, cfg["num_mels"], 800))
    assert y.shape == (1, 1, 800 * (256 if which == "22k" else 512))
    assert bool(torch.isfinite(y).all()) and float(y.abs().max()) <= 1.0


def _torch_layout(P, cfg):
    """A torch-layout checkpoint of the MLX-layout tree P, with the filters and a BatchNorm counter, as a released file holds them."""
    from mlx_audio_b200.codec.models.bigvgan import kaiser_sinc_filter1d, param_shapes
    out = {}
    for k, shape in param_shapes(cfg).items():
        v = P[k] if k in P else kaiser_sinc_filter1d(0.25, 0.3, 12).float().reshape(shape)
        if k.startswith("ups.") and v.dim() == 3:
            v = v.permute(2, 0, 1)
        elif v.dim() == 3:
            v = v.permute(0, 2, 1)
        out[k] = v.contiguous()
    out["conv_pre.num_batches_tracked"] = torch.tensor(0)
    return out


@pytest.mark.parametrize("resblock,tanh", [("1", False), ("2", True)])
def test_checkpoint_round_trip(resblock, tanh):
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    model, P, cfg = _model(OB.BIGVGAN_22K, upsample_initial_channel=256, resblock=resblock, use_tanh_at_final=tanh, use_bias_at_final=tanh)
    other = BigVGAN(BigVGANConfig(**cfg), device=DEV)
    other.load_weights(other.sanitize(_torch_layout(P, BigVGANConfig(**cfg))))
    mel = torch.randn(2, 80, 40, generator=torch.Generator().manual_seed(8)).to(DEV)
    y = model(mel)
    assert torch.equal(other(mel), y)
    want = OB.forward({k: v.double() for k, v in P.items()}, mel.double().cpu(), cfg)
    assert rel_rms(y, want) < 2e-3


def test_snake_raises():
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    with pytest.raises(NotImplementedError):
        BigVGAN(BigVGANConfig(**dict(OB.BIGVGAN_22K, activation="snake")), device=DEV)
