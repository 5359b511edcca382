"""Tensor-core GEMM (csrc/gemm_tc.cu, csrc/conv_fused.cu) against float64 across its configuration space: every N tile the dispatch
rule can choose, the three weight precisions (bf16-exact, fp16-exact, fp32 split into bf16 hi + lo) in both activation modes, the
split-K and grouped launches of the fused kernel, and the input range over which the fp16 mode stays fp32-grade.

Errors are max |y - ref| / max |ref|.  x2 (hi + lo activation planes) must be fp32-grade, <= 2e-5, for every weight kind.  x1 (one
16-bit activation plane) carries that plane's rounding: <= 4e-3 with bf16 planes (8 significant bits); fp16 planes have 11, three
more, so the same statistics give 4e-3 / 2^3 = 5e-4.  Negative controls drop one product (the activation lo plane; the weight lo
plane of an fp32 checkpoint) and must exceed 5x the x2 bound, so that bound would notice a kernel that lost a product."""
import dataclasses
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from oracle import nn as ON

TOL_X2 = 2e-5
TOL_X1 = {"bf16": 4e-3, "fp16": 5e-4, "fp32": 4e-3}
DEV = "cuda:0"


def _rand(*shape, seed=0, scale=1.0):
    return torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale


def rel_err(a, b):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def _nsm():
    from mlx_audio_b200 import _lib
    return _lib.lib().b2a_device_sm_count()


def _rows(tiles):
    """Rows giving `tiles` 128-row tiles, the last one ragged (37 rows)."""
    return (tiles - 1) * 128 + 37


def _weights(kind, cout, k, cin, seed):
    w = _rand(cout, k, cin, seed=seed, scale=0.05)
    if kind == "bf16":
        return w.to(torch.bfloat16).float()
    if kind == "fp16":
        w = w.half().float()
        assert not torch.equal(w.to(torch.bfloat16).float(), w)       # fp16-exact but not bf16-exact
        return w
    return w


def _pack(kind, w, bias):
    """pack_conv must classify the checkpoint: bf16 -> one bf16 plane, fp16 -> one fp16 plane, fp32 -> bf16 hi + lo planes."""
    from mlx_audio_b200 import ops
    cw = ops.pack_conv(w, bias, 1, DEV)
    assert cw.w_tc is not None
    assert cw.f16 == (kind == "fp16")
    assert cw.w_tc.dtype == (torch.float16 if kind == "fp16" else torch.bfloat16)
    assert (cw.w_tc_lo is not None) == (kind == "fp32")
    return cw


@pytest.fixture
def mode():
    from mlx_audio_b200 import ops
    old = ops.TC_MODE[0]

    def set_mode(m):
        ops.TC_MODE[0] = m
    yield set_mode
    ops.TC_MODE[0] = old


@pytest.fixture
def gemm_tc():
    """Route every dense layer through the pre-split planes + conv_tc_kernel (csrc/gemm_tc.cu)."""
    from mlx_audio_b200 import ops
    old, oldd = ops.FUSED[0], ops.FUSED_DISPATCH[0]
    ops.FUSED[0] = ops.FUSED_DISPATCH[0] = False
    yield
    ops.FUSED[0], ops.FUSED_DISPATCH[0] = old, oldd


@pytest.fixture(params=["gemm_tc", "fused"])
def path(request):
    """Both tensor-core kernels: the prologue pass + conv_tc_kernel, and the fused kernel that converts the activations itself."""
    from mlx_audio_b200 import ops
    old, oldd = ops.FUSED[0], ops.FUSED_DISPATCH[0]
    ops.FUSED[0] = ops.FUSED_DISPATCH[0] = request.param == "fused"
    yield request.param
    ops.FUSED[0], ops.FUSED_DISPATCH[0] = old, oldd


# ------------------------------------------------------------------------------------------------------------ N tiles of conv_tc_kernel
# (name, B, row tiles per batch row, Cout, N tile).  The wide cases are sized from the SM count so that the grid at the widest divisor
# of Cout covers at least half the SMs (the dispatch keeps that tile); the narrow ones leave most SMs idle and take 32-wide tiles.
def _tile_cases(nsm):
    return [
        ("bn128", 1, -(-nsm // 4), 256, 128),          # 2 N tiles
        ("bn128_b2", 2, -(-nsm // 8), 256, 128),
        ("bn96", 1, -(-nsm // 6), 288, 96),            # 3 N tiles
        ("bn64", 1, -(-nsm // 10), 320, 64),           # 5 N tiles
        ("bn32", 1, 3, 256, 32),
        ("bn32_b2", 2, 2, 320, 32),
    ]


TILE_NAMES = ["bn128", "bn128_b2", "bn96", "bn64", "bn32", "bn32_b2"]


@pytest.mark.parametrize("K,dil", [(1, 1), (5, 3)])
@pytest.mark.parametrize("name", TILE_NAMES)
def test_conv_tc_n_tiles_vs_float64(name, K, dil, gemm_tc, mode):
    """Every N tile of conv_tc_kernel, ragged last row tile, 1 and 5 dilated taps, bias + GELU + residual + out_scale epilogue."""
    from mlx_audio_b200 import ops
    _, B, tiles, Cout, bn = next(c for c in _tile_cases(_nsm()) if c[0] == name)
    L, Cin, pad = _rows(tiles), 160, (K - 1) * dil // 2
    x = _rand(B, L, Cin, seed=1)
    w = _weights("bf16", Cout, K, Cin, seed=2)
    bias = _rand(Cout, seed=3, scale=0.1)
    res = _rand(B, L, Cout, seed=4, scale=0.1)
    ref = (ON.gelu(ON.conv1d(x.double(), w.double(), 1, pad, dil, 1, bias.double())) + res.double()) * 0.5
    cw = _pack("bf16", w, bias)
    mode("x2")
    y = ops.conv1d(x.to(DEV), cw, dilation=dil, pad_left=pad, post_act=ops.ACT["gelu"], res=res.to(DEV), out_scale=0.5)
    cfg = ops.conv1d_tc_last_config()
    assert cfg["BN"] == bn and cfg["grid"] == (tiles, Cout // bn, B), cfg
    e = rel_err(y, ref)
    print(f"\n[n-tile] {name} BN {bn} K {K}: {e:.2e}")
    assert e < TOL_X2, e


def _bit_identity_case(ops, x, conv, ctas_at_128):
    """conv(x) at B = 1 (32-wide N tiles) and on x replicated to enough batch rows that the grid at 128-wide tiles covers half the SMs
    (``ctas_at_128``: CTAs per batch row at that tile): equal bits."""
    narrow = conv(x)
    assert ops.conv1d_tc_last_config()["BN"] == 32
    nb = -(-_nsm() // (2 * ctas_at_128))
    wide = conv(x.expand(nb, *x.shape[1:]).contiguous())
    assert ops.conv1d_tc_last_config()["BN"] == 128
    for b in range(nb):
        assert torch.equal(wide[b], narrow[0]), b


@pytest.mark.parametrize("tc_mode", ["x2", "x1"])
@pytest.mark.parametrize("kind", ["bf16", "fp16", "fp32"])
def test_conv_tc_bit_identical_across_n_tiles(kind, tc_mode, gemm_tc, mode):
    """Each output element sums its whole K range in one CTA in the same order whatever the tile: B = 1 (3 row tiles, 32-wide) equals
    every row of a batch wide enough for 128-wide tiles, for every weight kind and activation mode."""
    from mlx_audio_b200 import ops
    L, Cin, Cout = 300, 160, 256
    w = _weights(kind, Cout, 3, Cin, seed=5)
    cw = _pack(kind, w, _rand(Cout, seed=6, scale=0.1))
    res = _rand(1, L, Cout, seed=7).to(DEV)
    mode(tc_mode)

    def conv(x):
        return ops.conv1d(x, cw, pad_left=1, post_act=ops.ACT["gelu"], res=res.expand(x.shape[0], L, Cout).contiguous(), out_scale=0.5)
    _bit_identity_case(ops, _rand(1, L, Cin, seed=8).to(DEV), conv, 3 * (Cout // 128))


def test_convtr_tc_bit_identical_across_n_tiles(gemm_tc, mode):
    """The polyphase transposed mode (N = stride * Cout columns scattered to stride output phases) likewise."""
    from mlx_audio_b200 import ops
    L, Cin, Cout, K, stride, pad = 100, 128, 64, 8, 4, 2
    w, bias = _weights("bf16", Cout, K, Cin, seed=9), _rand(Cout, seed=10, scale=0.1)
    cw = _pack("bf16", w, bias)
    mode("x2")

    def conv(x):
        return ops.conv1d(x, cw, stride=stride, pad_left=pad, transpose=True, pre=ops.Pre(act=ops.ACT["lrelu"], p0=0.1))
    x = _rand(1, L, Cin, seed=11)
    ref = ON.conv_transpose1d(ON.leaky_relu(x.double(), 0.1), w.double(), stride, pad, 1, 0, 1, bias.double())
    x = x.to(DEV)
    assert rel_err(conv(x), ref) < TOL_X2
    _bit_identity_case(ops, x, conv, 1 * (stride * Cout // 128))     # 1 row tile (L + taps - 1 = 101 rows)


# ------------------------------------------------------------------------------------------------ weight precision x activation planes
PREC_SHAPE = (1, 300, 160, 128, 3)          # B, L, Cin, Cout, K: three K chunks, 32 pad channels, ragged last row tile


def _prec_case(kind, seed=20):
    B, L, Cin, Cout, K = PREC_SHAPE
    x = _rand(B, L, Cin, seed=seed)
    w = _weights(kind, Cout, K, Cin, seed=seed + 1)
    bias = _rand(Cout, seed=seed + 2, scale=0.1)
    ref = ON.conv1d(x.double(), w.double(), 1, 1, 1, 1, bias.double())
    return x, w, bias, ref


def _run(ops, path, x, cw):
    if path == "fused":
        assert ops.fused_eligible(x, cw, 1, 1)
    return ops.conv1d(x, cw, pad_left=1)


@pytest.mark.parametrize("kind", ["bf16", "fp16", "fp32"])
def test_weight_precision_vs_float64(kind, path, mode):
    """x2 is fp32-grade for every weight kind on both kernels; x1 within its plane's rounding; each dropped product is caught."""
    from mlx_audio_b200 import ops
    x, w, bias, ref = _prec_case(kind)
    cw = _pack(kind, w, bias)
    xd = x.to(DEV)
    mode("x2")
    e2 = rel_err(_run(ops, path, xd, cw), ref)
    mode("x1")
    e1 = rel_err(_run(ops, path, xd, cw), ref)
    msg = f"\n[precision] {path} {kind}: x2 {e2:.2e} x1 {e1:.2e}"
    assert e2 < TOL_X2, msg
    assert e1 < TOL_X1[kind], msg
    assert e1 > 5 * TOL_X2, msg                          # negative control: without the activation lo plane
    if kind == "fp32":
        mode("x2")
        e_nolo = rel_err(_run(ops, path, xd, dataclasses.replace(cw, w_tc_lo=None)), ref)
        msg += f" x2 without w_lo {e_nolo:.2e}"
        assert e_nolo > 5 * TOL_X2, msg                  # negative control: without the a_hi * w_lo product
    print(msg)


@pytest.mark.parametrize("kind", ["fp16", "fp32"])
def test_fused_split_k_vs_float64(kind, mode):
    """Decoder-sized layer (390 rows, 1090 -> 1024, k = 3): few output tiles, so the fused kernel splits K across CTAs and sums the
    partial tiles in its fix-up; with 16-bit-exact and split weights."""
    from mlx_audio_b200 import ops
    B, L, Cin, Cout, K = 1, 390, 1090, 1024, 3
    x = _rand(B, L, Cin, seed=30)
    w = _weights(kind, Cout, K, Cin, seed=31)
    bias = _rand(Cout, seed=32, scale=0.1)
    res = _rand(B, L, Cout, seed=33, scale=0.1)
    ref = ON.conv1d(x.double(), w.double(), 1, 1, 1, 1, bias.double()) + res.double()
    cw = _pack(kind, w, bias)
    xd = torch.zeros(B, L, Cin + 2, device=DEV)[:, :, :Cin]      # rows padded to 16 bytes, as the decoder's channel slices are
    xd.copy_(x)
    rd = res.to(DEV)
    errs = {}
    for m in ("x2", "x1"):
        mode(m)
        y = ops.conv_fused(ops.FusedProblem(xd, cw, pad_left=1, res=rd))[0]
        cfg = ops.conv1d_fused_last_config()
        assert cfg["BN"] == [128] and cfg["ksplit"][0] > 1, cfg
        errs[m] = rel_err(y, ref)
    if kind == "fp32":
        mode("x2")
        errs["x2 without w_lo"] = rel_err(ops.conv_fused(ops.FusedProblem(xd, dataclasses.replace(cw, w_tc_lo=None), pad_left=1, res=rd))[0], ref)
    print(f"\n[fused split-K] {kind} ksplit {cfg['ksplit'][0]}: {errs}")
    assert errs["x2"] < TOL_X2 and TOL_X1[kind] > errs["x1"] > 5 * TOL_X2, errs
    if kind == "fp32":
        assert errs["x2 without w_lo"] > 5 * TOL_X2, errs


def test_fused_group_split_weights_vs_float64(mode):
    """One grouped launch of two fp32-checkpoint problems on the same input (a k = 3 conv and its 1x1 shortcut, as in the decoder
    blocks): each problem against float64, K split, and the weight lo planes present in both."""
    from mlx_audio_b200 import ops
    B, L, Cin, Cout = 1, 390, 512, 256
    x = _rand(B, L, Cin, seed=40)
    w3, w1 = _weights("fp32", Cout, 3, Cin, seed=41), _weights("fp32", Cout, 1, Cin, seed=42)
    b3, b1 = _rand(Cout, seed=43, scale=0.1), _rand(Cout, seed=44, scale=0.1)
    pre = ops.Pre(act=ops.ACT["lrelu"], p0=0.2)
    v = ON.leaky_relu(x.double(), 0.2)
    refs = [ON.conv1d(v, w3.double(), 1, 1, 1, 1, b3.double()), ON.conv1d(v, w1.double(), 1, 0, 1, 1, b1.double())]
    cws = [_pack("fp32", w3, b3), _pack("fp32", w1, b1)]
    xd = x.to(DEV)

    def run(c3, c1):
        outs = ops.conv_fused([ops.FusedProblem(xd, c3, pad_left=1, pre=pre), ops.FusedProblem(xd, c1, pre=pre)])
        return [rel_err(o, r) for o, r in zip(outs, refs)]
    mode("x2")
    e2 = run(*cws)
    cfg = ops.conv1d_fused_last_config()
    assert cfg["BN"] == [128, 128] and min(cfg["ksplit"]) > 1, cfg
    e_nolo = run(*[dataclasses.replace(c, w_tc_lo=None) for c in cws])
    mode("x1")
    e1 = run(*cws)
    print(f"\n[fused group] ksplit {cfg['ksplit']}: x2 {e2} x1 {e1} x2 without w_lo {e_nolo}")
    assert max(e2) < TOL_X2, e2
    assert all(TOL_X1["fp32"] > e > 5 * TOL_X2 for e in e1), e1
    assert all(e > 5 * TOL_X2 for e in e_nolo), e_nolo


# ------------------------------------------------------------------------------------------------------------------- fp16 dynamic range
# The fp16 lo plane a - fp16(a) is about 2^-11 |a|; below |a| ~ 2^-3 it falls into fp16 subnormals (absolute step 2^-24), so x2 loses
# accuracy as the input shrinks.  Over input RMS 2^-7 .. 2^10 it stays fp32-grade.
FP16_GRADE_MIN_LOG2, FP16_GRADE_MAX_LOG2 = -7, 10


def test_fp16_x2_dynamic_range(path, mode):
    from mlx_audio_b200 import ops
    x, w, bias, _ = _prec_case("fp16", seed=50)
    cw = _pack("fp16", w, None)
    mode("x2")
    errs = {}
    for e in range(-13, FP16_GRADE_MAX_LOG2 + 1):
        xs = x * 2.0 ** e
        ref = ON.conv1d(xs.double(), w.double(), 1, 1, 1, 1)
        errs[e] = rel_err(_run(ops, path, xs.to(DEV), cw), ref)
    print(f"\n[fp16 x2 range] {path}: " + " ".join(f"2^{e}:{v:.1e}" for e, v in errs.items()))
    bad = {e: v for e, v in errs.items() if e >= FP16_GRADE_MIN_LOG2 and v >= TOL_X2}
    assert not bad, bad


def test_whisper_fp16_layer_inputs_inside_fp32_grade_range(monkeypatch):
    """Every fp16 tensor-core layer of the Whisper encoder and decoder (synthetic checkpoint) sees inputs whose RMS lies in the range
    test_fp16_x2_dynamic_range shows to be fp32-grade."""
    from mlx_audio_b200 import ops, synth
    from mlx_audio_b200.stt.models.whisper import Model, ModelDimensions
    from oracle import whisper as OW
    seen = []
    prep = ops.prep_bf16

    def recording_prep(x, pre, cpad, planes=2, f16=False):
        if f16:
            assert pre is None                         # the planes hold x itself
            seen.append((tuple(x.shape), x.double().pow(2).mean().sqrt()))
        return prep(x, pre, cpad, planes, f16)
    monkeypatch.setattr(ops, "prep_bf16", recording_prep)
    dims = OW.WHISPER_SMALL
    enc = Model(ModelDimensions.from_dict(dims), device=DEV).load_weights(synth.whisper_encoder_weights(dims))
    xa = enc.encode_audio(synth.whisper_audio(1, 480000))
    n_enc = len(seen)
    ddims = dict(dims, n_text_layer=4)
    dec = Model(ModelDimensions.from_dict(ddims), device=DEV).load_weights(synth.whisper_decoder_weights(ddims))
    spec = OW.TokenizerSpec()
    dec.decoder(torch.tensor([list(spec.sot_sequence)]).to(DEV), dec.decoder.new_cache(xa))
    torch.cuda.synchronize()
    rms = [(s, float(r)) for s, r in seen]
    log2 = [math.log2(r) for _, r in rms]
    print(f"\n[whisper fp16 inputs] {n_enc} encoder + {len(rms) - n_enc} decoder layers, log2 RMS {min(log2):.2f} .. {max(log2):.2f}")
    assert n_enc > 0 and len(rms) > n_enc
    out = [(s, r) for s, r in rms if not FP16_GRADE_MIN_LOG2 <= math.log2(r) <= FP16_GRADE_MAX_LOG2]
    assert not out, out
