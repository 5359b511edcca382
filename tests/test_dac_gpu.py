"""Descript Audio Codec on the GPU against the float64 oracle (oracle/dac.py, itself pinned to the reference's code by tests/test_dac_pins.py):
released shapes (44.1 kHz / 9 code books, 24 kHz / 32 code books), synthetic weights."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import synth
from oracle import dac as OD

DEV = "cuda:0"


def rel_rms(a, b):
    a, b = torch.as_tensor(a).double().cpu().reshape(-1), torch.as_tensor(b).double().cpu().reshape(-1)
    return float(torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean()))


def _model(cfg, P=None):
    from mlx_audio_b200.codec import DAC
    P = synth.dac_weights(cfg, encoder=True) if P is None else P
    return DAC(**cfg, device=DEV).load_weights(P), {k: v.double() for k, v in P.items()}


@pytest.fixture(scope="module")
def dac44():
    return _model(OD.DAC_44K) + (OD.DAC_44K,)


@pytest.fixture(scope="module")
def dac24():
    return _model(OD.DAC_24K) + (OD.DAC_24K,)


@pytest.fixture(params=["44k", "24k"])
def dac(request, dac44, dac24):
    return dac44 if request.param == "44k" else dac24


@pytest.mark.parametrize("batch", [1, 2])
def test_decode_parity(dac, batch):
    model, P64, cfg = dac
    g = torch.Generator().manual_seed(11)
    codes = torch.randint(0, cfg["codebook_size"], (batch, cfg["n_codebooks"], 19), generator=g)
    zq, zp, _ = model.quantizer.from_codes(codes)
    ozq, ozp, _ = OD.from_codes(P64, codes, cfg)
    assert zq.shape == ozq.shape and zp.shape == ozp.shape
    assert rel_rms(zq, ozq) < 1e-5, rel_rms(zq, ozq)
    assert torch.equal(zp.cpu().double(), ozp)
    ref = OD.decode(P64, ozq, cfg)
    y = model.decode(zq)
    assert y.shape == ref.shape == (batch, OD.output_length(cfg, 19), 1)
    # 30 dense layers deep at 1536 channels, unit-gain random weights through bf16 hi / lo operand planes (~2^-16 per product): measured
    # 1.08e-3 on an H100 at both shapes and batch sizes (the depthwise SNAC decoder and the quarter-width round trip below stay under 1e-3)
    assert rel_rms(y, ref) < 2e-3, rel_rms(y, ref)
    y2 = model.decode(ozq.float())                                            # decode(z) on a given z
    assert rel_rms(y2, ref) < 2e-3, rel_rms(y2, ref)
    # a prefix of the code books, as the reference decodes fewer quantizers
    zq3 = model.quantizer.from_codes(codes[:, :3])[0]
    assert rel_rms(zq3, OD.from_codes(P64, codes[:, :3], cfg)[0]) < 1e-5


def test_reference_length_pins_and_bad_codes(dac44, dac24):
    for (model, _, cfg), frames, n_out in ((dac44, 430, 220_235), (dac24, 375, 120_043), (dac24, 250, 80_043)):
        codes = torch.randint(0, 1024, (1, cfg["n_codebooks"], frames), generator=torch.Generator().manual_seed(frames))
        z = model.quantizer.from_codes(codes)[0]
        assert z.shape == (1, 1024, frames)
        y = model.decode(z)
        assert y.squeeze(-1).shape == (1, n_out) and bool(torch.isfinite(y).all()) and float(y.abs().max()) <= 1.0
    model, _, cfg = dac44
    codes = torch.randint(0, 1024, (1, 9, 12), generator=torch.Generator().manual_seed(1))
    codes[0, 5, 3] = 1024
    with pytest.raises(ValueError):
        model.quantizer.from_codes(codes)
    with pytest.raises(ValueError):
        model.quantizer.from_codes(codes[:, :, :0].reshape(1, 0, 12))


def _quantizer_case(cfg, P, n_quantizers, batch, frames, seed=5):
    """The quantiser alone on a given latent: fused kernel and level-by-level route on the GPU, the oracle on the same z."""
    from mlx_audio_b200.codec.models import dac as M
    q = M.ResidualVectorQuantize(OD.latent_dim(cfg), cfg["n_codebooks"], cfg["codebook_size"], cfg["codebook_dim"], DEV)
    q._load(P)
    z = torch.randn(batch, OD.latent_dim(cfg), frames, generator=torch.Generator().manual_seed(seed))
    fused = q(z.to(DEV), n_quantizers)
    M.FUSED_RVQ[0] = False
    try:
        levels = q(z.to(DEV), n_quantizers)
    finally:
        M.FUSED_RVQ[0] = True
    P64 = {k: v.double() for k, v in P.items()}
    want = OD.quantize(P64, z.double(), cfg, n_quantizers, with_margin=True)
    return fused, levels, want, q


def _check_against_oracle(fused, levels, want):
    zq, codes, latents, closs, bloss = fused
    ozq, ocodes, olat, oloss, _, margins = want
    assert codes.shape == ocodes.shape and codes.dtype == torch.int64 and latents.shape == olat.shape and zq.shape == ozq.shape
    assert torch.equal(codes, levels[1]), f"fused and level-by-level codes differ on {int((codes != levels[1]).any(1).sum())} frames"
    assert torch.equal(zq, levels[0]) and torch.equal(latents, levels[2])
    clear = (margins > 1e-5).all(dim=1)                                       # [B, T]: frames decided by more than the fp32 error at every level
    frac = float(clear.float().mean())
    same = (codes.cpu() == ocodes).all(dim=1)
    assert bool(same[clear].all()) and frac >= 0.95, f"{int((~same & clear).sum())} clear frames differ; clear fraction {frac:.4f}"
    sel = clear[:, None, :]
    for name, a, b in (("z_q", zq, ozq), ("latents", latents, olat)):
        a, b = a.cpu().double(), b
        m = sel.expand_as(b)
        assert float((a - b)[m].abs().max() / b[m].abs().max()) < 1e-5, name
    if bool(clear.all()):
        assert abs(float(closs) - float(oloss)) < 1e-5 * float(oloss) and float(closs) == float(bloss)
    assert abs(float(levels[3]) - float(closs)) < 1e-5 * float(closs)


@pytest.mark.parametrize("n_quantizers", [None, 1, 3])
@pytest.mark.parametrize("which,batch,frames", [("44k", 1, 203), ("24k", 2, 117)])       # 203 and 234 rows: not multiples of the 8-frame tile
def test_quantizer_against_oracle_and_level_route(dac44, dac24, which, batch, frames, n_quantizers):
    _, P64, cfg = dac44 if which == "44k" else dac24
    P = {k: v.float() for k, v in P64.items() if k.startswith("quantizer.")}
    fused, levels, want, _ = _quantizer_case(cfg, P, n_quantizers, batch, frames)
    assert fused[1].shape == (batch, cfg["n_codebooks"] if n_quantizers is None else n_quantizers, frames)
    _check_against_oracle(fused, levels, want)


def test_quantizer_list_valued_codebook_dim_and_from_latents():
    cfg = dict(OD.DAC_44K, n_codebooks=4, codebook_dim=[8, 4, 16, 12], decoder_dim=32)
    P = {k: v for k, v in synth.dac_weights(cfg, encoder=True).items() if k.startswith("quantizer.")}
    fused, levels, want, q = _quantizer_case(cfg, P, None, 2, 61)
    assert fused[2].shape == (2, 40, 61)
    _check_against_oracle(fused, levels, want)
    zq, zp, codes = q.from_latents(fused[2])
    assert torch.equal(codes, fused[1])
    P64 = {k: v.double() for k, v in P.items()}
    ozq, ozp, _ = OD.from_latents(P64, fused[2].cpu().double(), cfg)
    assert rel_rms(zq, ozq) < 1e-5 and zp.shape == ozp.shape
    zq2, _, codes2 = q.from_latents(fused[2][:, :13])                          # 8 + 4 channels and one more: two code books
    assert codes2.shape == (2, 2, 61) and torch.equal(codes2, fused[1][:, :2])
    # a codebook_dim that the level-by-level route's search kernel does not take still runs fused
    from mlx_audio_b200.codec.models import dac as M
    cfg6 = dict(cfg, n_codebooks=2, codebook_dim=[6, 3])
    P6 = {k: v for k, v in synth.dac_weights(cfg6, encoder=True).items() if k.startswith("quantizer.")}
    q6 = M.ResidualVectorQuantize(1024, 2, 1024, [6, 3], DEV)
    q6._load(P6)
    z = torch.randn(1, 1024, 30, generator=torch.Generator().manual_seed(2))
    got = q6(z.to(DEV))
    want = OD.quantize({k: v.double() for k, v in P6.items()}, z.double(), cfg6, with_margin=True)
    clear = (want[5] > 1e-5).all(dim=1)
    assert bool((got[1].cpu() == want[1]).all(dim=1)[clear].all()) and float(clear.float().mean()) >= 0.9


def test_quantizer_exact_tie_takes_the_lower_index(dac44):
    _, P64, cfg = dac44
    P = {k: v.float().clone() for k, v in P64.items() if k.startswith("quantizer.")}
    cb = P["quantizer.quantizers.0.codebook.weight"]
    cb[512:] = cb[:512]                                                        # every row of the first code book exists twice
    fused, levels, want, _ = _quantizer_case(cfg, P, 2, 2, 50)
    assert int(fused[1][:, 0].max()) < 512 and torch.equal(fused[1], levels[1])
    assert float((fused[1][:, 0].cpu() == want[1][:, 0]).float().mean()) >= 0.95


@pytest.mark.parametrize("n", [8000])
def test_encode_matches_the_oracle(dac, n):
    model, P64, cfg = dac
    audio = torch.randn(2, 1, n, generator=torch.Generator().manual_seed(3)) * 0.3
    x = model.preprocess(audio, cfg["sample_rate"])
    frames = math.ceil(n / OD.hop(cfg))
    z = model.encode_latent(x)
    z_ref = OD.encoder(P64, OD.preprocess(audio.double(), cfg).transpose(1, 2), cfg)
    assert z.shape == z_ref.shape == (2, frames, 1024)
    # max-norm error of the latent: measured 2.1e-4 (44.1 kHz) and 2.4e-4 (24 kHz) on an H100 -- the dense k7 stack lets the split-plane
    # rounding grow a little past the 2e-4 the depthwise SNAC encoder keeps
    err = float((z.double().cpu() - z_ref).abs().max() / z_ref.abs().max())
    assert err < 5e-4, err
    zq, codes, latents, closs, bloss = model.encode(x)
    want = OD.quantize(P64, z_ref.transpose(1, 2), cfg)
    assert zq.shape == (2, 1024, frames) and codes.shape == (2, cfg["n_codebooks"], frames) and latents.shape == (2, 8 * cfg["n_codebooks"], frames)
    assert float((codes[:, 0].cpu() == want[1][:, 0]).float().mean()) >= 0.9
    assert int(codes.min()) >= 0 and int(codes.max()) < 1024 and float(closs) == float(bloss) > 0
    assert torch.equal(model.quantizer.from_latents(latents)[2], codes)
    r = model(audio, cfg["sample_rate"], 3)
    assert r["codes"].shape == (2, 3, frames) and r["audio"].shape == (2, OD.output_length(cfg, frames), 1) and torch.equal(r["codes"], codes[:, :3])
    from mlx_audio_b200.codec import DAC
    with pytest.raises(ValueError):
        DAC(**cfg, device=DEV).load_weights(synth.dac_weights(cfg, encoder=False)).encode(x)


def test_compress_decompress_round_trip(tmp_path):
    """3.3 s in 1 s windows: four windows, the last one zero-padded.  The released 44.1 kHz rates and code books at a quarter of the
    width, which keeps the float64 oracle's decode of 348 frames to seconds; the full-width kernels are covered above."""
    from mlx_audio_b200.codec import DACFile
    cfg = dict(OD.DAC_44K, encoder_dim=16, decoder_dim=384)
    model, P64 = _model(cfg)
    sr = cfg["sample_rate"]
    g = torch.Generator().manual_seed(9)
    audio = 0.05 * torch.randn(int(3.3 * sr), generator=g)
    f = model.compress(audio, win_duration=1.0)
    win = OD.window_samples(cfg, 1.0)
    assert win == 44544 and f.chunk_length == 87 and f.codes.shape == (1, 9, 4 * 87) and f.padding is False and f.sample_rate == sr
    assert abs(f.original_length - audio.numel() / sr) < 1e-12
    input_db = float(20 * torch.log10(torch.sqrt((audio.double() ** 2).mean() + 1e-12) + 1e-12))
    assert abs(f.input_db - input_db) < 1e-4
    scaled = audio * float(10.0 ** ((-16 - f.input_db) / 20))
    padded = torch.nn.functional.pad(scaled, (0, 4 * win - scaled.numel()))
    one_by_one = torch.cat([model.encode(padded[i * win:(i + 1) * win].reshape(1, 1, -1))[1] for i in range(4)], dim=-1)
    assert torch.equal(f.codes, one_by_one)
    g2 = DACFile.load(f.save(tmp_path / "clip"))
    assert torch.equal(g2.codes, f.codes.cpu()) and g2.chunk_length == 87
    y = model.decompress(g2)
    ref = OD.decompress(P64, {"codes": f.codes.cpu(), "chunk_length": 87, "input_db": f.input_db}, cfg)
    assert y.shape == ref.shape == (1, 4 * OD.output_length(cfg, 87))
    assert rel_rms(y, ref) < 1e-3
    assert torch.equal(model.decompress(f), y)
    # shorter than the window: one padded window, n_quantizers respected
    f1 = model.compress(audio[:30000].numpy(), win_duration=1.0, n_quantizers=4)
    assert f1.padding is True and f1.codes.shape == (1, 4, math.ceil(30000 / 512)) and f1.chunk_length == f1.codes.shape[-1]
    with pytest.raises(NotImplementedError):
        model.compress("clip.wav")


def test_constructor_leaves_a_usable_model():
    """The body of the reference's test_descript_16khz (codec/tests/test_descript.py) with tensors for mx.arrays."""
    from mlx_audio.codec import DAC
    model = DAC(encoder_dim=64, encoder_rates=[2, 4, 5, 8], decoder_dim=1536, decoder_rates=[8, 5, 4, 2], n_codebooks=12, codebook_size=1024,
                codebook_dim=8, sample_rate=16_000)
    x = model.preprocess(torch.zeros(1, 1, 80_000), 16_000)
    z, codes, latents, _, _ = model.encode(x)
    assert z.shape == (1, 1024, 250) and codes.shape == (1, 12, 250) and latents.shape == (1, 96, 250)
    assert model.decode(z).squeeze(-1).shape == (1, 80_043)
