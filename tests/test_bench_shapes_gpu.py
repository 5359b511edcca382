"""Parity at the shapes the benchmarks time (VERDICT r01: "make the benched shapes the tested shapes").  The float64 oracle takes
seconds to minutes at these sizes, so its outputs are cached in tests/golden/bench_shapes_golden.npz (make_bench_shape_golden.py; the
Kokoro cfg2 case lives in test_kokoro_gpu.py).  Inputs are rebuilt from ``mlx_audio_b200.synth`` with the generator's seeds."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import synth
from mlx_audio_b200.configs import MIMI_202407, SNAC_24K, WHISPER_SMALL

WIN = 16384


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "bench_shapes_golden.npz"))


def _windows(n):
    return [0, (n // 2 // 128) * 128, n - WIN]


def _check_windows(y, g, tag, tol=1e-3):
    y = y.reshape(-1).double().cpu()
    assert y.numel() == int(g[f"{tag}_len"])
    rms = float(np.sqrt(g[f"{tag}_ms"]))
    assert abs(float(torch.sqrt((y ** 2).mean())) / rms - 1.0) < 1e-3                       # global level of the whole stream
    for i, s in enumerate(_windows(y.numel())):
        want = torch.as_tensor(g[f"{tag}_win{i}"]).double()
        err = float(torch.sqrt(((y[s:s + WIN] - want) ** 2).mean())) / rms
        assert err < tol, (tag, i, err)


def test_snac_2048_frames_multi_wave_persistent_path(g):
    """SNAC-24k, 2 048 fine frames -> 1 048 651 samples: the last decoder layers have 8 000+ output tiles (many waves of the
    wgmma conv kernel, the staged depthwise kernel's interior path)."""
    from mlx_audio_b200.codec import SNAC
    model = SNAC.from_config(SNAC_24K, device="cuda:0").load_weights(synth.snac_weights(SNAC_24K))
    y = model.decode(synth.snac_codes(SNAC_24K, 2048, 1), noises=synth.snac_noises(SNAC_24K, 1))
    _check_windows(y, g, "snac")


def test_mimi_2000_frames(g):
    """Mimi, 2 000 frames -> 3 840 000 samples (4 000 transformer positions against the 250-position window)."""
    from mlx_audio_b200.codec import Mimi, mimi_202407
    model = Mimi(mimi_202407(32), device="cuda:0").load_weights(synth.mimi_weights(MIMI_202407))
    y = model.decode(synth.mimi_codes(MIMI_202407, 2000, 1))
    _check_windows(y, g, "mimi")


def test_whisper_full_12_layer_decoder(g):
    """Whisper-small TextDecoder with all 12 layers (BASELINE config 3's model): first-position logits 1e-3 of the logit scale, 8 greedy
    tokens identical, log-probabilities and no-speech probabilities."""
    from mlx_audio_b200.stt.models.whisper import Model, ModelDimensions
    from mlx_audio_b200.stt.models.whisper.whisper import TokenizerSpec
    dims = dict(WHISPER_SMALL)
    model = Model(ModelDimensions.from_dict(dims), device="cuda:0").load_weights(synth.whisper_decoder_weights(dims))
    xa = torch.randn(2, 1500, 768, generator=torch.Generator().manual_seed(0))
    spec = TokenizerSpec(suppress=(11, 12))
    tok0 = torch.tensor([list(spec.sot_sequence)] * 2)
    logits = model.decoder(tok0.cuda(), model.decoder.new_cache(xa))
    want = torch.as_tensor(g["whisper_logits"]).double()
    assert float((logits.double().cpu() - want).abs().max() / want.abs().max()) < 1e-3
    tokens, lp, ns = model.greedy_decode(xa, spec, sample_len=8)
    assert tokens == g["whisper_tokens"].tolist()
    assert torch.allclose(lp.cpu().double(), torch.as_tensor(g["whisper_sum_logprobs"]), rtol=1e-3, atol=1e-3)
    assert torch.allclose(ns.cpu().double(), torch.as_tensor(g["whisper_no_speech"]), rtol=1e-2, atol=1e-30)


def test_qwen3_full_model_25_frames(g):
    """Qwen3-TTS-0.6B talker + code predictor (28 + 5 layers), 25 frames x 16 code books with injected uniforms: every sampled code
    equals the oracle's (bit-exact index work), first-frame talker logits 2e-4."""
    from test_qwen3_gpu import _talker
    model, Pt, flat = _talker({})
    ids = g["qwen3_ids"].tolist()
    got = model.prepare_generation_inputs_from_ids(ids, language_id=2050, speaker_id=2100)
    u = torch.rand(25, 16, generator=torch.Generator().manual_seed(2))
    codes = model.generate_codes(*got, max_tokens=25, u=u[:, :, None])
    want = torch.as_tensor(g["qwen3_codes"])
    assert codes.shape[1] >= want.shape[0]
    assert torch.equal(codes[0, : want.shape[0]].cpu(), want), (codes[0, : want.shape[0]].cpu() != want).nonzero()[:5]
    model.talker.reset_cache(1, 64)
    lg, _ = model.talker(got[0])
    w0 = torch.as_tensor(g["qwen3_logits0"]).double()
    assert float((lg[0, -1].double().cpu() - w0).abs().max() / w0.abs().max()) < 2e-4
