"""Vocos, CPU side: the float64 oracle against the fixture made from the reference's own code, the reference's shape pins, sanitize,
the import paths its callers use, the exported C symbols, and what ptxas makes of the new kernels and the re-templated log-mel kernel."""
import importlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from mlx_audio_b200 import build
from oracle import vocos as OV

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import synth_params  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "vocos_golden.npz")
HAVE_REFERENCE = os.path.isdir("/root/reference/mlx_audio")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _close(a, b, what):
    a = a.numpy() if hasattr(a, "numpy") else np.asarray(a)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.abs(a - b).max(initial=0.0) <= 1e-12 * max(1.0, float(np.abs(b).max(initial=0.0))), what


def _params(golden, tag):
    return {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(golden[f"{tag}_params"]).items()}


def test_log_mel_matches_the_reference(golden):
    for n, m in golden["lm_cases"]:
        y = OV.log_mel_spectrogram(golden[f"lm_audio{n}_{m}"], n_mels=int(m))
        assert y.shape == (1, n // 256, m)
        _close(y, golden[f"lm_mel{n}_{m}"], f"n={n} n_mels={m}")


def test_mel_model_and_default_gamma(golden):
    cfg = json.loads(str(golden["mel_cfg"]))
    P = _params(golden, "mel")
    names = json.loads(str(golden["mel_gamma_names"]))
    a = OV.backbone_args(cfg)
    assert len(names) == a["num_layers"] and np.all(golden["mel_gamma_values"] == OV.default_gamma(a))
    assert not any(k.endswith(".gamma") for k in P)                     # the oracle fills the constructor's gamma itself
    for k, v in zip(names, golden["mel_gamma_values"]):
        P[k] = torch.as_tensor(v)
    y = OV.forward(P, golden["mel_audio"], cfg)[0]
    assert y.shape == (OV.output_length(cfg, n_samples=len(golden["mel_audio"])),)
    _close(y, golden["mel_wave"], "mel Vocos")


def test_adaln_backbone_per_row_conditions(golden):
    cfg = json.loads(str(golden["ada_cfg"]))
    P = _params(golden, "ada")
    assert "backbone.final_layer_norm.bias" not in P                   # bias=False
    h = OV.backbone(P, golden["ada_x"], cfg, golden["ada_cond"])
    _close(h, golden["ada_h"], "AdaLN backbone, B = 2")
    assert not np.allclose(golden["ada_h"][0], golden["ada_h"][1])
    _close(OV.decode(P, golden["ada_x"][:1], cfg, golden["ada_cond"][:1])[0], golden["ada_wave0"], "decode row 0")


@pytest.mark.parametrize("n_fft,hop", [(1024, 256), (1280, 320)])
def test_istft_head(golden, n_fft, hop):
    P = _params(golden, f"head{n_fft}")
    for T in golden["head_T"]:
        y = OV.head(P, golden[f"head{n_fft}_x{T}"], n_fft, hop)[0]
        assert y.shape == ((T - 1) * hop,)
        _close(y, golden[f"head{n_fft}_y{T}"], f"T={T}")
    _, clipped = OV.head_spectrum(P, golden[f"head{n_fft}_xclip"], n_fft)
    assert clipped > 0.3, clipped
    _close(OV.head(P, golden[f"head{n_fft}_xclip"], n_fft, hop)[0], golden[f"head{n_fft}_yclip"], "clipped")


def test_from_pretrained_remap(golden):
    from mlx_audio_b200.codec import Vocos
    keys_in, keys_out = json.loads(str(golden["pre_in_keys"])), json.loads(str(golden["pre_out_keys"]))
    ckpt = {k: torch.as_tensor(golden[f"pre_in_{i}"]) for i, k in enumerate(keys_in)}
    for new in (OV.sanitize(ckpt), Vocos.sanitize(ckpt)):
        for i, k in enumerate(keys_out):
            assert torch.equal(torch.as_tensor(new[k]), torch.as_tensor(golden[f"pre_out_{i}"])), k
        assert "head.istft.window" not in new and "feature_extractor.mel_spec.spectrogram.window" not in new
        assert set(new) - set(keys_out) == {"feature_extractor.encodec.quantizer.x"}       # ignored by the non-strict load
    np_new = Vocos.sanitize({k: v.numpy() for k, v in ckpt.items()})
    assert all(np.array_equal(np_new[k], golden[f"pre_out_{i}"]) for i, k in enumerate(keys_out))
    only_head = Vocos.sanitize({"head.istft.window": ckpt["head.istft.window"]})             # one try: nothing dropped
    assert "head.istft.window" in only_head


def test_model_parameter_tree_matches_the_reference(golden):
    """The keys and shapes the model loads are exactly the reference's parameter tree."""
    from mlx_audio_b200.codec.models.vocos import ISTFTHead, VocosBackbone
    cfg = json.loads(str(golden["pre_cfg"]))
    ours = {**VocosBackbone(**cfg["backbone"]["init_args"], device="cpu").param_shapes(),
            **ISTFTHead(**cfg["head"]["init_args"], device="cpu").param_shapes()}
    keys_out = json.loads(str(golden["pre_out_keys"]))
    assert sorted(ours) == keys_out
    for i, k in enumerate(keys_out):
        assert tuple(golden[f"pre_out_{i}"].shape) == ours[k], k


def test_reference_shape_pins(golden):
    """codec/tests/test_vocos.py: 120 000 samples -> 119 552 (mel), 375 EnCodec-config frames -> 119 680."""
    assert tuple(golden["pin_mel_shape"]) == (119552,) == (OV.output_length(OV.CONFIG_MEL, n_samples=120_000),)
    assert tuple(golden["pin_encodec_shape"]) == (119680,) == (OV.output_length(OV.CONFIG_ENCODEC, frames=375),)


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference source is only present in the build container")
def test_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_vocos_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-2000:]
    new, old = np.load(tmp_path / "vocos_golden.npz"), np.load(GOLDEN)
    assert sorted(new.files) == sorted(old.files)
    for k in old.files:
        a, b = new[k], old[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        if a.dtype.kind == "f":
            assert np.abs(a - b).max(initial=0.0) <= 1e-12 * max(1.0, float(np.abs(b).max(initial=0.0))), k
        else:
            assert np.array_equal(a, b), k


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference source is only present in the build container")
def test_oracle_agrees_with_the_reference_code_on_random_configurations():
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_vocos_golden.py"), "--live", "6"], cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="4"), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "LIVE OK" in r.stdout, (r.stdout[-1500:], r.stderr[-1500:])


def test_product_configs_match_the_oracle_configs():
    from mlx_audio_b200 import configs as C
    assert C.VOCOS_MEL_24K == OV.CONFIG_MEL and C.VOCOS_ENCODEC_24K == OV.CONFIG_ENCODEC


def test_import_paths():
    from mlx_audio_b200.codec import Vocos, VocosBackbone
    from mlx_audio_b200.codec.models import vocos as V
    assert V.Vocos is Vocos and V.VocosBackbone is VocosBackbone
    for mod in ("mlx_audio.codec", "mlx_audio.codec.models"):
        assert importlib.import_module(mod).Vocos is Vocos, mod
    m = importlib.import_module("mlx_audio.codec.models.vocos")
    assert m.Vocos is Vocos and m.VocosBackbone is VocosBackbone
    m = importlib.import_module("mlx_audio.codec.models.vocos.vocos")
    for name in ("Vocos", "VocosBackbone", "ISTFTHead", "MelSpectrogramFeatures", "log_mel_spectrogram"):
        assert getattr(m, name) is getattr(V, name), name
    assert importlib.import_module("mlx_audio.codec.models.vocos.mel").log_mel_spectrogram is V.log_mel_spectrogram


def test_unsupported_configurations_raise_on_the_host():
    from mlx_audio_b200.codec.models.vocos import MelSpectrogramFeatures, Vocos
    with pytest.raises(NotImplementedError):
        MelSpectrogramFeatures(n_fft=2048, hop_length=512, device="cpu")
    with pytest.raises(ValueError):
        MelSpectrogramFeatures(padding="valid", device="cpu")
    m = Vocos.from_hparams(OV.CONFIG_ENCODEC, device="cpu")
    for call in (lambda: m(torch.zeros(4000), bandwidth_id=[3, 3, 3, 3]), lambda: m.get_encodec_codes(torch.zeros(4000), 3),
                 lambda: m.decode_from_codes(torch.zeros(8, 1, 10, dtype=torch.long))):
        with pytest.raises(NotImplementedError):
            call()


def test_symbols_exported_and_declared():
    from mlx_audio_b200 import _lib
    header = open(os.path.join(ROOT, "include", "b200audio.h")).read()
    for sym in ("b2a_vocos_dwnorm", "b2a_vocos_istft_head", "b2a_vocos_logmel"):
        assert re.search(rf"\b{sym}\s*\(", header), sym
        assert sym in _lib.PROTOTYPES and getattr(_lib.lib(), sym) is not None, sym


def test_ptxas_no_spills(tmp_path):
    assert "vocos.cu" in build.SOURCES
    obj = str(tmp_path / "vocos.o")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "vocos.cu"), "-o", obj], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    props = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    for k, n in (("vocos_dwnorm_kernel", 4), ("vocos_istft_head_kernel", 1), ("spk_logmel_kernelILi512ELb0", 1)):
        hits = [(int(s), int(l)) for name, s, l in props if k in name]
        assert hits == [(0, 0)] * n, (k, hits)
