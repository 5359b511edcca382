"""BigVGAN, CPU side: the float64 oracle against the fixture made from the reference's own code, the reference's shape pins, sanitize, the
import paths its callers use, the exported C symbol, and what ptxas makes of the anti-aliased activation kernel."""
import importlib
import json
import math
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from mlx_audio_b200 import build
from oracle import bigvgan as OB

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import synth_params  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "bigvgan_golden.npz")
HAVE_REFERENCE = os.path.isdir("/root/reference/mlx_audio")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _close(a, b, what):
    a = a.numpy() if hasattr(a, "numpy") else np.asarray(a)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.abs(a - b).max() <= 1e-12 * max(1.0, float(np.abs(b).max())), what


@pytest.mark.parametrize("tag", ["a", "b", "asym"])
def test_oracle_reproduces_the_reference(golden, tag):
    cfg = json.loads(str(golden[f"{tag}_cfg"]))
    P = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(golden[f"{tag}_params"]).items()}
    if tag == "asym":
        for name in json.loads(str(golden["asym_names"])):
            assert name in P and not torch.equal(P[name].reshape(-1), P[name].reshape(-1).flip(0))
    for T in (1, 2, 7):
        y = OB.forward(P, torch.as_tensor(golden[f"{tag}_mel{T}"]), cfg)
        assert y.shape == (2, 1, OB.output_length(cfg, T))
        _close(y, golden[f"{tag}_audio{T}"], f"{tag} T={T}")


def test_oracle_filters_are_the_constructors(golden):
    """The fixture's filters are the values the reference's constructor computes; the oracle's (and the model's) fall-back is the same."""
    f = OB.kaiser_sinc_filter1d(0.25, 0.3, 12).numpy()
    names, vals = json.loads(str(golden["filter_names"])), golden["filter_values"]
    assert len(names) == vals.shape[0] > 10 and all(n.endswith((".upsample.filter", ".downsample.lowpass.filter")) for n in names)
    assert np.abs(vals - f[None]).max() < 1e-15
    assert np.allclose(f, f[::-1], rtol=0, atol=1e-15) and abs(f.sum() - 1) < 1e-15      # symmetric: a flip would not show with them
    from mlx_audio_b200.codec.models.bigvgan import kaiser_sinc_filter1d
    assert torch.equal(kaiser_sinc_filter1d(0.25, 0.3, 12), torch.as_tensor(f))


def test_activation1d_alone(golden):
    from oracle.bigvgan import activation1d
    P = {"x.act.alpha": torch.as_tensor(golden["act_alpha"]), "x.act.beta": torch.as_tensor(golden["act_beta"])}
    _close(torch.as_tensor(golden["act_f_up"]).reshape(-1), OB.kaiser_sinc_filter1d(0.25, 0.3, 12).numpy(), "f_up")
    for L in golden["act_lengths"]:
        _close(activation1d(P, "x", torch.as_tensor(golden[f"act_x{L}"]), True), golden[f"act_y{L}"], f"L={L}")
    P["x.upsample.filter"] = torch.as_tensor(golden["act_asym_f_up"])
    P["x.downsample.lowpass.filter"] = torch.as_tensor(golden["act_asym_f_down"])
    _close(activation1d(P, "x", torch.as_tensor(golden["act_asym_x"]), True), golden["act_asym_y"], "non-symmetric filters")


def test_reference_snake_fails_when_t_differs_from_c(golden):
    assert str(golden["snake_raises"]) == "ValueError"
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    with pytest.raises(NotImplementedError):
        BigVGAN(BigVGANConfig(**dict(OB.BIGVGAN_22K, activation="snake")), device="cpu")


@pytest.mark.parametrize("cfg,hop", [(OB.BIGVGAN_22K, 256), (OB.BIGVGAN_44K, 512)], ids=["22k", "44k"])
def test_reference_shape_pins(cfg, hop):
    """codec/tests/test_bigvgan.py: 800 mel frames -> 800 * prod(upsample_rates) samples."""
    assert math.prod(cfg["upsample_rates"]) == hop
    assert OB.output_length(cfg, 800) == 800 * hop


def test_sanitize_matches_the_reference(golden):
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    cfg = json.loads(str(golden["a_cfg"]))
    model = BigVGAN(BigVGANConfig(**cfg), device="cpu")
    keys_in, keys_out = json.loads(str(golden["san_in_keys"])), json.loads(str(golden["san_out_keys"]))
    ckpt = {k: torch.as_tensor(golden[f"san_in_{i}"]) for i, k in enumerate(keys_in)}
    new = model.sanitize(ckpt)
    assert list(new) == keys_out and "conv_pre.num_batches_tracked" not in new
    for i, k in enumerate(keys_out):
        assert torch.equal(new[k], torch.as_tensor(golden[f"san_out_{i}"])), k
    from mlx_audio_b200.codec.models.bigvgan import param_shapes
    assert {k: tuple(v.shape) for k, v in new.items()} == param_shapes(BigVGANConfig(**cfg))
    np_new = model.sanitize({k: v.numpy() for k, v in ckpt.items()})                    # NumPy arrays take the same route
    assert all(np.array_equal(np_new[k], new[k].numpy()) for k in keys_out)


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference source is only present in the build container")
def test_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_bigvgan_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    new, old = np.load(tmp_path / "bigvgan_golden.npz"), np.load(GOLDEN)
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
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_bigvgan_golden.py"), "--live", "4"], cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="4"), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "LIVE OK" in r.stdout, (r.stdout[-1500:], r.stderr[-1500:])


def test_import_paths():
    from mlx_audio_b200.codec import BigVGAN, BigVGANConfig
    for mod in ("mlx_audio.codec.models.bigvgan", "mlx_audio.codec.models.bigvgan.bigvgan", "mlx_audio_b200.codec.models.bigvgan"):
        m = importlib.import_module(mod)
        assert m.BigVGAN is BigVGAN and m.BigVGANConfig is BigVGANConfig, mod


def test_symbol_exported_and_declared():
    from mlx_audio_b200 import _lib
    header = open(os.path.join(ROOT, "include", "b200audio.h")).read()
    assert re.search(r"\bb2a_aa_snakebeta\s*\(", header)
    assert "b2a_aa_snakebeta" in _lib.PROTOTYPES and _lib.lib().b2a_aa_snakebeta is not None


def test_ptxas_no_spills(tmp_path):
    obj = str(tmp_path / "bigvgan.o")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "bigvgan.cu"), "-o", obj], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    pat = re.compile(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                     r"ptxas info\s*: Used (\d+) registers")
    props = [m for m in pat.finditer(r.stdout) if "aa_snakebeta_kernel" in m.group(1)]
    assert len(props) == 1, r.stdout
    m = props[0]
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0, f"spills {m.group(2)} / {m.group(3)} bytes"
    assert 256 * int(m.group(4)) * 4 <= 65536, f"{m.group(4)} registers: fewer than four 256-thread CTAs per SM"
