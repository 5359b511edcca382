"""Descript Audio Codec, CPU side: the float64 oracle against the fixture made from the reference's own code, the reference's shape pins,
the import paths its callers use, the exported C symbols, and what ptxas makes of the two quantiser kernels."""
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
from oracle import dac as OD

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import synth_params  # noqa: E402

GOLDEN = os.path.join(HERE, "golden", "dac_golden.npz")
HAVE_REFERENCE = os.path.isdir("/root/reference/mlx_audio")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def _close(a, b, what):
    a = a.numpy() if hasattr(a, "numpy") else np.asarray(a)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.abs(a - b).max() <= 1e-12 * max(1.0, float(np.abs(b).max())), what


@pytest.mark.parametrize("tag", ["a", "b"])
def test_oracle_reproduces_the_reference(golden, tag):
    g = lambda k: golden[f"{tag}_{k}"]
    cfg = json.loads(str(g("cfg")))
    P = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g("params")).items()}
    assert int(g("delay")) == 0 and int(g("output_length")) == 1000
    audio = torch.as_tensor(g("audio"))
    z, codes, latents, closs, bloss = OD.encode(P, OD.preprocess(audio, cfg), cfg)
    assert np.array_equal(codes.numpy(), g("codes"))
    _close(z, g("z"), "z"); _close(latents, g("latents"), "latents")
    assert abs(float(closs) - float(g("closs"))) < 1e-12 and abs(float(bloss) - float(g("bloss"))) < 1e-12
    z2, codes2, latents2, closs2, _ = OD.encode(P, OD.preprocess(audio, cfg), cfg, 2)
    assert np.array_equal(codes2.numpy(), g("codes_nq2")) and abs(float(closs2) - float(g("closs_nq2"))) < 1e-12
    _close(z2, g("z_nq2"), "z nq2"); _close(latents2, g("latents_nq2"), "latents nq2")
    _close(OD.decode(P, z, cfg), g("decoded"), "decode")
    zq, zp, _ = OD.from_codes(P, codes[:, :2], cfg)
    _close(zq, g("fc2_zq"), "from_codes z_q"); _close(zp, g("fc2_zp"), "from_codes z_p")
    zq, zp, c = OD.from_latents(P, latents, cfg)
    assert np.array_equal(c.numpy(), g("fl_codes"))
    _close(zq, g("fl_zq"), "from_latents z_q"); _close(zp, g("fl_zp"), "from_latents z_p")
    zq, _, c = OD.from_latents(P, latents[:, :-1], cfg)
    assert np.array_equal(c.numpy(), g("flp_codes"))
    _close(zq, g("flp_zq"), "from_latents (partial) z_q")
    r = OD.forward(P, audio, cfg, 3)
    assert np.array_equal(r["codes"].numpy(), g("call_codes"))
    _close(r["audio"], g("call_audio"), "__call__ audio"); _close(r["z"], g("call_z"), "__call__ z")
    for name in ("long", "short"):
        meta = json.loads(str(g(f"{name}_meta")))
        f = OD.compress(P, torch.as_tensor(g(f"{name}_signal")), cfg, win_duration=meta["win_duration"], n_quantizers=None if name == "long" else 2)
        assert np.array_equal(f["codes"].numpy(), g(f"{name}_codes"))
        assert (f["chunk_length"], f["padding"], f["channels"], f["sample_rate"]) == (meta["chunk_length"], meta["padding"], meta["channels"], meta["sample_rate"])
        assert abs(f["input_db"] - meta["input_db"]) < 1e-12 and abs(f["original_length"] - meta["original_length"]) < 1e-12
        _close(OD.decompress(P, f, cfg), g(f"{name}_recon"), f"decompress {name}")
    assert golden["a_long_codes"].shape[-1] // json.loads(str(golden["a_long_meta"]))["chunk_length"] > 1      # more than one window


REFERENCE_PINS = [   # codec/tests/test_descript.py: (config, samples in, frames, latent channels, samples out)
    (OD.DAC_16K, 80_000, 250, 96, 80_043), (OD.DAC_24K, 120_000, 375, 256, 120_043), (OD.DAC_44K, 220_000, 430, 72, 220_235)]


@pytest.mark.parametrize("cfg,n,frames,lat,n_out", REFERENCE_PINS, ids=["16k", "24k", "44k"])
def test_reference_shape_pins(cfg, n, frames, lat, n_out):
    # by arithmetic at full width
    assert math.ceil(n / OD.hop(cfg)) == frames and OD.latent_dim(cfg) == 1024 and sum(OD.codebook_dims(cfg)) == lat
    assert OD.output_length(cfg, frames) == n_out
    # and by running the oracle with the reference's rates and code books at reduced width
    from mlx_audio_b200 import synth
    small = dict(cfg, encoder_dim=2, decoder_dim=32, codebook_size=16)
    P = {k: v.double() for k, v in synth.dac_weights(small, encoder=True).items()}
    z, codes, latents, _, _ = OD.encode(P, OD.preprocess(torch.zeros(1, 1, n, dtype=torch.float64), small), small)
    assert z.shape == (1, 32, frames) and codes.shape == (1, cfg["n_codebooks"], frames) and latents.shape == (1, lat, frames)
    assert OD.decode(P, z, small).squeeze(-1).shape == (1, n_out)


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference source is only present in the build container")
def test_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_dac_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    new, old = np.load(tmp_path / "dac_golden.npz"), np.load(GOLDEN)
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
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_dac_golden.py"), "--live", "4"], cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="4"), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "LIVE OK" in r.stdout, (r.stdout[-1500:], r.stderr[-1500:])


def test_import_paths():
    from mlx_audio_b200.codec import DAC, DACFile
    for mod, name, obj in (("mlx_audio.codec", "DAC", DAC), ("mlx_audio.codec.models", "DAC", DAC), ("mlx_audio.codec.models.descript", "DAC", DAC),
                           ("mlx_audio.codec.models.descript.dac", "DAC", DAC), ("mlx_audio.codec.models.descript.base", "DACFile", DACFile),
                           ("mlx_audio.codec", "DACFile", DACFile)):
        assert getattr(importlib.import_module(mod), name) is obj, (mod, name)


def test_symbols_exported_and_declared():
    from mlx_audio_b200 import _lib
    header = open(os.path.join(ROOT, "include", "b200audio.h")).read()
    lib = _lib.lib()
    for name in ("b2a_dac_rvq_encode", "b2a_dac_from_codes", "b2a_dac_rvq_encode_smem_bytes"):
        assert re.search(rf"\b{name}\s*\(", header), name
        assert name in _lib.PROTOTYPES and getattr(lib, name) is not None
    assert lib.b2a_dac_rvq_encode_smem_bytes(1024) == 2 * 8 * 1024 * 4


def test_dacfile_round_trip(tmp_path):
    from mlx_audio_b200.codec import DACFile
    codes = torch.randint(0, 1024, (1, 9, 40), generator=torch.Generator().manual_seed(0))
    f = DACFile(codes=codes, chunk_length=10, original_length=1.25, input_db=-23.5, channels=1, sample_rate=44100, padding=False, dac_version="1.0.0")
    path = f.save(tmp_path / "clip.wav")
    assert path.suffix == ".dac"
    g = DACFile.load(path)
    assert torch.equal(g.codes, codes) and (g.chunk_length, g.original_length, g.input_db, g.padding) == (10, 1.25, -23.5, False)
    art = np.load(path, allow_pickle=True)[()]
    art["metadata"]["dac_version"] = "0.0.1"
    with open(tmp_path / "old.dac", "wb") as fh:
        np.save(fh, art)
    with pytest.raises(RuntimeError):
        DACFile.load(tmp_path / "old.dac")


# ---- compile-level guard: what ptxas makes of csrc/dac.cu, which no numerical test can see --------------------------------------------
@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("dac") / "dac.o")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "dac.cu"), "-o", obj], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


@pytest.mark.parametrize("kernel,static_smem", [("dac_rvq_encode_kernel", True), ("dac_from_codes_kernel", False)])
def test_kernels_do_not_spill_and_fit_their_launch(ptxas_log, kernel, static_smem):
    pat = re.compile(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                     r"ptxas info\s*: Used (\d+) registers(?:, used \d+ barriers)?(?:, (\d+) bytes smem)?")
    props = [m for m in pat.finditer(ptxas_log) if kernel in m.group(1)]
    assert len(props) == 1, f"no ptxas report for {kernel}"
    m = props[0]
    assert int(m.group(2)) == 0 and int(m.group(3)) == 0, f"{kernel} spills {m.group(2)} / {m.group(3)} bytes"
    assert 256 * int(m.group(4)) <= 65536, f"{m.group(4)} registers x 256 threads do not fit one CTA on an SM"
    static = int(m.group(5) or 0)
    assert (static > 0) == static_smem
    # the encode launch asks for 2 x 8 frames x D floats of dynamic shared memory on top of the kernel's static arrays: at D = 1024 three
    # CTAs must still fit an SM's 227 KB, and the largest D the launch accepts (160 KB dynamic) must fit at all
    assert 3 * (2 * 8 * 1024 * 4 + static + 1024) <= 227 * 1024 and 160 * 1024 + static + 1024 <= 227 * 1024
