"""EnCodec, CPU side: the float64 oracle against the fixture made from the reference's own code and against an independent
implementation (transformers' EncodecModel on the same weights), the reference's shape pins, the bandwidth table, host-side errors, a
local from_pretrained round trip, import paths, exported symbols, and what ptxas makes of encodec.cu."""
import importlib
import json
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from mlx_audio_b200 import build, configs, synth
from oracle import encodec as OE

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLDEN = os.path.join(HERE, "golden", "encodec_golden.npz")
HAVE_REFERENCE = os.path.isdir("/root/reference/mlx_audio")

# reduced-width configurations of the two families (the fixture uses the same ones)
# (frame rate 100: 1, 3 and 6 code books at 1.5, 3 and 6 kbps; 48 kHz-style chunks of 100 samples at a stride of 90)
SMALL_24K = dict(configs.ENCODEC_24K, num_filters=4, hidden_size=8, codebook_dim=8, upsampling_ratios=[2, 3], target_bandwidths=[1.5, 3.0, 6.0],
                 sampling_rate=600)
SMALL_48K = dict(configs.ENCODEC_48K, num_filters=4, hidden_size=8, codebook_dim=8, upsampling_ratios=[2, 2], target_bandwidths=[3.0, 6.0],
                 sampling_rate=400, chunk_length_s=0.25, overlap=0.1)


def _params(cfg, seed=15):
    return {k: v.double() for k, v in synth.encodec_weights(cfg, seed).items()}


def _close(a, b, what, tol=1e-12):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert np.abs(a - b).max(initial=0.0) <= tol * max(1.0, float(np.abs(b).max(initial=0.0))), (what, np.abs(a - b).max())


# ---------------------------------------------------------------------------------------------------------------- fixture
@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def test_oracle_reproduces_the_fixture(golden):
    for tag in json.loads(str(golden["cases"])):
        cfg = json.loads(str(golden[f"{tag}_cfg"]))
        P = _params(cfg, int(golden[f"{tag}_seed"]))
        x, mask = golden[f"{tag}_x"], golden[f"{tag}_mask"]
        for bw in golden[f"{tag}_bws"]:
            codes, scales = OE.encode(P, x, cfg, mask, bandwidth=float(bw))
            assert np.array_equal(codes.numpy(), golden[f"{tag}_codes{bw}"]), (tag, bw)
            if cfg["normalize"]:
                _close(np.stack([s.numpy() for s in scales]), golden[f"{tag}_scales{bw}"], f"{tag} scales")
            y = OE.decode(P, codes, scales, cfg, mask)
            _close(y, golden[f"{tag}_audio{bw}"], f"{tag} decode {bw}")


def test_preprocess_audio_matches_the_fixture(golden):
    clips = [golden[f"pre_clip{i}"] for i in range(int(golden["pre_n"]))]
    for tag, cl, st in (("plain", None, None), ("chunked", 96, 80)):
        inputs, masks = OE.preprocess_audio(clips, 400, cl, st)
        _close(inputs, golden[f"pre_{tag}_inputs"], tag)
        assert np.array_equal(masks.numpy(), golden[f"pre_{tag}_masks"])
        from mlx_audio_b200.codec.models.encodec import preprocess_audio
        pi, pm = preprocess_audio([torch.as_tensor(c) for c in clips], 400, cl, st, device="cpu")
        _close(pi, golden[f"pre_{tag}_inputs"], tag, tol=1e-7)
        assert np.array_equal(pm.numpy(), golden[f"pre_{tag}_masks"])


def test_reference_lstm_is_only_right_for_one_row(golden):
    """The reference's Metal kernel (encodec.py:100-133), emulated by its index arithmetic: at B = 2 row 0 matches its own B = 1 run and
    row 1 does not; the oracle's rows are each their B = 1 run."""
    assert float(golden["lstm_b2_row0_err"]) < 1e-12 and float(golden["lstm_b2_row1_err"]) > 1e-3
    _close(golden["lstm_b1_rows"][0], golden["lstm_b2_out"][0], "row 0")


def test_reference_error_paths(golden):
    msgs = json.loads(str(golden["errors"]))
    cfg = SMALL_48K
    P = _params(cfg)
    for key, call in (("bandwidth", lambda: OE.encode(P, np.zeros((1, 190, 2)), cfg, bandwidth=7.0)),
                      ("channels", lambda: OE.encode(P, np.zeros((1, 190, 3)), cfg)),
                      ("padding", lambda: OE.encode(P, np.zeros((1, 170, 2)), cfg))):
        with pytest.raises(ValueError) as e:
            call()
        assert str(e.value) == msgs[key], key
    with pytest.raises(ValueError) as e:
        OE.decode(_params(SMALL_24K), torch.zeros(1, 2, 2, 5, dtype=torch.long), [None], SMALL_24K)
    assert str(e.value) == msgs["one_frame"]


@pytest.mark.skipif(not HAVE_REFERENCE, reason="the reference source is only present in the build container")
def test_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_encodec_golden.py")], cwd=ROOT, env=env, capture_output=True,
                       text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    new, old = np.load(tmp_path / "encodec_golden.npz"), np.load(GOLDEN)
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
    r = subprocess.run([sys.executable, os.path.join(HERE, "golden", "make_encodec_golden.py"), "--live", "4"], cwd=ROOT,
                       env=dict(os.environ, OMP_NUM_THREADS="4"), capture_output=True, text=True, timeout=900)
    assert r.returncode == 0 and "LIVE OK" in r.stdout, (r.stdout[-1500:], r.stderr[-1500:])


# ---------------------------------------------------------------------------------------------------------------- shapes and tables
def test_reference_shape_pins():
    """codec/tests/test_encodec.py: zeros [1, 120000, 1] at 24 kHz -> codes (1, 1, 2, 375) by default, (1, 1, 8, 375) at 6 kbps, and
    120 000 samples back -- by arithmetic at full width and by running the oracle at reduced width."""
    cfg = configs.ENCODEC_24K
    assert OE.encoded_frames(cfg, 120_000) == 375
    assert OE.num_quantizers_for_bandwidth(cfg, cfg["target_bandwidths"][0]) == 2 and OE.num_quantizers_for_bandwidth(cfg, 6.0) == 8
    assert 375 * 320 == 120_000
    small = dict(cfg, num_filters=2, hidden_size=4, codebook_dim=4, num_lstm_layers=1)
    P = _params(small)
    for bw, nq in ((None, 2), (6.0, 8)):
        codes, scales = OE.encode(P, np.zeros((1, 120_000, 1)), small, bandwidth=bw)
        assert tuple(codes.shape) == (1, 1, nq, 375)
        assert tuple(OE.decode(P, codes, scales, small).shape) == (1, 120_000, 1)


def test_bandwidth_tables():
    from mlx_audio_b200.codec import Encodec
    for cfg, table in ((configs.ENCODEC_24K, {None: 32, 1.5: 2, 3.0: 4, 6.0: 8, 12.0: 16, 24.0: 32}),
                       (configs.ENCODEC_48K, {None: 16, 3.0: 2, 6.0: 4, 12.0: 8, 24.0: 16})):
        m = Encodec(cfg, device="cpu")
        for bw, n in table.items():
            assert OE.num_quantizers_for_bandwidth(cfg, bw) == n == m.get_num_quantizers_for_bandwidth(bw), (bw, n)
    m = Encodec(configs.ENCODEC_48K, device="cpu")
    assert (m.chunk_length, m.chunk_stride, m.channels, m.sampling_rate) == (48000, 47520, 2, 48000)
    assert (OE.chunk_length(configs.ENCODEC_48K), OE.chunk_stride(configs.ENCODEC_48K)) == (48000, 47520)


def test_product_configs_and_parameter_tree():
    from mlx_audio_b200.codec.models.encodec import param_shapes
    assert configs.ENCODEC_24K == OE.CONFIG_24K and configs.ENCODEC_48K == OE.CONFIG_48K
    for cfg in (configs.ENCODEC_24K, configs.ENCODEC_48K, SMALL_24K, SMALL_48K):
        assert param_shapes(cfg) == OE.param_shapes(cfg)


# ---------------------------------------------------------------------------------------------------------------- independent implementation
def _to_transformers(P, cfg):
    """The MLX-layout tree in transformers' EncodecModel layout: weight norm removed (the weights are the folded ones), conv weights
    [out, in, k], transposed convs [in, out, k], the LSTM's one bias as bias_ih with bias_hh = 0."""
    from torch.nn.utils import parametrize
    from transformers import EncodecConfig, EncodecModel
    hf = EncodecModel(EncodecConfig(**{k: v for k, v in cfg.items() if k != "model_type"})).double().eval()
    for mod in list(hf.modules()):
        if parametrize.is_parametrized(mod, "weight"):
            parametrize.remove_parametrizations(mod, "weight")
    sd = hf.state_dict()
    new = {}
    for k, ref in sd.items():
        if ".lstm.weight_ih_l" in k or ".lstm.weight_hh_l" in k or ".lstm.bias_" in k:
            pre, name = k.rsplit(".lstm.", 1)
            kind, j = name.rsplit("_l", 1)
            src = f"{pre}.lstm.{j}." + {"weight_ih": "Wx", "weight_hh": "Wh", "bias_ih": "bias"}.get(kind, "")
            new[k] = torch.zeros_like(ref) if kind == "bias_hh" else P[src]
        elif k.endswith(".conv.weight"):
            w = P[k]
            transposed = isinstance(hf.get_submodule(k[: -len(".weight")]), torch.nn.ConvTranspose1d)
            new[k] = w.permute(2, 0, 1) if transposed else w.permute(0, 2, 1)
        elif k in P:
            new[k] = P[k]
        else:
            new[k] = ref
    hf.load_state_dict({k: v.to(sd[k].dtype).contiguous() for k, v in new.items()})
    return hf


@pytest.mark.parametrize("tag", ["24k", "48k"])
def test_oracle_agrees_with_transformers(tag):
    """Codes identical and audio to 1e-10 against transformers' EncodecModel on the same weights.  The 48 kHz-style model (stereo,
    non-causal, time_group_norm, normalize) runs unchunked here: transformers cuts chunks on a different grid (one more chunk than the
    reference for the same padded input); the chunk grid and overlap-add are pinned by the fixture instead."""
    pytest.importorskip("transformers")
    if tag == "24k":
        cfg = dict(SMALL_24K, num_filters=8, hidden_size=16, codebook_dim=16)
    else:
        cfg = dict(SMALL_48K, num_filters=8, chunk_length_s=None, overlap=None)
    P = _params(cfg, seed=21)
    hf = _to_transformers(P, cfg)
    g = torch.Generator().manual_seed(5)
    x = 0.3 * torch.randn(1, 1800 if tag == "24k" else 400, cfg["audio_channels"], generator=g, dtype=torch.float64)
    bw = cfg["target_bandwidths"][-1]
    with torch.no_grad():
        out = hf.encode(x.transpose(1, 2), bandwidth=bw)
        codes, scales = OE.encode(P, x, cfg, bandwidth=bw)
        assert codes.shape[2] > 1 and torch.equal(codes, out.audio_codes), tag
        if cfg["normalize"]:
            _close(scales[0].reshape(-1), out.audio_scales[0].reshape(-1), "scale", tol=1e-12)
        y = OE.decode(P, codes, scales, cfg)
        ref = hf.decode(out.audio_codes, out.audio_scales)[0].transpose(1, 2)
    _close(y, ref, tag, tol=1e-10)


# ---------------------------------------------------------------------------------------------------------------- host surface
def test_host_errors():
    from mlx_audio_b200.codec import Encodec
    with pytest.raises(NotImplementedError):
        Encodec(dict(configs.ENCODEC_24K, num_residual_layers=2), device="cpu")
    with pytest.raises(NotImplementedError):
        OE.encoder({}, np.zeros((1, 100, 1)), dict(configs.ENCODEC_24K, num_residual_layers=2))
    with pytest.raises(ValueError):                                           # reflect pad of >= the input's length (quirk 3)
        OE.pad1d(torch.zeros(1, 3, 1, dtype=torch.float64), 3, 0, "reflect")
    OE.pad1d(torch.zeros(1, 4, 1, dtype=torch.float64), 3, 3, "reflect")
    m = Encodec(SMALL_48K, device="cpu")
    with pytest.raises(ValueError, match="bandwidth"):
        m.encode(torch.zeros(1, 190, 2), bandwidth=7.0)
    with pytest.raises(ValueError, match="channels"):
        m.encode(torch.zeros(1, 190, 3))
    with pytest.raises(ValueError, match="properly padded"):
        m.encode(torch.zeros(1, 170, 2))
    with pytest.raises(ValueError, match="Expected one frame"):
        Encodec(SMALL_24K, device="cpu").decode(torch.zeros(1, 2, 2, 5, dtype=torch.long), [None])
    with pytest.raises(FileNotFoundError):
        Encodec.from_pretrained("mlx-community/encodec-24khz-float32", device="cpu")


def test_from_pretrained_round_trip(tmp_path):
    from safetensors.torch import save_file
    from mlx_audio_b200.codec import Encodec
    P = synth.encodec_weights(SMALL_24K)
    save_file({k: v.float().contiguous() for k, v in P.items()}, str(tmp_path / "model.safetensors"))
    (tmp_path / "config.json").write_text(json.dumps(dict(SMALL_24K, architectures=["EncodecModel"], use_conv_shortcut=True, extra=1)))
    m, proc = Encodec.from_pretrained(str(tmp_path), device="cpu")
    assert m.config.upsampling_ratios == [2, 3] and m._W is not None
    assert torch.equal(m._W["q"]["cb"][0].cpu(), P["quantizer.layers.0.codebook.embed"].float())
    x, mask = proc([np.ones(10), np.ones(7)])
    assert tuple(x.shape) == (2, 10, 1) and mask.sum().item() == 17
    with pytest.raises(ValueError, match="unexpected"):
        Encodec(SMALL_24K, device="cpu").load_weights({**P, "extra.weight": torch.zeros(1)})


def test_vocos_encodec_features_need_an_attached_model():
    from mlx_audio_b200.codec.models.vocos import EncodecFeatures
    fe = EncodecFeatures()
    assert fe.encodec is None
    for call in (lambda: fe(torch.zeros(100), bandwidth_id=0), lambda: fe.get_encodec_codes(torch.zeros(100), 0),
                 lambda: fe.get_features_from_codes(torch.zeros(2, 1, 3, dtype=torch.long))):
        with pytest.raises(NotImplementedError):
            call()


def test_import_paths():
    from mlx_audio_b200.codec import Encodec, EncodecConfig
    from mlx_audio_b200.codec.models import encodec as E
    assert E.Encodec is Encodec and E.EncodecConfig is EncodecConfig
    for mod in ("mlx_audio.codec", "mlx_audio.codec.models", "mlx_audio.codec.models.encodec", "mlx_audio.codec.models.encodec.encodec"):
        assert importlib.import_module(mod).Encodec is Encodec, mod
    m = importlib.import_module("mlx_audio.codec.models.encodec.encodec")
    assert m.preprocess_audio is E.preprocess_audio and m.EncodecConfig is EncodecConfig


def test_symbols_exported_and_declared():
    from mlx_audio_b200 import _lib
    header = open(os.path.join(ROOT, "include", "b200audio.h")).read()
    for sym in ("b2a_encodec_lstm", "b2a_encodec_pad", "b2a_encodec_gn_ws_bytes", "b2a_encodec_gn_coeffs", "b2a_encodec_normalize",
                "b2a_encodec_ola"):
        assert re.search(rf"\b{sym}\s*\(", header), sym
        assert sym in _lib.PROTOTYPES and getattr(_lib.lib(), sym) is not None, sym


def test_ptxas_no_spills_and_one_cta_per_sm(tmp_path):
    assert "encodec.cu" in build.SOURCES
    obj = str(tmp_path / "encodec.o")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "encodec.cu"), "-o", obj], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    props = re.findall(r"Compiling entry function '(\S+)'.*?\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                       r"ptxas info\s*: Used (\d+) registers", r.stdout, re.S)
    names = [p[0] for p in props]
    for k, n in (("encodec_lstm_kernel", 6), ("encodec_pad_kernel", 1), ("encodec_gn_partials_kernel", 1), ("encodec_gn_coeffs_kernel", 1),
                 ("encodec_normalize_kernel", 1), ("encodec_ola_kernel", 1)):
        assert sum(k in nm for nm in names) == n, (k, names)
    for name, stack, st, ld, regs in props:
        assert (int(st), int(ld)) == (0, 0), name
        if "encodec_lstm_kernel" in name:
            assert int(regs) * 256 <= 65536, (name, regs)                 # one 256-thread CTA per SM
    for H in (128, 256, 512):                                              # shared memory of the 4-row variant: one CTA per SM
        assert 8 * 32 * 8 * (H // 32) * 4 + 2 * 4 * H * 4 + 16 <= 227 * 1024
