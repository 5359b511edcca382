"""Golden vectors from the REFERENCE'S OWN Vocos (codec/models/vocos/{vocos,mel}.py with dsp.py's stft / istft / mel_filters) executed in
float64 with NumPy standing in for MLX (numpy_mlx_nn.py), at reduced configurations plus the reference test's two shape pins.  Run from
the repo root in the build container: python tests/golden/make_vocos_golden.py  ->  tests/golden/vocos_golden.npz;  ``--live N``: N random
configurations, the reference and oracle/vocos.py side by side (to 1e-9).

``mlx_audio.utils`` (which pulls in the whole package) is replaced by a module re-exporting dsp.py's hanning / istft / stft / mel_filters;
``yaml``, ``huggingface_hub`` and the ``..encodec`` import are stubbed (EncodecFeatures is never constructed here)."""
import json
import os
import sys
import tempfile
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import numpy_mlx_nn as shim          # noqa: E402
import synth_params                  # noqa: E402

REF = "/root/reference/mlx_audio"
mx, nn = shim.install(precise=True)

# AdaLayerNorm calls mx.fast.layer_norm with keywords (vocos.py:212); the shared stand-in takes them positionally.  Adapted here, for
# this generator's process only.
_layer_norm = mx.fast.layer_norm
mx.fast.layer_norm = lambda x, weight=None, bias=None, eps=1e-5: _layer_norm(x, weight, bias, eps)

for name, path in (("mlx_audio", REF), ("mlx_audio.codec", f"{REF}/codec"), ("mlx_audio.codec.models", f"{REF}/codec/models"),
                   ("mlx_audio.codec.models.vocos", f"{REF}/codec/models/vocos")):
    shim.stub_package(name, path)
import mlx_audio.dsp as _dsp         # noqa: E402

utils = types.ModuleType("mlx_audio.utils")
utils.hanning, utils.istft, utils.stft, utils.mel_filters = _dsp.hanning, _dsp.istft, _dsp.stft, _dsp.mel_filters
sys.modules["mlx_audio.utils"] = utils
enc = types.ModuleType("mlx_audio.codec.models.encodec")
enc.Encodec = None
sys.modules["mlx_audio.codec.models.encodec"] = enc
hub = types.ModuleType("huggingface_hub")
hub.snapshot_download = None
sys.modules["huggingface_hub"] = hub
yaml = types.ModuleType("yaml")
yaml.config = None
yaml.safe_load = lambda _f: yaml.config
sys.modules["yaml"] = yaml


def mel_cfg(dim, inter, layers, n_mels=100, **bb):
    return {"feature_extractor": {"class_path": "vocos.feature_extractors.MelSpectrogramFeatures",
                                  "init_args": {"sample_rate": 24000, "n_fft": 1024, "hop_length": 256, "n_mels": n_mels}},
            "backbone": {"class_path": "vocos.models.VocosBackbone",
                         "init_args": dict(input_channels=n_mels, dim=dim, intermediate_dim=inter, num_layers=layers, **bb)},
            "head": {"class_path": "vocos.heads.ISTFTHead", "init_args": {"dim": dim, "n_fft": 1024, "hop_length": 256}}}


def feat_cfg(cin, dim, inter, layers, n_fft, hop, **bb):
    return {"feature_extractor": {"class_path": "vocos.feature_extractors.EncodecFeatures", "init_args": {}},
            "backbone": {"class_path": "vocos.models.VocosBackbone",
                         "init_args": dict(input_channels=cin, dim=dim, intermediate_dim=inter, num_layers=layers, **bb)},
            "head": {"class_path": "vocos.heads.ISTFTHead", "init_args": {"dim": dim, "n_fft": n_fft, "hop_length": hop, "padding": "same"}}}


CFG_MEL = mel_cfg(64, 96, 2)                                                     # default gamma: the constructor's 1 / num_layers
CFG_PRE = mel_cfg(8, 16, 2, n_mels=6)                                            # small: the remap case stores every parameter in and out
CFG_PRE["head"]["init_args"].update(n_fft=16, hop_length=4)
CFG_ADA = feat_cfg(12, 32, 48, 2, 64, 16, adanorm_num_embeddings=4, layer_scale_init_value=0.5, bias=False, input_kernel_size=5,
                   dw_kernel_size=3)
LOGMEL = ((513, 100), (1000, 100), (2600, 100), (2000, 40))
HEADS = ((1024, 256), (1280, 320))
HEAD_T = (1, 2, 5, 9)
HEAD_T_LIVE = 40                                                                 # checked live only: its waveforms would dominate the fixture


def _rule(n):
    if n.endswith(".scale.bias"):
        return "scale0.1"                                                         # AdaLN scales around 1 +- (cond . w)
    if n.startswith("head.out"):
        return "scale0.5"                                                         # log-magnitudes mostly below log(100)
    return None


def build(cfg, keep=lambda n: False):
    """The reference model (feature extractor left out for feature-input configs) with synthetic parameters except the names ``keep``
    accepts, which stay the constructor's.  Returns the model, the manifest entries set and the kept values."""
    from mlx_audio.codec.models.vocos.vocos import ISTFTHead, MelSpectrogramFeatures, Vocos, VocosBackbone
    fe = MelSpectrogramFeatures(**cfg["feature_extractor"]["init_args"]) if "Mel" in cfg["feature_extractor"]["class_path"] else None
    model = Vocos(fe, VocosBackbone(**cfg["backbone"]["init_args"]), ISTFTHead(**cfg["head"]["init_args"]))
    names, kept = [], {}
    for n, v in shim.flat_parameters(model):
        if keep(n):
            kept[n] = np.asarray(v)
            continue
        names.append((n, v.shape, _rule(n)))
        shim.set_parameter(model, n, synth_params.value(*names[-1]))
    return model, names, kept


def logmel_cases(out):
    from mlx_audio.codec.models.vocos.mel import log_mel_spectrogram
    rng = np.random.default_rng(71)
    for n, m in LOGMEL:
        a = (0.3 * rng.standard_normal(n)).astype(np.float32)          # inputs stored as float32 (exact in float64)
        out[f"lm_audio{n}_{m}"], out[f"lm_mel{n}_{m}"] = a, np.asarray(log_mel_spectrogram(mx.array(a), n_mels=m))
    out["lm_cases"] = np.array(LOGMEL)


def mel_model_case(out):
    model, names, kept = build(CFG_MEL, keep=lambda n: n.endswith(".gamma"))
    out["mel_params"], out["mel_cfg"] = synth_params.manifest(names), json.dumps(CFG_MEL)
    out["mel_gamma_names"] = json.dumps(sorted(kept))
    out["mel_gamma_values"] = np.stack([kept[k] for k in sorted(kept)])
    a = (0.3 * np.random.default_rng(72).standard_normal(2000)).astype(np.float32)
    out["mel_audio"], out["mel_wave"] = a, np.asarray(model(mx.array(a)))
    print("mel model", out["mel_wave"].shape, "gamma", float(out["mel_gamma_values"].mean()))


def ada_case(out):
    model, names, _ = build(CFG_ADA)
    out["ada_params"], out["ada_cfg"] = synth_params.manifest(names), json.dumps(CFG_ADA)
    rng = np.random.default_rng(73)
    x = rng.standard_normal((2, 12, 9))                                           # channels-first: the backbone transposes it
    cond = np.array([[3.0, 3.0, 3.0, 3.0], [0.5, -1.0, 2.0, 0.0]])
    out["ada_x"], out["ada_cond"] = x, cond
    out["ada_h"] = np.asarray(model.backbone(mx.array(x), bandwidth_id=mx.array(cond)))
    one = model.decode(mx.array(x[:1]), bandwidth_id=mx.array(cond[:1]))
    out["ada_wave0"] = np.asarray(one)
    print("ada backbone", out["ada_h"].shape, "decode row 0", out["ada_wave0"].shape)


def head_cases(out):
    from mlx_audio.codec.models.vocos.vocos import ISTFTHead
    rng = np.random.default_rng(74)
    for n_fft, hop in HEADS:
        dim = 16
        hd = ISTFTHead(dim, n_fft, hop)
        names = []
        for n, v in shim.flat_parameters(hd):
            names.append((f"head.{n}", v.shape, _rule(f"head.{n}")))
            shim.set_parameter(hd, n, synth_params.value(*names[-1]))
        out[f"head{n_fft}_params"] = synth_params.manifest(names)
        for T in HEAD_T:
            x = rng.standard_normal((1, T, dim))
            out[f"head{n_fft}_x{T}"], out[f"head{n_fft}_y{T}"] = x, np.asarray(hd(mx.array(x)))
        x = 30.0 * rng.standard_normal((1, 5, dim))                              # many log-magnitudes above log(100)
        out[f"head{n_fft}_xclip"], out[f"head{n_fft}_yclip"] = x, np.asarray(hd(mx.array(x)))
    out["heads"], out["head_T"] = np.array(HEADS), np.array(HEAD_T)


def pretrained_case(out):
    """Vocos.from_pretrained on a torch-layout checkpoint (conv weights [out, in, k], the two stored windows, an encodec key)."""
    from mlx_audio.codec.models.vocos.vocos import Vocos
    model, names, _ = build(CFG_PRE)
    ckpt = {}
    for n, v in shim.flat_parameters(model):
        v = np.asarray(v)
        if v.ndim == 3:
            v = np.swapaxes(v, 1, 2)
        ckpt[n] = mx.array(v)
    ckpt["feature_extractor.mel_spec.spectrogram.window"] = mx.array(np.ones(16))
    ckpt["head.istft.window"] = mx.array(np.ones(16))
    ckpt["feature_extractor.encodec.quantizer.x"] = mx.array(np.ones(3))
    mx.load = lambda _f: dict(ckpt)
    yaml.config = CFG_PRE
    with tempfile.TemporaryDirectory() as d:
        for f in ("model.safetensors", "config.yaml"):
            open(os.path.join(d, f), "w").close()
        loaded = Vocos.from_pretrained(d)
    got = dict(shim.flat_parameters(loaded))
    out["pre_in_keys"] = json.dumps(list(ckpt))
    for i, (k, v) in enumerate(ckpt.items()):
        out[f"pre_in_{i}"] = np.asarray(v)
    out["pre_cfg"], out["pre_out_keys"] = json.dumps(CFG_PRE), json.dumps(sorted(got))
    for i, k in enumerate(sorted(got)):
        out[f"pre_out_{i}"] = np.asarray(got[k])


def shape_pins(out):
    """codec/tests/test_vocos.py: 120 000 zeros through the released mel model, and 375 feature frames through the EnCodec-config
    backbone and head (its feature extractor needs EnCodec, so the features are fed directly)."""
    from mlx_audio.codec.models.vocos.vocos import ISTFTHead, MelSpectrogramFeatures, Vocos, VocosBackbone
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import vocos as OV
    m = Vocos.from_hparams(OV.CONFIG_MEL)
    out["pin_mel_shape"] = np.array(np.asarray(m(mx.zeros((120_000,)))).shape)
    c = OV.CONFIG_ENCODEC
    m = Vocos(MelSpectrogramFeatures(), VocosBackbone(**c["backbone"]["init_args"]), ISTFTHead(**c["head"]["init_args"]))
    y = m.decode(mx.zeros((1, 375, 128)), bandwidth_id=mx.array(np.array([[3, 3, 3, 3]], dtype=np.float64)))
    out["pin_encodec_shape"] = np.array(np.asarray(y).shape)
    print("pins", out["pin_mel_shape"], out["pin_encodec_shape"])


def main():
    out = {}
    logmel_cases(out)
    mel_model_case(out)
    ada_case(out)
    head_cases(out)
    pretrained_case(out)
    shape_pins(out)
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "vocos_golden.npz"), **out)


def live(n):
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import vocos as OV
    worst = 0.0
    for seed in range(n):
        rng = np.random.default_rng(7000 + seed)
        dim = int(rng.choice([8, 16, 24]))
        n_fft = int(rng.choice([16, 32, 40, 64]))
        hop = n_fft // int(rng.choice([2, 4]))
        bb = dict(num_layers=int(rng.integers(1, 4)), input_kernel_size=int(rng.choice([3, 5, 7])), dw_kernel_size=int(rng.choice([3, 7, 9])),
                  bias=bool(rng.integers(0, 2)), layer_scale_init_value=float(rng.choice([0.0, 0.3])))
        if rng.integers(0, 2):
            bb["adanorm_num_embeddings"] = int(rng.integers(1, 5))
        cin = int(rng.integers(3, 10))
        cfg = feat_cfg(cin, dim, 2 * dim, hop=hop, n_fft=n_fft, **{"layers": bb.pop("num_layers")}, **bb)
        model, names, _ = build(cfg)
        P = {k: torch.as_tensor(synth_params.value(k, sh, r)) for k, sh, r in names}
        T = int(rng.integers(1, 12))
        x = rng.standard_normal((1, T, cin))
        cond = rng.standard_normal((1, bb["adanorm_num_embeddings"])) if "adanorm_num_embeddings" in bb else None
        kw = {} if cond is None else {"bandwidth_id": mx.array(cond)}
        y = np.asarray(model.decode(mx.array(x), **kw))
        o = OV.decode(P, torch.as_tensor(x), cfg, cond)[0].numpy()
        assert y.shape == o.shape == ((T - 1) * hop,), (y.shape, o.shape)
        err = float(np.abs(y - o).max(initial=0.0))
        worst = max(worst, err)
        n = int(rng.integers(513, 3000))
        a = rng.standard_normal(n)
        from mlx_audio.codec.models.vocos.mel import log_mel_spectrogram
        lm = np.asarray(log_mel_spectrogram(mx.array(a)))
        err2 = float(np.abs(lm - OV.log_mel_spectrogram(a).numpy()).max())
        worst = max(worst, err2)
        print("vocos", "dim", dim, "n_fft", n_fft, "hop", hop, "T", T, "ada", cond is not None, "err", err, "logmel n", n, "err", err2)
    from mlx_audio.codec.models.vocos.vocos import ISTFTHead
    for n_fft, hop in HEADS:                                                    # the released head geometries at 40 frames
        rng = np.random.default_rng(7100 + n_fft)
        hd = ISTFTHead(16, n_fft, hop)
        names = []
        for k, v in shim.flat_parameters(hd):
            names.append((f"head.{k}", v.shape, _rule(f"head.{k}")))
            shim.set_parameter(hd, k, synth_params.value(*names[-1]))
        P = {k: torch.as_tensor(synth_params.value(k, sh, r)) for k, sh, r in names}
        x = rng.standard_normal((1, HEAD_T_LIVE, 16))
        y, o = np.asarray(hd(mx.array(x))), OV.head(P, torch.as_tensor(x), n_fft, hop)[0].numpy()
        assert y.shape == o.shape == ((HEAD_T_LIVE - 1) * hop,)
        err = float(np.abs(y - o).max())
        worst = max(worst, err)
        print("head", n_fft, hop, "T", HEAD_T_LIVE, "err", err)
    assert worst < 1e-9, worst
    print("LIVE OK", worst)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--live":
        live(int(sys.argv[2]))
    else:
        main()
