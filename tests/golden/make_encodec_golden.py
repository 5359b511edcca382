"""Golden vectors from the REFERENCE'S OWN EnCodec (codec/models/encodec/encodec.py) executed in float64 with NumPy standing in for MLX
(numpy_mlx_nn.py), at reduced widths.  Run from the repo root in the build container: python tests/golden/make_encodec_golden.py ->
tests/golden/encodec_golden.npz;  ``--live N``: N random configurations, the reference and oracle/encodec.py side by side (to 1e-9).

Two things the shared stand-in lacks are added here, for this generator's process only: ``mx.fast.metal_kernel`` -- a NumPy emulation of
the one kernel encodec.py builds (its LSTM cell, encodec.py:89-122), reproducing its index arithmetic thread by thread (out-of-range
writes dropped, out-of-range reads 0) -- and ``nn.GroupNorm(..., pytorch_compatible=True)``.  ``huggingface_hub`` is stubbed.

Cases: a reduced 24 kHz-style model (B = 1, two LSTM layers) encoded at two bandwidths and decoded; a reduced 48 kHz-style stereo model
over 3 chunks with a padding-mask truncation; preprocess_audio on clips of different lengths; the error messages; and the LSTM at B = 2,
where the reference's kernel gets row 1 wrong (row 0 is its B = 1 result)."""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
import numpy_mlx_nn as shim          # noqa: E402

REF = "/root/reference/mlx_audio"
mx, nn = shim.install(precise=True)


def _metal_kernel(name, input_names, output_names, header, source, **_k):
    assert name == "lstm" and "thread_position_in_grid" in source

    def sig(v):
        y = 1 / (1 + np.exp(-np.abs(v)))
        return np.where(v < 0, 1 - y, y)

    def run(inputs, output_shapes, output_dtypes, grid, threadgroup, **_kk):
        x, h_in, cell = (np.asarray(a, dtype=np.float64).reshape(-1) for a in inputs[:3])
        H, t, T = int(inputs[3]), int(inputs[4]), int(inputs[5])
        hs, cs = np.zeros(int(np.prod(output_shapes[0]))), np.zeros(int(np.prod(output_shapes[1])))
        rd = lambda a, i: a[i] if 0 <= i < a.size else 0.0            # noqa: E731
        d = 4 * H
        for b in range(grid[0]):
            for yy in range(grid[1]):
                elem = b * d + yy
                idx, xi = elem, b * T * d + t * d + elem
                i = sig(rd(h_in, idx) + rd(x, xi))
                f = sig(rd(h_in, idx + H) + rd(x, xi + H))
                g = np.tanh(rd(h_in, idx + 2 * H) + rd(x, xi + 2 * H))
                o = sig(rd(h_in, idx + 3 * H) + rd(x, xi + 3 * H))
                if elem < cs.size:
                    cs[elem] = f * rd(cell, elem) + i * g
                    hs[elem] = o * np.tanh(cs[elem])
        return [hs.reshape(output_shapes[0]).view(shim.array), cs.reshape(output_shapes[1]).view(shim.array)]
    return run


mx.fast.metal_kernel = _metal_kernel


class GroupNorm(nn.Module):
    def __init__(self, num_groups, dims, eps=1e-5, affine=True, pytorch_compatible=False):
        super().__init__()
        assert pytorch_compatible and num_groups == 1
        self.eps = eps
        self.weight, self.bias = np.ones(dims).view(shim.array), np.zeros(dims).view(shim.array)

    def __call__(self, x):
        x = np.asarray(x)
        m = x.mean(axis=(1, 2), keepdims=True)
        v = ((x - m) ** 2).mean(axis=(1, 2), keepdims=True)
        return ((x - m) / np.sqrt(v + self.eps) * np.asarray(self.weight) + np.asarray(self.bias)).view(shim.array)


nn.GroupNorm = GroupNorm
for name, path in (("mlx_audio", REF), ("mlx_audio.codec", f"{REF}/codec"), ("mlx_audio.codec.models", f"{REF}/codec/models"),
                   ("mlx_audio.codec.models.encodec", f"{REF}/codec/models/encodec")):
    shim.stub_package(name, path)
hub = types.ModuleType("huggingface_hub")
hub.snapshot_download = None
sys.modules["huggingface_hub"] = hub

import torch                          # noqa: E402
from mlx_audio_b200 import configs, synth   # noqa: E402
from oracle import encodec as OE     # noqa: E402
from mlx_audio.codec.models.encodec import encodec as RE   # noqa: E402

sys.path.insert(0, os.path.join(ROOT, "tests"))
from test_encodec_pins import SMALL_24K, SMALL_48K   # noqa: E402


def build(cfg, seed):
    model = RE.Encodec(RE.EncodecConfig(**RE.filter_dataclass_fields(cfg, RE.EncodecConfig)))
    P = synth.encodec_weights(cfg, seed)
    names = [n for n, _ in shim.flat_parameters(model)]
    assert sorted(names) == sorted(P), sorted(set(names) ^ set(P))[:6]
    for n in names:
        shim.set_parameter(model, n, P[n].double().numpy())
    return model, {k: v.double() for k, v in P.items()}


def model_case(out, tag, cfg, seed, x, mask, bws):
    model, _ = build(cfg, seed)
    out[f"{tag}_cfg"], out[f"{tag}_seed"], out[f"{tag}_x"], out[f"{tag}_mask"] = json.dumps(cfg), np.array(seed), x, mask
    out[f"{tag}_bws"] = np.array(bws)
    for bw in bws:
        codes, scales = model.encode(mx.array(x), mx.array(mask), bandwidth=float(bw))
        out[f"{tag}_codes{bw}"] = np.asarray(codes).astype(np.int64)
        if cfg["normalize"]:
            out[f"{tag}_scales{bw}"] = np.stack([np.asarray(s) for s in scales])
        y = model.decode(codes, scales, mx.array(mask))
        out[f"{tag}_audio{bw}"] = np.asarray(y)
        print(tag, bw, out[f"{tag}_codes{bw}"].shape, out[f"{tag}_audio{bw}"].shape)


def main():
    out = {}
    rng = np.random.default_rng(81)
    x = (0.3 * rng.standard_normal((1, 600, 1))).astype(np.float32).astype(np.float64)
    model_case(out, "small24", SMALL_24K, 15, x, np.ones((1, 600), dtype=bool), [1.5, 6.0])
    clip = (0.3 * rng.standard_normal((300, 2))).astype(np.float32).astype(np.float64)
    cl, st = OE.chunk_length(SMALL_48K), OE.chunk_stride(SMALL_48K)
    inp, mask = RE.preprocess_audio([mx.array(clip)], 400, cl, st)
    model_case(out, "small48", SMALL_48K, 16, np.asarray(inp), np.asarray(mask), [3.0, 6.0])
    assert out["small48_codes6.0"].shape[0] >= 3 and out["small48_audio6.0"].shape[1] == out["small48_x"].shape[1]
    out["cases"] = json.dumps(["small24", "small48"])
    clips = [(0.3 * rng.standard_normal(n)).astype(np.float32).astype(np.float64) for n in (50, 130, 97)]
    out["pre_n"] = np.array(len(clips))
    for i, c in enumerate(clips):
        out[f"pre_clip{i}"] = c
    for tag, c, s in (("plain", None, None), ("chunked", 96, 80)):
        a, m = RE.preprocess_audio([mx.array(c) for c in clips], 400, c, s)
        out[f"pre_{tag}_inputs"], out[f"pre_{tag}_masks"] = np.asarray(a), np.asarray(m).astype(bool)
    errs = {}
    m48, _ = build(SMALL_48K, 15)
    for key, call in (("bandwidth", lambda: m48.encode(mx.zeros((1, 190, 2)), bandwidth=7.0)),
                      ("channels", lambda: m48.encode(mx.zeros((1, 190, 3)))),
                      ("padding", lambda: m48.encode(mx.zeros((1, 170, 2)))),
                      ("one_frame", lambda: build(SMALL_24K, 15)[0].decode(mx.zeros((1, 2, 2, 5), dtype=mx.int64), [None]))):
        try:
            call()
            raise AssertionError(key)
        except ValueError as e:
            errs[key] = str(e)
    out["errors"] = json.dumps(errs)
    lstm_case(out)
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "encodec_golden.npz"), **out)


def lstm_case(out):
    rng = np.random.default_rng(82)
    H, T = 6, 5
    layer = RE.LSTM(H, H)
    for n in ("Wx", "Wh", "bias"):
        shim.set_parameter(layer, n, 0.5 * rng.standard_normal(np.asarray(getattr(layer, n)).shape))
    x = rng.standard_normal((2, T, H))
    two = np.asarray(layer(mx.array(x)))
    ones = np.stack([np.asarray(layer(mx.array(x[b:b + 1])))[0] for b in range(2)])
    out["lstm_b2_out"], out["lstm_b1_rows"] = two, ones
    out["lstm_b2_row0_err"] = np.array(np.abs(two[0] - ones[0]).max())
    out["lstm_b2_row1_err"] = np.array(np.abs(two[1] - ones[1]).max())
    P = {"l.Wx": torch.as_tensor(np.asarray(layer.Wx)), "l.Wh": torch.as_tensor(np.asarray(layer.Wh)), "l.bias": torch.as_tensor(np.asarray(layer.bias))}
    assert np.abs(OE.lstm_layer(P, "l", torch.as_tensor(x)).numpy() - ones).max() < 1e-12
    print("lstm B = 2: row 0 err", float(out["lstm_b2_row0_err"]), "row 1 err", float(out["lstm_b2_row1_err"]))


def live(n):
    worst = 0.0
    for seed in range(n):
        rng = np.random.default_rng(8000 + seed)
        base = SMALL_48K if rng.integers(0, 2) else SMALL_24K
        cfg = dict(base, num_filters=int(rng.choice([2, 4])), num_lstm_layers=int(rng.integers(1, 3)), kernel_size=int(rng.choice([3, 5, 7])),
                   last_kernel_size=int(rng.choice([3, 7])), residual_kernel_size=int(rng.choice([1, 3])), compress=int(rng.choice([1, 2])),
                   trim_right_ratio=float(rng.choice([1.0, 0.5])), use_causal_conv=bool(rng.integers(0, 2)))
        model, P = build(cfg, 100 + seed)
        if cfg["chunk_length_s"] is None:
            x = rng.standard_normal((1, int(rng.integers(100, 400)), cfg["audio_channels"]))
            mask = np.ones(x.shape[:2], dtype=bool)
        else:
            inp, m = RE.preprocess_audio([mx.array(rng.standard_normal((int(rng.integers(100, 300)), 2)))], cfg["sampling_rate"],
                                         OE.chunk_length(cfg), OE.chunk_stride(cfg))
            x, mask = np.asarray(inp), np.asarray(m)
        bw = float(rng.choice(cfg["target_bandwidths"]))
        codes, scales = model.encode(mx.array(x), mx.array(mask), bandwidth=bw)
        y = np.asarray(model.decode(codes, scales, mx.array(mask)))
        oc, os_ = OE.encode(P, x, cfg, mask, bandwidth=bw)
        assert np.array_equal(np.asarray(codes), oc.numpy()), seed
        oy = OE.decode(P, oc, os_, cfg, mask).numpy()
        err = float(np.abs(y - oy).max() / max(1.0, np.abs(oy).max()))
        worst = max(worst, err)
        print("encodec", "normalize", cfg["normalize"], "causal", cfg["use_causal_conv"], "codes", tuple(oc.shape), "err", err)
    assert worst < 1e-9, worst
    print("LIVE OK", worst)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--live":
        live(int(sys.argv[2]))
    else:
        main()
