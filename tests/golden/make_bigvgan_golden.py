"""Golden vectors from the REFERENCE'S OWN BigVGAN (codec/models/bigvgan/{bigvgan,amp,activation,resample,conv}.py) executed in float64
with NumPy standing in for MLX (numpy_mlx_nn.py), at reduced configurations.  Run from the repo root in the build container:
python tests/golden/make_bigvgan_golden.py  ->  tests/golden/bigvgan_golden.npz;  ``--live N``: N random configurations, the reference
and oracle/bigvgan.py side by side (to 1e-9).

The resampling filters are module parameters; they keep the values the reference's constructor computes (the fixture stores them),
except in the "asym" case, which gives two of them deliberately non-symmetric values so that a flipped kernel cannot go unnoticed."""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import numpy_mlx_nn as shim          # noqa: E402
import synth_params                  # noqa: E402

REF = "/root/reference/mlx_audio"
mx, nn = shim.install(precise=True)

# mlx.nn.Module is a dict of its attributes (``"bias" in self``, conv.py:58): added here, for this generator's process only.
shim.Module.__contains__ = lambda self, key: key in self.__dict__

for name, path in (("mlx_audio", REF), ("mlx_audio.codec", f"{REF}/codec"), ("mlx_audio.codec.models", f"{REF}/codec/models"),
                   ("mlx_audio.codec.models.bigvgan", f"{REF}/codec/models/bigvgan")):
    shim.stub_package(name, path)

CFG_A = dict(num_mels=6, upsample_rates=[2, 4], upsample_kernel_sizes=[4, 8], upsample_initial_channel=16, resblock="1",
             resblock_kernel_sizes=[3, 5], resblock_dilation_sizes=[[1, 3], [1, 2, 3]], activation="snakebeta", snake_logscale=True,
             use_bias_at_final=True, use_tanh_at_final=True)
CFG_B = dict(num_mels=5, upsample_rates=[3, 2], upsample_kernel_sizes=[7, 4], upsample_initial_channel=12, resblock="2",
             resblock_kernel_sizes=[3, 7, 5], resblock_dilation_sizes=[[1, 3], [2], [1, 2, 4]], activation="snakebeta", snake_logscale=True,
             use_bias_at_final=False, use_tanh_at_final=False)
ASYM = ("activation_post.upsample.filter", "resblocks.0.activations.1.downsample.lowpass.filter")
FRAMES = (1, 2, 7)


def _rule(n, cfg):
    leaf = n.rsplit(".", 1)[-1]
    if leaf in ("alpha", "beta") and cfg["snake_logscale"]:
        return "small"                                                 # log-domain gains around exp(0) = 1
    if n == "conv_post.weight_g":
        return "scale0.03"                                             # keeps tanh mostly unsaturated
    return None


def build(cfg, asym=()):
    """The reference model with synthetic parameters; filters stay the constructor's (except the names in ``asym``).  Returns the
    model, the manifest entries of the values set, and the filters left as computed."""
    from mlx_audio.codec.models.bigvgan.bigvgan import BigVGAN, BigVGANConfig
    model = BigVGAN(BigVGANConfig(**cfg))
    names, filters = [], {}
    for n, v in shim.flat_parameters(model):
        if n.endswith(".filter") and n not in asym:
            filters[n] = np.asarray(v)
            continue
        names.append((n, v.shape, _rule(n, cfg)))
        shim.set_parameter(model, n, synth_params.value(*names[-1]))
    return model, names, filters


def run(model, mel):
    return np.asarray(model(mx.array(mel)))


def cases(out, tag, cfg, seed, asym=()):
    model, names, filters = build(cfg, asym)
    out[f"{tag}_params"], out[f"{tag}_cfg"] = synth_params.manifest(names), json.dumps(cfg)
    rng = np.random.default_rng(seed)
    for T in FRAMES:
        mel = rng.standard_normal((2, cfg["num_mels"], T))
        out[f"{tag}_mel{T}"], out[f"{tag}_audio{T}"] = mel, run(model, mel)
    y = out[f"{tag}_audio{FRAMES[-1]}"]
    print(tag, {T: out[f"{tag}_audio{T}"].shape for T in FRAMES}, "max", float(np.abs(y).max()), "saturated", float((np.abs(y) > 0.999).mean()))
    return filters


def activation_cases(out):
    """Activation1d(SnakeBeta) on its own, with the constructor's filters and with a non-symmetric pair."""
    from mlx_audio.codec.models.bigvgan.activation import SnakeBeta
    from mlx_audio.codec.models.bigvgan.resample import Activation1d
    C = 5
    rng = np.random.default_rng(81)
    act = Activation1d(SnakeBeta(C, alpha_logscale=True))
    act.act.alpha, act.act.beta = mx.array(0.3 * rng.standard_normal(C)), mx.array(0.3 * rng.standard_normal(C))
    out["act_alpha"], out["act_beta"] = np.asarray(act.act.alpha), np.asarray(act.act.beta)
    out["act_f_up"], out["act_f_down"] = np.asarray(act.upsample.filter), np.asarray(act.downsample.lowpass.filter)
    lengths = (1, 2, 3, 9, 33)
    out["act_lengths"] = np.array(lengths)
    for L in lengths:
        x = 2.0 * rng.standard_normal((2, L, C))
        out[f"act_x{L}"], out[f"act_y{L}"] = x, np.asarray(act(mx.array(x)))
    fu, fd = rng.standard_normal((1, 12, 1)), rng.standard_normal((1, 12, 1))
    act.upsample.filter, act.downsample.lowpass.filter = mx.array(fu), mx.array(fd)
    out["act_asym_f_up"], out["act_asym_f_down"] = fu, fd
    x = 2.0 * rng.standard_normal((2, 9, C))
    out["act_asym_x"], out["act_asym_y"] = x, np.asarray(act(mx.array(x)))


def sanitize_case(out):
    """BigVGAN.sanitize on a torch-layout checkpoint made from CFG_A's parameter tree (plus a BatchNorm counter it must drop)."""
    from mlx_audio.codec.models.bigvgan.bigvgan import BigVGAN, BigVGANConfig
    model = BigVGAN(BigVGANConfig(**CFG_A))
    ckpt = {}
    for n, v in shim.flat_parameters(model):
        v = synth_params.value(n, v.shape, None)
        if n.startswith("ups.") and v.ndim == 3:
            v = np.transpose(v, (2, 0, 1))                             # (out, K, in) -> torch ConvTranspose1d (in, out, K)
        elif v.ndim == 3:
            v = np.transpose(v, (0, 2, 1))                             # (out, K, in) -> torch Conv1d (out, in, K); filters (1, 1, K)
        ckpt[n] = mx.array(v)
    ckpt["conv_pre.num_batches_tracked"] = mx.array(np.array(3))
    new = model.sanitize(ckpt)
    out["san_in_keys"] = json.dumps(list(ckpt))
    for i, (k, v) in enumerate(ckpt.items()):
        out[f"san_in_{i}"] = np.asarray(v)
    out["san_out_keys"] = json.dumps(list(new))
    for i, (k, v) in enumerate(new.items()):
        out[f"san_out_{i}"] = np.asarray(v)


def snake_case(out):
    """The reference's Snake indexes alpha[None, :, None] against (B, T, C): it raises unless T == C."""
    from mlx_audio.codec.models.bigvgan.bigvgan import BigVGAN, BigVGANConfig
    model = BigVGAN(BigVGANConfig(**dict(CFG_A, activation="snake")))
    for n, v in shim.flat_parameters(model):
        if not n.endswith(".filter"):
            shim.set_parameter(model, n, synth_params.value(n, v.shape, _rule(n, CFG_A)))
    try:
        run(model, np.zeros((1, CFG_A["num_mels"], 3)))
        raised = ""
    except Exception as e:                                             # noqa: BLE001 -- the failure itself is the datum
        raised = type(e).__name__
    print("snake, T != C:", raised or "no error")
    out["snake_raises"] = raised


def main():
    out = {}
    filters = cases(out, "a", CFG_A, 91)
    cases(out, "b", CFG_B, 92)
    cases(out, "asym", CFG_A, 93, asym=ASYM)
    out["asym_names"] = json.dumps(list(ASYM))
    out["filter_names"] = json.dumps(sorted(filters))
    out["filter_values"] = np.stack([filters[k].reshape(-1) for k in sorted(filters)])
    activation_cases(out)
    sanitize_case(out)
    snake_case(out)
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "bigvgan_golden.npz"), **out)


def live(n):
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import bigvgan as OB
    worst = 0.0
    for seed in range(n):
        rng = np.random.default_rng(5000 + seed)
        ns = int(rng.integers(1, 4))
        rates = [int(v) for v in rng.choice([2, 3, 4], size=ns)]
        kernels = [int(u * 2 + rng.integers(0, 2)) for u in rates]     # (k - u) odd: the output is one row longer than L u
        nk = int(rng.integers(1, 4))
        cfg = dict(num_mels=int(rng.integers(2, 9)), upsample_rates=rates, upsample_kernel_sizes=kernels,
                   upsample_initial_channel=int(rng.choice([4, 8])) * 2 ** ns, resblock=str(rng.choice(["1", "2"])),
                   resblock_kernel_sizes=[int(v) for v in rng.choice([1, 3, 5, 7], size=nk)],
                   resblock_dilation_sizes=[[int(v) for v in rng.choice([1, 2, 3, 5], size=int(rng.integers(1, 4)))] for _ in range(nk)],
                   activation="snakebeta", snake_logscale=True, use_bias_at_final=bool(rng.integers(0, 2)),
                   use_tanh_at_final=bool(rng.integers(0, 2)))
        asym = ("activation_post.upsample.filter",) if rng.integers(0, 2) else ()
        model, names, _ = build(cfg, asym)
        P = {k: torch.as_tensor(synth_params.value(k, sh, r)) for k, sh, r in names}
        mel = rng.standard_normal((int(rng.integers(1, 3)), cfg["num_mels"], int(rng.integers(1, 12))))
        y, o = run(model, mel), OB.forward(P, torch.as_tensor(mel), cfg).numpy()
        assert y.shape == o.shape == (mel.shape[0], 1, OB.output_length(cfg, mel.shape[2])), (y.shape, o.shape, cfg)
        err = float(np.abs(y - o).max())
        print("bigvgan", cfg["resblock"], "rates", rates, "kernels", kernels, "dil", cfg["resblock_dilation_sizes"], "T", mel.shape[2], "err", err)
        worst = max(worst, err)
    assert worst < 1e-9, worst
    print("LIVE OK", worst)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--live":
        live(int(sys.argv[2]))
    else:
        main()
