"""Golden vectors from the REFERENCE'S OWN Descript Audio Codec (codec/models/descript/{dac,base}.py, nn/{layers,quantize}.py) executed
in float64 with NumPy standing in for MLX (numpy_mlx_nn.py), at reduced configurations.  Run from the repo root in the build container:
python tests/golden/make_dac_golden.py  ->  tests/golden/dac_golden.npz;  ``--live N``: N random configurations, the reference and
oracle/dac.py side by side (floats to 1e-9, integers identical)."""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import numpy_mlx_nn as shim          # noqa: E402
import synth_params                  # noqa: E402

REF = "/root/reference/mlx_audio"
mx, nn = shim.install(precise=True)

# Two things DAC touches that the shared stand-in does not have are added to the installed modules here, for this generator's process only:
# mlx.nn.Module is a dict of its attributes (``"bias" in self``, nn/layers.py:58), and nn.losses.mse_loss (nn/quantize.py:29-30).
shim.Module.__contains__ = lambda self, key: key in self.__dict__


def _mse_loss(predictions, targets, reduction="mean"):
    d = np.square(np.asarray(predictions) - np.asarray(targets)).view(shim.array)
    return {"none": lambda: d, "mean": d.mean, "sum": d.sum}[reduction]()


nn.losses = types.ModuleType("mlx.nn.losses")
nn.losses.mse_loss = _mse_loss
for name, path in (("mlx_audio", REF), ("mlx_audio.codec", f"{REF}/codec"), ("mlx_audio.codec.models", f"{REF}/codec/models"),
                   ("mlx_audio.codec.models.descript", f"{REF}/codec/models/descript"),
                   ("mlx_audio.codec.models.descript.nn", f"{REF}/codec/models/descript/nn")):
    shim.stub_package(name, path)
hub = types.ModuleType("huggingface_hub")
hub.snapshot_download = hub.hf_hub_download = None
sys.modules["huggingface_hub"] = hub
audio_io = types.ModuleType("mlx_audio.audio_io")      # compress() reads its input through audio_io.read: hand it the array instead
audio_io.signal = None
audio_io.read = lambda _path: audio_io.signal
sys.modules["mlx_audio.audio_io"] = audio_io

CFG_A = dict(encoder_dim=4, encoder_rates=[2, 3, 2, 2], latent_dim=None, decoder_dim=32, decoder_rates=[3, 2, 2, 2], n_codebooks=5,
             codebook_size=32, codebook_dim=4, sample_rate=240)
CFG_B = dict(encoder_dim=4, encoder_rates=[2, 4], latent_dim=12, decoder_dim=16, decoder_rates=[4, 2], n_codebooks=3, codebook_size=16,
             codebook_dim=[4, 8, 2], sample_rate=160)


def build(cfg):
    from mlx_audio.codec.models.descript.dac import DAC
    model = DAC(**cfg)
    last = f"decoder.model.layers.{len(cfg['decoder_rates']) + 2}.weight_g"
    names = [(n, v.shape, "scale0.03" if n == last else None) for n, v in shim.flat_parameters(model)]   # keeps tanh mostly unsaturated
    for n, sh, r in names:
        shim.set_parameter(model, n, synth_params.value(n, sh, r))
    return model, names


def compress(model, signal, **kw):
    audio_io.signal = (signal, model.sample_rate)
    return model.compress("unused.wav", **kw)


def cases(out, tag, cfg, seed):
    model, names = build(cfg)
    out[f"{tag}_params"], out[f"{tag}_cfg"] = synth_params.manifest(names), json.dumps(cfg)
    rng = np.random.default_rng(seed)
    hop = int(np.prod(cfg["encoder_rates"]))
    out[f"{tag}_delay"], out[f"{tag}_output_length"] = np.int64(model.delay), np.int64(model.get_output_length(1000))
    model.padding = False                                              # the setter finds no layer: nothing below may change
    audio = 0.5 * rng.standard_normal((2, 1, 9 * hop - 5))
    x = model.preprocess(mx.array(audio), cfg["sample_rate"])
    z, codes, latents, closs, bloss = model.encode(x)
    out[f"{tag}_audio"], out[f"{tag}_z"], out[f"{tag}_codes"], out[f"{tag}_latents"] = audio, np.asarray(z), np.asarray(codes), np.asarray(latents)
    out[f"{tag}_closs"], out[f"{tag}_bloss"] = np.float64(closs), np.float64(bloss)
    z2, codes2, latents2, closs2, _ = model.encode(x, 2)
    out[f"{tag}_z_nq2"], out[f"{tag}_codes_nq2"], out[f"{tag}_latents_nq2"], out[f"{tag}_closs_nq2"] = np.asarray(z2), np.asarray(codes2), np.asarray(latents2), np.float64(closs2)
    out[f"{tag}_decoded"] = np.asarray(model.decode(z))
    zq, zp, _ = model.quantizer.from_codes(codes[:, :2])
    out[f"{tag}_fc2_zq"], out[f"{tag}_fc2_zp"] = np.asarray(zq), np.asarray(zp)
    zq, zp, c = model.quantizer.from_latents(latents)
    out[f"{tag}_fl_zq"], out[f"{tag}_fl_zp"], out[f"{tag}_fl_codes"] = np.asarray(zq), np.asarray(zp), np.asarray(c)
    part = latents[:, : latents.shape[1] - 1]                          # one channel short of the last code book: it is left out
    zq, zp, c = model.quantizer.from_latents(part)
    out[f"{tag}_flp_zq"], out[f"{tag}_flp_codes"] = np.asarray(zq), np.asarray(c)
    r = model(mx.array(audio), cfg["sample_rate"], 3)
    out[f"{tag}_call_audio"], out[f"{tag}_call_codes"], out[f"{tag}_call_z"] = np.asarray(r["audio"]), np.asarray(r["codes"]), np.asarray(r["z"])
    print(tag, "encode", np.asarray(z).shape, np.asarray(codes).shape, np.asarray(latents).shape, "decode", out[f"{tag}_decoded"].shape,
          "saturated", float((np.abs(out[f"{tag}_decoded"]) > 0.999).mean()))
    # compress -> decompress over more than one window, and a signal shorter than the window (a single, padded one)
    sr = cfg["sample_rate"]
    for name, n, win in (("long", int(2.6 * sr), 0.5), ("short", int(0.7 * sr) + 3, 1.0)):
        sig = 0.1 * rng.standard_normal(n)
        f = compress(model, sig, win_duration=win, n_quantizers=None if name == "long" else 2)
        out[f"{tag}_{name}_signal"], out[f"{tag}_{name}_codes"] = sig, np.asarray(f.codes)
        out[f"{tag}_{name}_meta"] = json.dumps({"chunk_length": int(f.chunk_length), "original_length": float(f.original_length),
                                                "input_db": float(f.input_db), "channels": int(f.channels), "sample_rate": int(f.sample_rate),
                                                "padding": bool(f.padding), "win_duration": win})
        out[f"{tag}_{name}_recon"] = np.asarray(model.decompress(f))
        print(tag, name, "codes", np.asarray(f.codes).shape, "chunk", f.chunk_length, "padding", f.padding, "recon", out[f"{tag}_{name}_recon"].shape)
    assert model.padding is False


def main():
    out = {}
    cases(out, "a", CFG_A, 71)
    cases(out, "b", CFG_B, 72)
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "dac_golden.npz"), **out)
    print({k: getattr(v, "shape", None) for k, v in out.items()})


def live(n):
    import torch
    sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
    from oracle import dac as OD
    worst = 0.0

    def err(a, b):
        a, b = np.asarray(a), b.numpy() if hasattr(b, "numpy") else np.asarray(b)
        assert a.shape == b.shape, (a.shape, b.shape)
        return float(np.abs(a - b).max())

    for seed in range(n):
        rng = np.random.default_rng(4000 + seed)
        nr = int(rng.integers(2, 5))
        nq = int(rng.integers(1, 6))
        cfg = dict(encoder_dim=int(rng.choice([2, 4])), encoder_rates=[int(v) for v in rng.choice([2, 3, 4, 5], size=nr)], latent_dim=None,
                   decoder_dim=4 * 2 ** nr, decoder_rates=[int(v) for v in rng.choice([2, 3, 4, 5, 8], size=nr)], n_codebooks=nq,
                   codebook_size=int(rng.integers(8, 40)), sample_rate=int(rng.integers(100, 400)),
                   codebook_dim=int(rng.choice([2, 4, 8])) if rng.integers(0, 2) else [int(v) for v in rng.choice([2, 3, 4, 8], size=nq)])
        model, names = build(cfg)
        P = {k: torch.as_tensor(synth_params.value(k, sh, r)) for k, sh, r in names}
        hop = int(np.prod(cfg["encoder_rates"]))
        audio = 0.5 * rng.standard_normal((2, 1, int(rng.integers(2, 6)) * hop - int(rng.integers(0, hop))))
        nqs = None if rng.integers(0, 2) else int(rng.integers(1, nq + 1))
        z, codes, latents, cl, _ = model.encode(model.preprocess(mx.array(audio), cfg["sample_rate"]), nqs)
        oz, ocodes, olat, ocl, _ = OD.encode(P, OD.preprocess(torch.as_tensor(audio), cfg), cfg, nqs)
        assert np.array_equal(np.asarray(codes), ocodes.numpy()), ("codes", cfg)
        errs = [err(z, oz), err(latents, olat), abs(float(cl) - float(ocl)), err(model.decode(z), OD.decode(P, oz, cfg))]
        k = int(rng.integers(1, codes.shape[1] + 1))
        zq, zp, _ = model.quantizer.from_codes(codes[:, :k])
        ozq, ozp, _ = OD.from_codes(P, ocodes[:, :k], cfg)
        errs += [err(zq, ozq), err(zp, ozp)]
        zq, zp, c = model.quantizer.from_latents(latents)
        ozq, ozp, oc = OD.from_latents(P, olat, cfg)
        assert np.array_equal(np.asarray(c), oc.numpy()), ("from_latents", cfg)
        errs += [err(zq, ozq), err(zp, ozp)]
        sig = 0.1 * rng.standard_normal(int(rng.integers(1, 4) * cfg["sample_rate"] * 0.9))
        win = float(rng.choice([0.5, 1.0, 5.0]))
        f = compress(model, sig, win_duration=win, n_quantizers=nqs)
        of = OD.compress(P, torch.as_tensor(sig), cfg, win_duration=win, n_quantizers=nqs)
        assert np.array_equal(np.asarray(f.codes), of["codes"].numpy()) and f.chunk_length == of["chunk_length"] and f.padding == of["padding"], ("compress", cfg)
        errs += [abs(float(f.input_db) - of["input_db"]), err(model.decompress(f), OD.decompress(P, of, cfg))]
        assert model.delay == 0 and model.get_output_length(777) == 777
        print("dac enc", cfg["encoder_rates"], "dec", cfg["decoder_rates"], "nq", nq, "cd", cfg["codebook_dim"], "n_quantizers", nqs, "win", win,
              "windows", np.asarray(f.codes).shape[-1] // f.chunk_length, "err", max(errs))
        worst = max(worst, max(errs))
    assert worst < 1e-9, worst
    print("LIVE OK", worst)


if __name__ == "__main__":
    if len(sys.argv) > 2 and sys.argv[1] == "--live":
        live(int(sys.argv[2]))
    else:
        main()
