"""Golden vectors of Mimi's incremental API from the REFERENCE'S OWN code (codec/models/mimi/mimi.py:164-176 decode_step / encode_step over
modules/conv.py, seanet.py and transformer.py) executed in float64 with NumPy standing in for MLX, at the reduced configuration of
make_codec_golden.py (context 6 positions = 3 frames).  Run from the repo root in the build container:
python tests/golden/make_mimi_stream_golden.py  ->  tests/golden/mimi_stream_golden.npz"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_codec_golden as G       # noqa: E402  (installs the NumPy stand-in and the reference package stubs)
import synth_params                 # noqa: E402

mx = G.mx
DEC_FRAMES = 12                                        # four times the attention context
ENC_CHUNKINGS = {"whole": [1920] * 8, "partial": [2500, 2500, 4600, 3400, 6200]}   # every call completes at least one frame


def model():
    from mlx_audio.codec.models.mimi import mimi as M
    from mlx_audio.codec.models.mimi.modules import SeanetConfig, TransformerConfig
    c = G.MIMI_ORACLE
    seanet = SeanetConfig(dimension=c["dimension"], channels=1, causal=True, nfilters=c["nfilters"], nresidual_layers=1, ratios=c["ratios"],
                          ksize=c["ksize"], residual_ksize=c["residual_ksize"], last_ksize=c["last_ksize"], dilation_base=2, pad_mode="constant",
                          true_skip=True, compress=c["compress"])
    tr = TransformerConfig(d_model=c["d_model"], num_heads=c["num_heads"], num_layers=c["num_layers"], causal=True, norm_first=True, bias_ff=False,
                           bias_attn=False, layer_scale=c["layer_scale"], positional_embedding="rope", use_conv_bias=True, gating=False,
                           norm="layer_norm", context=c["context"], max_period=c["max_period"], max_seq_len=8192, kv_repeat=1,
                           dim_feedforward=c["dim_feedforward"], conv_layout=True, use_conv_block=False, cross_attention=False, conv_kernel_size=3)
    cfg = M.MimiConfig(channels=1, sample_rate=24000, frame_rate=12.5, renormalize=True, seanet=seanet, transformer=tr, quantizer_nq=c["nq"],
                       quantizer_bins=c["bins"], quantizer_dim=c["qdim"])
    m = M.Mimi(cfg)
    return m, G.fill(m)


def fresh(m):
    """A new stream.  Mimi.reset_state (mimi.py:138-144) leaves the top-level up- and down-sampler's step state alone (ConvTrUpsample1d's
    held-back tail, ConvDownsample1d's carried rows), so a second stream would start from the first one's leftovers; reset them as well."""
    m.reset_state()
    m.upsample.reset_state()
    m.downsample.reset_state()


def main():
    m, names = model()
    c = G.MIMI_ORACLE
    out = {"params": synth_params.manifest(names), "cfg": json.dumps(c)}
    rng = np.random.default_rng(63)
    codes = rng.integers(0, c["bins"], size=(2, c["nq"], DEC_FRAMES))
    fresh(m)
    steps = [np.asarray(m.decode_step(mx.array(codes[:, :, t:t + 1]))) for t in range(DEC_FRAMES)]
    out["dec_codes"], out["dec_pcm_steps"] = codes, np.concatenate(steps, axis=-1)
    full = np.asarray(m.decode(mx.array(codes)))
    print("decode_step frame by frame vs decode", float(np.abs(out["dec_pcm_steps"] - full).max()))
    pcm = 0.5 * rng.standard_normal((2, 1, 19200))
    out["enc_pcm"] = pcm
    for tag, chunks in ENC_CHUNKINGS.items():
        fresh(m)
        a, got = 0, []
        for n in chunks:
            got.append(np.asarray(m.encode_step(mx.array(pcm[:, :, a:a + n]))))
            a += n
        assert all(g.shape[-1] > 0 for g in got), tag
        out[f"enc_{tag}_chunks"] = np.asarray(chunks)
        out[f"enc_{tag}_counts"] = np.asarray([g.shape[-1] for g in got])
        out[f"enc_{tag}_codes"] = np.concatenate(got, axis=-1)
        print("encode_step", tag, out[f"enc_{tag}_counts"].tolist())
    np.savez_compressed(os.path.join(os.environ.get("GOLDEN_OUT", HERE), "mimi_stream_golden.npz"), **out)
    print({k: getattr(v, "shape", None) for k, v in out.items()})


if __name__ == "__main__":
    main()
