"""Golden vectors from the REFERENCE'S OWN Soprano code (tts/models/soprano/{soprano,decoder,text}.py, lm/sample_utils.py) executed with
NumPy standing in for MLX (numpy_mlx_nn.py).  Run from the repo root in the build container:
python tests/golden/make_soprano_golden.py  ->  tests/golden/soprano_golden.json

Recorded: ``clean_text`` on 64 strings, ``Model._preprocess_text`` on multi-sentence inputs (the short-sentence merge cases included),
``sanitize`` key names, the ``__post_init__`` model-path rule, and make_sampler's keep sets / tokens on crafted rows at V = 32 000
(uniforms injected through the ``categorical`` queue; rows have no ties at the keep boundary because the stand-in's argsort is not
stable).  ``build()`` returns the same dict, which tests/test_soprano_pins.py compares against the fixture when the reference is present."""
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/mlx_audio"

TEXTS = ["Hello World!", "I have 5 apples.", "$5", "$1.01", "$0.50", "$.5", "$1.2.3", "$1,234.56", "1st 2nd 3rd 4th 21st 101st 112th", "#1 fan",
         "5K run, 3m, 2b, 7T", "1,000,000 people", "In 1999 and 2005 and 2000 and 1900 and 1805 and 2999", "-5 degrees", "3.14",
         "Mr. Smith & Mrs. Jones", "Dr. Who at St. Paul", "TTS on GPUs via APIs: 5 KB, 10 MBs", "café naïve résumé", "a@b.com", "50% off; now~",
         "x+y=z", "a/b\\c_d", "<tag>", "hello....", "what?!?!", "wow!!!", "hello,,,, world", "  spaced   out  ", "tab\there", "end .",
         "ümlaut Ñandú", "1kHz and 5Hz", "etc. Ave", "Capt. Sgt. Lt. Col.", "Jr. Esq. Ltd. Co.", "It's 10:30; ok", "Numbers 12,34 and 1,2",
         "2nd-to-last", "99th 100th 0th 10th 11th 13th 20th 30th 45th", "$", "#", "$$5", "1e5", "0.001", "007", "中文 text", "Emoji 😀 here",
         "quote \"x\" 'y'", "(paren) [bracket] {brace}", "dash - and — em", "...", "?!", "!?", "a.b.c", "...,,,...", "e.g. i.e.",
         "3rd-party 5th", "MBs KBs GBs TBs CLIs CPUs", "$2,000.05 and $1.00", "$10.5", "2k", "12,345th", "1,234st"]
PREPROCESS = [["Hi. This sentence is long enough to stand alone. Ok!"], ["Short. Tiny. End."], ["A sentence that is definitely long enough. Yes."],
              ["One sentence only without a stop"], ["First text is long enough to be kept.", "Second. Also a reasonably long sentence here!"],
              ["Wait... what? Really! This one is the long sentence of the group."], [""], ["  Padded text with 3 numbers: 1, 2 and 3.  "]]


def _rows():
    """Crafted sampler rows (V = 32 000) -> [(logits, temp, top_p, u)]."""
    g = np.random.default_rng(7)
    V = 32000
    out = []
    base = (g.standard_normal(V) * 2.0 - 9.0).astype(np.float32)         # exp-sum ~ 0.09: a 0.95 filter bites hard
    for top_p in (0.0, 0.5, 0.95, 1.0):
        out.append((base, 0.3, top_p, 0.37))
    out.append((base, 0.0, 0.95, 0.5))
    big = (g.standard_normal(V) * 3.0 + 20.0).astype(np.float32)         # large logits: nothing is filtered
    out.append((big, 1.0, 0.95, 0.81))
    ovf = (g.standard_normal(V) * 3.0).astype(np.float32)
    ovf[[5, 999, 20000]] = (95.0, 120.0, 200.0)                           # exp overflows to inf from rank V - 2 up
    out.append((ovf, 0.7, 0.5, 0.12))
    mid = (g.standard_normal(V) * 4.0 - 14.0).astype(np.float32)
    out.append((mid, 0.5, 0.999, 0.66))
    return out


LM_CFG = dict(model_type="qwen3", hidden_size=64, num_hidden_layers=2, num_attention_heads=4, num_key_value_heads=2, intermediate_size=96,
              vocab_size=256, head_dim=16, rms_norm_eps=1e-5, max_position_embeddings=512, rope_theta=10000.0, tie_word_embeddings=False)
LM_RUNS = (([2, 9, 31, 7, 200, 3], 0.7, 0.9, 12), ([5, 17], 1.0, 0.95, 10))        # (prompt, temperature, top_p, max_tokens)
DECODERS = {"small": dict(hidden=64, dim=32, inter=48, layers=2, input_kernel=3), "k1": dict(hidden=512, dim=768, inter=2304, layers=8, input_kernel=1),
            "k3": dict(hidden=512, dim=768, inter=2304, layers=8, input_kernel=3)}
DEC_L = (1, 2, 5)


def _rule(name):
    if name.endswith("head.out.weight") or name.endswith("head.out.bias"):
        return "scale0.5"                                                  # log-magnitudes mostly below log(100): the clip does not hide errors
    if name.endswith("lm_head.weight"):
        return "scale4"                                                    # logits spread wide enough that top-p filtering bites
    return None


def lm_uniforms(run: int, n: int) -> np.ndarray:
    return np.random.default_rng(100 + run).random(n)


def hidden_input(key: str, L: int, H: int) -> np.ndarray:
    return np.random.default_rng(1000 * L + H + len(key)).standard_normal((1, L, H))


def build():
    sys.path.insert(0, HERE)
    import numpy_mlx_nn as shim
    import synth_params
    mx, nn = shim.install(precise=True)
    for name, path in (("mlx_audio", REF), ("mlx_audio.lm", f"{REF}/lm"), ("mlx_audio.lm.models", f"{REF}/lm/models"), ("mlx_audio.tts", f"{REF}/tts"),
                       ("mlx_audio.tts.models", f"{REF}/tts/models"), ("mlx_audio.tts.models.soprano", f"{REF}/tts/models/soprano"),
                       ("mlx_audio.codec", f"{REF}/codec"), ("mlx_audio.codec.models", f"{REF}/codec/models"),
                       ("mlx_audio.codec.models.vocos", f"{REF}/codec/models/vocos")):
        shim.stub_package(name, path)
    for stub, names in (("huggingface_hub", ("snapshot_download", "hf_hub_download")), ("transformers", ("AutoTokenizer",))):
        m = types.ModuleType(stub)
        for n in names:
            setattr(m, n, None)
        sys.modules[stub] = m
    enc = types.ModuleType("mlx_audio.codec.models.encodec")
    enc.Encodec = None
    sys.modules["mlx_audio.codec.models.encodec"] = enc
    layers, dist = types.ModuleType("mlx.nn.layers"), types.ModuleType("mlx.nn.layers.distributed")
    dist.shard_linear = None                                              # qwen3.py imports it for tensor-parallel sharding only
    mx.distributed = types.SimpleNamespace(Group=object)
    sys.modules["mlx.nn.layers"], sys.modules["mlx.nn.layers.distributed"] = layers, dist
    import mlx_audio.dsp as _dsp
    u = types.ModuleType("mlx_audio.utils")
    u.hanning, u.istft, u.stft, u.mel_filters = _dsp.hanning, _dsp.istft, _dsp.stft, _dsp.mel_filters
    sys.modules["mlx_audio.utils"] = u
    yaml = types.ModuleType("yaml")
    yaml.safe_load = None
    sys.modules["yaml"] = yaml
    import mlx_audio.codec.models.vocos.vocos as _vocos
    sys.modules["mlx_audio.codec.models.vocos"].VocosBackbone = _vocos.VocosBackbone
    from mlx_audio.lm import sample_utils as SU
    from mlx_audio.tts.models.soprano import soprano as S
    from mlx_audio.tts.models.soprano import text as T

    G = {"clean_text": [[s, T.clean_text(s)] for s in TEXTS]}
    cfg = S.ModelConfig(model_type="qwen3", hidden_size=64, num_hidden_layers=1, num_attention_heads=2, num_key_value_heads=1, intermediate_size=64,
                        vocab_size=128, head_dim=32, rms_norm_eps=1e-5, max_position_embeddings=256, rope_theta=10000.0, tie_word_embeddings=False,
                        decoder_config=S.DecoderConfig(decoder_num_layers=1, decoder_dim=32, decoder_intermediate_dim=48))
    model = S.Model(cfg)
    G["preprocess"] = [[t, [list(r) for r in model._preprocess_text(t)]] for t in PREPROCESS]
    w = {"model.embed_tokens.weight": mx.zeros((4, 4)), "model.layers.0.input_layernorm.weight": mx.zeros((4,)),
         "decoder.backbone.weight": mx.zeros((4, 4), dtype=np.float16), "lm_head.weight": mx.zeros((4, 4), dtype=np.float16),
         "language_model.norm.weight": mx.zeros((4,), dtype=np.float16), "model.decoder.head.out.bias": mx.zeros((4,), dtype=np.float16)}
    G["sanitize"] = sorted(model.sanitize(w))                           # names only: the stand-in computes in float64
    G["post_init"] = []
    for path in (None, "", "/models/Soprano-1.1-80M-bf16", "/models/soprano-80m", "ekwek/Soprano-80M", "x/SOPRANO-1.1"):
        c = S.ModelConfig(model_type="qwen3", hidden_size=8, num_hidden_layers=1, num_attention_heads=1, num_key_value_heads=1, intermediate_size=8,
                          vocab_size=8, head_dim=8, rms_norm_eps=1e-5, max_position_embeddings=8, rope_theta=1e4, tie_word_embeddings=False,
                          model_path=path)
        d = c.decoder_config
        G["post_init"].append([path, [d.decoder_dim, d.decoder_intermediate_dim, d.input_kernel]])
    G["sampler"] = []
    rnd = sys.modules["mlx.core.random"]
    for x, temp, top_p, uu in _rows():
        sampler = SU.make_sampler(temp, top_p)
        keep = None
        if 0 < top_p < 1:
            keep = np.isfinite(np.asarray(SU.apply_top_p(mx.array(x[None], dtype=np.float64), top_p))[0])
        rnd.queue.append(("categorical", np.array([uu])))
        tok = int(np.asarray(sampler(mx.array(x[None], dtype=np.float64))).reshape(-1)[0])
        rnd.queue.clear()
        G["sampler"].append({"temp": temp, "top_p": top_p, "u": uu, "token": tok,
                             "n_keep": None if keep is None else int(keep.sum()), "keep_min_index": None if keep is None else int(np.flatnonzero(keep)[0])})
    # ---- the LM loop: tokens and yielded hidden states, one run to max_tokens and the same prompt again with a stop id
    dec_small = DECODERS["small"]
    lm_cfg = S.ModelConfig(**LM_CFG, decoder_config=S.DecoderConfig(decoder_num_layers=dec_small["layers"], decoder_dim=dec_small["dim"],
                                                                   decoder_intermediate_dim=dec_small["inter"], input_kernel=3))
    lm_model = S.Model(lm_cfg)
    entries = [(n, tuple(v.shape), _rule(n)) for n, v in shim.flat_parameters(lm_model)]
    lm_model.load_weights([(n, synth_params.value(n, sh, r)) for n, sh, r in entries])
    arrays = {"lm_manifest": np.array(synth_params.manifest(entries))}
    G["lm_runs"] = []
    for ri, (ids, temp, top_p, n) in enumerate(LM_RUNS):
        for stop in (None, "pick"):
            if stop == "pick":
                stop = int(arrays[f"lm_tokens_{ri}_0"][3])                 # a token the free run produced: the rerun ends on it
            lm_model._stop_token_id = stop
            rnd.queue.extend(("categorical", np.array([x])) for x in lm_uniforms(ri, n))
            toks, hid = [], []
            for tok, h in lm_model.stream_generate(mx.array(np.array(ids, dtype=np.int32)), max_tokens=n, temperature=temp, top_p=top_p):
                if tok is not None:
                    toks.append(int(np.asarray(tok).reshape(-1)[0]))
                hid.append(np.asarray(h, dtype=np.float64).reshape(-1))
            rnd.queue.clear()
            k = 0 if stop is None else 1
            arrays[f"lm_tokens_{ri}_{k}"] = np.array(toks, dtype=np.int64)
            arrays[f"lm_hidden_{ri}_{k}"] = np.stack(hid)
            G["lm_runs"].append({"run": ri, "k": k, "ids": ids, "temperature": temp, "top_p": top_p, "max_tokens": n, "stop": stop})
    # ---- the decoder: waveforms for L = 1, 2, 5 and the head's output shape
    from mlx_audio.tts.models.soprano import decoder as SD
    G["decoders"] = {}
    for key, d in DECODERS.items():
        dec = SD.SopranoDecoder(num_input_channels=d["hidden"], decoder_num_layers=d["layers"], decoder_dim=d["dim"],
                                decoder_intermediate_dim=d["inter"], input_kernel=d["input_kernel"])
        entries = [("decoder." + n, tuple(v.shape), _rule(n)) for n, v in shim.flat_parameters(dec)]
        dec.load_weights([(n[len("decoder."):], synth_params.value(n, sh, r)) for n, sh, r in entries])
        arrays[f"dec_manifest_{key}"] = np.array(synth_params.manifest(entries))
        for L in DEC_L:
            arrays[f"dec_{key}_{L}"] = np.asarray(dec(mx.array(hidden_input(key, L, d["hidden"]))), dtype=np.float64)
        G["decoders"][key] = d
    head = SD.ISTFTHead(dim=16, n_fft=64, hop_length=16)
    G["head_shape"] = list(np.asarray(head(mx.array(np.zeros((1, 5, 16))))).shape)
    arrays["meta"] = np.array(json.dumps(G, ensure_ascii=False))
    return arrays


def sampler_rows():
    return _rows()


if __name__ == "__main__":
    out = os.path.join(HERE, "soprano_golden.npz")
    np.savez_compressed(out, **build())
    print("wrote", out)
