"""Soprano on the host (CPU): the text front end, configuration, ``sanitize``, the loader's resolution, the float64 sampler oracle against
the reference, the float64 LM loop and decoder against the reference (tests/golden/soprano_golden.npz, made by
tests/golden/make_soprano_golden.py from the reference's own code), the reference's own TestSoprano assertions, import paths, declared
symbols and ptxas."""
import json
import os
import re
import subprocess

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "soprano_golden.npz")
REF = "/root/reference/mlx_audio"


@pytest.fixture(scope="module")
def fixture():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


@pytest.fixture(scope="module")
def golden(fixture):
    return json.loads(str(fixture["meta"]))


def _generator():
    import sys
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_soprano_golden as MG
    import synth_params
    return MG, synth_params


def _config(**kw):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.soprano import ModelConfig
    return ModelConfig.from_dict({**synth.SOPRANO_LM, **kw})


def _model(**kw):
    from mlx_audio_b200.tts.models.soprano import Model
    return Model(_config(**kw), device="cpu")


def test_clean_text_matches_reference(golden):
    from mlx_audio.tts.models.soprano import clean_text
    assert len(golden["clean_text"]) >= 60
    for s, want in golden["clean_text"]:
        assert clean_text(s) == want, s


def test_preprocess_text_matches_reference(golden):
    m = _model()
    for texts, want in golden["preprocess"]:
        assert [list(r) for r in m._preprocess_text(texts)] == want, texts


def test_sanitize_and_post_init(golden):
    from mlx_audio_b200.tts.models.soprano import ModelConfig
    m = _model()
    w = {"model.embed_tokens.weight": torch.zeros(4, 4), "model.layers.0.input_layernorm.weight": torch.zeros(4),
         "decoder.backbone.weight": torch.zeros(4, 4, dtype=torch.float16), "lm_head.weight": torch.zeros(4, 4, dtype=torch.float16),
         "language_model.norm.weight": torch.zeros(4, dtype=torch.float16), "model.decoder.head.out.bias": torch.zeros(4, dtype=torch.float16)}
    s = m.sanitize(w)
    assert sorted(s) == golden["sanitize"]
    assert s["decoder.backbone.weight"].dtype == torch.float32 and s["language_model.lm_head.weight"].dtype == torch.float16
    for path, want in golden["post_init"]:
        d = _config(model_path=path).decoder_config
        assert [d.decoder_dim, d.decoder_intermediate_dim, d.input_kernel] == want, path


def test_sampler_oracle_matches_reference(golden):
    MG, _ = _generator()
    from oracle import soprano as OS
    rows = MG.sampler_rows()
    assert len(rows) == len(golden["sampler"])
    for (x, temp, top_p, u), g in zip(rows, golden["sampler"]):
        tok, keep, _ = OS.sample(x, u, temp, top_p)
        assert tok == g["token"], g
        if g["n_keep"] is not None:
            keep = OS.keep_mask(x, top_p)
            assert int(keep.sum()) == g["n_keep"] and int(np.flatnonzero(keep)[0]) == g["keep_min_index"]
    big = np.full(8, 300.0, dtype=np.float32)                             # exp overflows everywhere: every token kept
    assert OS.keep_mask(big, 0.5).all()
    tiny = np.full(8, -50.0, dtype=np.float32)                            # nothing reaches 1 - top_p: nothing kept, token 0
    assert not OS.keep_mask(tiny, 0.5).any() and OS.sample(tiny, 0.3, 1.0, 0.5)[0] == 0


def test_lm_loop_oracle_matches_reference(fixture, golden):
    """oracle/soprano.py's stream_generate against the reference's: identical tokens, hidden states to 1e-12, for a run ending on
    max_tokens and one ending on the stop id, at two prompt lengths."""
    MG, SP = _generator()
    from oracle import soprano as OS
    P = {k: torch.from_numpy(v) for k, v in SP.from_manifest(fixture["lm_manifest"]).items()}
    assert len(golden["lm_runs"]) == 4 and {r["stop"] is None for r in golden["lm_runs"]} == {True, False}
    for r in golden["lm_runs"]:
        u = MG.lm_uniforms(r["run"], r["max_tokens"])
        toks, hid = OS.stream_generate(P, r["ids"], MG.LM_CFG, u, r["temperature"], r["top_p"], r["max_tokens"],
                                       stop_ids=() if r["stop"] is None else (r["stop"],))
        want_t, want_h = fixture[f"lm_tokens_{r['run']}_{r['k']}"], fixture[f"lm_hidden_{r['run']}_{r['k']}"]
        assert toks.tolist() == want_t.tolist(), r
        assert hid.shape == want_h.shape and float((hid - torch.from_numpy(want_h)).abs().max()) < 1e-12, r
        assert len(want_t) == r["max_tokens"] if r["stop"] is None else r["stop"] not in want_t.tolist()


def test_decoder_oracle_matches_reference(fixture, golden):
    """oracle/soprano.py's decode against the reference's SopranoDecoder at a small configuration and the released geometry (dim 768,
    2048 / 512, input kernel 1 and 3) for L = 1, 2, 5 (2048 (L - 1) samples each), to 1e-12 of the waveform's scale; the head's shape pin."""
    MG, SP = _generator()
    from oracle import soprano as OS
    for key, d in golden["decoders"].items():
        P = {k: torch.from_numpy(v) for k, v in SP.from_manifest(fixture[f"dec_manifest_{key}"]).items()}
        cfg = OS.decoder_cfg(d["hidden"], d["dim"], d["inter"], d["layers"], d["input_kernel"], 3)
        for L in MG.DEC_L:
            want = fixture[f"dec_{key}_{L}"]
            assert want.shape == (1, 2048 * (L - 1))
            if L == 1:
                continue
            got = OS.decode(P, MG.hidden_input(key, L, d["hidden"]), cfg).numpy()
            assert np.abs(got - want).max() <= 1e-12 * max(1.0, np.abs(want).max()), (key, L)
    assert golden["head_shape"] == [1, 16 * (5 - 1)]                         # ISTFTHead keeps the batch axis: [1, hop (L - 1)]


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree not present")
def test_fixture_regenerates_from_reference(fixture, tmp_path):
    import sys
    code = ("import sys, numpy as np; sys.path.insert(0, 'tests/golden'); import make_soprano_golden as M; "
            "np.savez(sys.argv[1], **M.build())")
    out = str(tmp_path / "soprano_golden.npz")
    subprocess.run([sys.executable, "-c", code, out], cwd=ROOT, capture_output=True, text=True, check=True)
    with np.load(out) as z:
        assert sorted(z.files) == sorted(fixture)
        for k in z.files:
            if z[k].dtype.kind in "fc":
                assert np.allclose(z[k], fixture[k], rtol=0, atol=1e-13), k
            else:
                assert np.array_equal(z[k], fixture[k]), k


@pytest.mark.skipif(not os.path.isdir(REF), reason="reference tree not present")
def test_clean_text_live_random_against_reference():
    import importlib.util
    import random
    from mlx_audio_b200.tts.models.soprano import text as T
    spec = importlib.util.spec_from_file_location("_ref_soprano_text", f"{REF}/tts/models/soprano/text.py")
    R = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(R)
    rnd = random.Random(0)
    alphabet = "ab .,!?$#%&@:;+/\\<>=~_-0123456789KMBTstndrh \t\n'é"
    for _ in range(3000):
        s = "".join(rnd.choice(alphabet) for _ in range(rnd.randint(0, 30)))
        assert T.clean_text(s) == R.clean_text(s), repr(s)
    for n in range(-50, 3100, 7):
        assert T._num_to_words(n) == R._num_to_words(n) and (n < 0 or T._ordinal_to_words(n) == R._ordinal_to_words(n))


def test_reference_test_soprano_assertions():
    """The assertions of the reference's TestSoprano (tts/tests/test_models.py)."""
    from mlx_audio.tts.models.soprano import DecoderConfig, Model
    from mlx_audio.tts.models.soprano.text import (_num_to_words, _ordinal_to_words, clean_text, collapse_whitespace, convert_to_ascii,
                                                   dedup_punctuation, expand_abbreviations, expand_special_characters, normalize_numbers)
    d = DecoderConfig()
    assert (d.decoder_num_layers, d.decoder_dim, d.decoder_intermediate_dim, d.hop_length, d.n_fft, d.upscale, d.input_kernel, d.dw_kernel,
            d.token_size, d.receptive_field) == (8, 768, 2304, 512, 2048, 4, 1, 3, 2048, 4)
    c = _config(decoder_config=None)
    assert c.sample_rate == 32000 and isinstance(c.decoder_config, DecoderConfig)
    m = Model(_config(num_hidden_layers=4), device="cpu")
    assert m.language_model is not None and m.decoder is not None and m.sample_rate == 32000 and len(m.layers) == 4
    assert [m._format_duration(s) for s in (0, 1.5, 61.25, 3661.123)] == ["00:00:00.000", "00:00:01.500", "00:01:01.250", "01:01:01.123"]
    assert clean_text("Hello World!") == "hello world!" and clean_text("I have 5 apples.") == "i have five apples."
    for s, w in (("5", "five"), ("20", "twenty"), ("100", "hundred"), ("$5", "dollar"), ("1st", "first")):
        assert w in normalize_numbers(s)
    assert "mister" in expand_abbreviations("Mr.") and "doctor" in expand_abbreviations("Dr.") and "text to speech" in expand_abbreviations("TTS")
    assert all(w in expand_special_characters(s) for s, w in (("@", "at"), ("&", "and"), ("%", "percent")))
    assert [collapse_whitespace(s) for s in ("hello  world", "  hello   world  ", "hello ,world")] == ["hello world", "hello world", "hello,world"]
    assert [dedup_punctuation(s) for s in ("hello....", "hello,,,,", "hello??!!")] == ["hello.", "hello,", "hello?"]
    assert convert_to_ascii("café") == "cafe" and convert_to_ascii("naïve") == "naive"
    assert [_num_to_words(n) for n in (0, 1, 10, 21, 100, 1000, -5)] == ["zero", "one", "ten", "twenty one", "one hundred", "one thousand", "minus five"]
    assert [_ordinal_to_words(n) for n in (1, 2, 3, 10, 21)] == ["first", "second", "third", "tenth", "twenty first"]
    from mlx_audio_b200.tts.models.soprano import SopranoDecoder
    dec = SopranoDecoder(num_input_channels=512, decoder_dim=256, device="cpu")
    assert dec.intermediate_dim == 768 and dec.upscale == 4
    from mlx_audio.tts.models.soprano.decoder import ISTFTHead
    assert ISTFTHead(64, 2048, 512, device="cpu").n_fft == 2048


def test_loader_resolution(tmp_path):
    from mlx_audio_b200.utils import get_model_class
    parts = lambda name: name.lower().replace("_", "-").split("-")
    assert get_model_class("qwen3", "tts", parts("Soprano-1.1-80M-bf16")).__name__ == "mlx_audio_b200.tts.models.soprano"
    assert get_model_class("soprano", "tts").__name__ == "mlx_audio_b200.tts.models.soprano"
    assert get_model_class("kokoro", "tts", parts("Kokoro-82M")).__name__ == "mlx_audio_b200.tts.models.kokoro"
    assert get_model_class("qwen3_tts", "tts", parts("Qwen3-TTS-12Hz")).__name__ == "mlx_audio_b200.tts.models.qwen3_tts"
    assert get_model_class("whisper", "stt", parts("whisper-tiny")).__name__ == "mlx_audio_b200.stt.models.whisper"
    with pytest.raises(ValueError):
        get_model_class("qwen3", "tts", parts("some-other-model"))
    # the generic loader sets model_path: 1.1 keeps the 768 decoder, the first release gets the 512 / k3 one
    assert _config(model_path=str(tmp_path / "Soprano-1.1-80M-bf16")).decoder_config.decoder_dim == 768
    d = _config(model_path=str(tmp_path / "Soprano-80M")).decoder_config
    assert (d.decoder_dim, d.decoder_intermediate_dim, d.input_kernel) == (512, 1536, 3)


def test_tied_and_quantised_raise():
    with pytest.raises(NotImplementedError):
        _model(tie_word_embeddings=True)
    m = _model()
    with pytest.raises(NotImplementedError):
        m.sanitize({"model.layers.0.mlp.up_proj.weight": torch.zeros(4, 4, dtype=torch.uint32)})


def test_import_paths_and_symbols():
    import mlx_audio.tts.models.soprano as A
    import mlx_audio.tts.models.soprano.decoder as Dm
    import mlx_audio.tts.models.soprano.soprano as S
    import mlx_audio.tts.models.soprano.text as T
    from mlx_audio_b200 import _lib
    for n in ("Model", "ModelConfig", "DecoderConfig", "clean_text"):
        assert hasattr(A, n)
    for n in ("Model", "ModelConfig", "DecoderConfig", "SopranoModel", "SopranoDecoder"):
        assert hasattr(S, n)
    assert hasattr(Dm, "ISTFTHead") and hasattr(Dm, "SopranoDecoder") and hasattr(T, "normalize_numbers")
    header = open(os.path.join(ROOT, "include", "b200audio.h")).read()
    for sym in ("b2a_lm_sample_mlx", "b2a_soprano_upsample", "b2a_soprano_store_rows"):
        assert re.search(rf"\b{sym}\(", header) and sym in _lib.PROTOTYPES


def test_ptxas_no_spills(tmp_path):
    from mlx_audio_b200 import build
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "soprano.cu"), "-o", str(tmp_path / "soprano.o")]
    out = subprocess.run(cmd, capture_output=True, text=True, check=True).stderr
    props = re.findall(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", out)
    assert len(props) == 3 and all(p == ("0", "0", "0") for p in props), out
