"""In-context voice cloning, host side and compile time: the speech-tokenizer encoder's checkpoint mapping against what the reference's
sanitize returns, and what ptxas makes of the tensor-core prefill attention (no spills, an asynchronous wgmma pipeline)."""
import json
import os
import re
import subprocess
import sys
import zlib

import numpy as np
import torch

from mlx_audio_b200 import build

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_encoder_sanitize_matches_the_reference_sanitize():
    """sanitize_golden.json["qwen3_tokenizer_encoder"] = key -> (shape, CRC-32 of the float32 bytes) of the encoder half of the REFERENCE's
    Qwen3TTSSpeechTokenizer.sanitize (speech_tokenizer.py:1251-1437) on transformers' Mimi encoder state dict under ``encoder.``."""
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import checkpoint_layouts as L
    from mlx_audio_b200.tts.models.qwen3_tts import Qwen3TTSSpeechTokenizer, Qwen3TTSSpeechTokenizerEncoder
    want = json.load(open(os.path.join(HERE, "sanitize_golden.json")))["qwen3_tokenizer_encoder"]
    w = {k: torch.as_tensor(np.asarray(v)) for k, v in L.qwen3_tokenizer_encoder_hf().items()}
    got = Qwen3TTSSpeechTokenizerEncoder.sanitize(w)
    assert {k: [list(v.shape), zlib.crc32(np.ascontiguousarray(v.float().numpy()).tobytes())] for k, v in got.items()} == want
    assert not Qwen3TTSSpeechTokenizer.sanitize(w)                      # the decoder's sanitize leaves the encoder alone


def test_product_encoder_config_says_what_the_oracle_says():
    from mlx_audio_b200 import configs as C
    from oracle import qwen3 as OQ
    assert C.QWEN3_TOKENIZER_ENCODER == OQ.TOKENIZER_ENCODER


def test_prefill_attention_compiles_without_spills(tmp_path):
    src = os.path.join(build.CSRC, "attn_prefill.cu")
    obj = str(tmp_path / "attn_prefill.o")
    r = subprocess.run([build._nvcc(), *build.NVCC_FLAGS, "-c", src, "-o", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    props = re.findall(r"Function properties for (\S*attn_prefill_kernel\S*)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", r.stdout)
    assert len(props) == 1, r.stdout
    assert props[0][1:] == ("0", "0"), f"attn_prefill_kernel spills {props[0][1]} / {props[0][2]} bytes"
    serialised = [l for l in r.stdout.splitlines() if re.search(r"\(C75\d\d\)", l) and "attn_prefill" in l]
    assert not serialised, "\n".join(serialised)
    sass = subprocess.run([os.path.join(os.path.dirname(build._nvcc()), "cuobjdump"), "-sass", obj], stdout=subprocess.PIPE, text=True,
                          check=True).stdout
    # per key tile: one group of 24 score MMAs and one of 12 P V MMAs, each waited for once
    assert len(re.findall(r"\bHGMMA\.", sass)) == 36 and len(re.findall(r"\bWARPGROUP\.DEPBAR\b", sass)) == 2
