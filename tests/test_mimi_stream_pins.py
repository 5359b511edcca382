"""Mimi's incremental API pinned to the reference's own code: tests/golden/mimi_stream_golden.npz holds ``decode_step`` frame by frame over
12 frames (four attention contexts) and ``encode_step`` over whole-frame and partial-frame chunkings, executed through the NumPy stand-in by
tests/golden/make_mimi_stream_golden.py.  ``oracle.mimi_stream`` restates both as slices of the one-shot oracle decode / encode."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ROOT = os.path.dirname(os.path.dirname(HERE))
FIXTURE = "mimi_stream_golden.npz"


def _load():
    if HERE not in sys.path:
        sys.path.insert(0, HERE)
    import synth_params
    g = np.load(os.path.join(HERE, FIXTURE), allow_pickle=False)
    P = {k: torch.as_tensor(v) for k, v in synth_params.from_manifest(g["params"]).items()}
    return g, P, json.loads(str(g["cfg"]))


def test_oracle_decode_stream_matches_the_reference_decode_step():
    from oracle import mimi_stream as MS
    g, P, cfg = _load()
    codes = torch.as_tensor(g["dec_codes"]).long()
    T = codes.shape[-1]
    assert T * cfg["upsample_stride"] > 2 * cfg["context"]             # the stream outruns the attention window
    steps = MS.decode_stream(P, codes, [1] * T, cfg)
    assert all(s.shape == (2, 1, 1920) for s in steps)
    got = torch.cat(steps, dim=-1).numpy()
    assert np.abs(got - g["dec_pcm_steps"]).max() < 1e-12


def test_oracle_decode_stream_is_chunking_independent():
    from oracle import mimi_stream as MS
    g, P, cfg = _load()
    codes = torch.as_tensor(g["dec_codes"]).long()
    for chunks in ([4, 8], [1, 3, 7, 1], [12]):
        got = torch.cat(MS.decode_stream(P, codes, chunks, cfg), dim=-1).numpy()
        assert np.abs(got - g["dec_pcm_steps"]).max() < 1e-12, chunks


@pytest.mark.parametrize("tag", ["whole", "partial"])
def test_oracle_encode_stream_matches_the_reference_encode_step(tag):
    from oracle import mimi_stream as MS
    g, P, cfg = _load()
    chunks = [int(c) for c in g[f"enc_{tag}_chunks"]]
    pcm = torch.as_tensor(g["enc_pcm"])[..., :sum(chunks)]
    parts = MS.encode_stream(P, pcm, chunks, cfg)
    assert [p.shape[-1] for p in parts] == g[f"enc_{tag}_counts"].tolist()
    assert np.array_equal(torch.cat(parts, dim=-1).numpy(), g[f"enc_{tag}_codes"])


def test_oracle_encode_stream_sub_frame_chunk_completes_nothing():
    from oracle import mimi_stream as MS
    g, P, cfg = _load()
    pcm = torch.as_tensor(g["enc_pcm"])[..., :700 + 1920 + 1220]
    parts = MS.encode_stream(P, pcm, [700, 1920, 1220], cfg)
    assert [p.shape[-1] for p in parts] == [0, 1, 1]


@pytest.mark.skipif(not os.path.isdir("/root/reference/mlx_audio"), reason="the reference source is only present in the build container")
def test_stream_fixture_is_what_the_reference_code_produces(tmp_path):
    env = dict(os.environ, GOLDEN_OUT=str(tmp_path), OMP_NUM_THREADS="4")
    r = subprocess.run([sys.executable, os.path.join(HERE, "make_mimi_stream_golden.py")], cwd=ROOT, env=env, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    new, old = np.load(tmp_path / FIXTURE), np.load(os.path.join(HERE, FIXTURE))
    assert sorted(new.files) == sorted(old.files)
    for k in old.files:
        a, b = new[k], old[k]
        assert a.dtype == b.dtype and a.shape == b.shape, k
        if a.dtype.kind == "f":
            assert np.abs(a - b).max(initial=0.0) <= 1e-12 * max(1.0, float(np.abs(b).max(initial=0.0))), k
        else:
            assert np.array_equal(a, b), k
