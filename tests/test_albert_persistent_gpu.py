"""The persistent ALBERT kernel (ops.albert_encoder) across alternating CUDA-graph replays and eager calls.

Its grid barrier lives in a per-call workspace that a memset node resets in front of every launch; a barrier state left over from a
previous call, another T or another layer count would show up here as a wrong result or as the error word a timed-out barrier sets."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from mlx_audio_b200 import ops, synth

STATE = ("X", "t_en", "pred", "idx", "total")


@pytest.fixture(scope="module")
def kokoro():
    from mlx_audio_b200.configs import KOKORO_82M
    from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig
    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    return Model(ModelConfig.from_dict(KOKORO_82M), device="cuda:0").load_weights(list(P.items()))


def _inputs(T):
    ids, ref_s = synth.kokoro_inputs(T - 2, seed=T)
    return ids[0].cuda(), ref_s.cuda()


def _separate_ops(model, ids, ref_s):
    model._albert_planes = lambda T_: False
    try:
        st = model._text_side(ids, ref_s)
    finally:
        del model._albert_planes
    torch.cuda.synchronize()
    return st


def test_albert_graph_and_eager_calls_interleaved(kokoro):
    model = kokoro
    pb = model.config.plbert
    n_layers = pb["num_hidden_layers"]
    err = None
    try:
        for T, layers, graph in [(130, n_layers, False), (130, n_layers, True), (257, n_layers, True), (130, n_layers, True),
                                 (257, n_layers - 3, False), (130, n_layers - 3, True), (130, n_layers, False), (257, n_layers, True)]:
            pb["num_hidden_layers"] = layers
            ids, ref_s = _inputs(T)
            assert model._albert_planes(T)
            if graph:
                # the text graph is cached per (T, speed): drop it when the layer count changed since its capture
                key = ("text", T, 1.0, False)
                ent = model._graphs.get(key)
                if ent is not None and ent.get("layers") != layers:
                    model._graphs.pop(key)
                ent = model._text_graph(T, 1.0, False)
                ent["layers"] = layers
                ent["ids"].copy_(ids)
                ent["ref_s"].copy_(ref_s)
                ent["graph"].replay()
                st = ent["st"]
            else:
                st = model._text_side(ids, ref_s)
            torch.cuda.synchronize()
            err = ops.albert_error_word("cuda:0")
            assert int(err.item()) == 0, (T, layers, graph)
            ref = _separate_ops(model, ids, ref_s)
            for k in STATE:
                assert torch.equal(st[k], ref[k]), (T, layers, graph, k)
    finally:
        pb["num_hidden_layers"] = n_layers
        model._graphs.clear()
