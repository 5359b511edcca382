"""A Kokoro model is freed as soon as its last reference goes, also after generate() has cached a pipeline on it.

The cached KokoroPipeline refers back to its model; a strong reference would make a model <-> pipeline cycle, and the model's weights
and CUDA graphs would then stay in GPU memory until some later garbage-collection pass, in the middle of whatever runs next."""
import gc
import weakref

from mlx_audio_b200 import synth
from mlx_audio_b200.configs import KOKORO_82M
from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig


def test_kokoro_model_with_a_cached_pipeline_is_freed_by_reference_counting():
    model = Model(ModelConfig.from_dict(KOKORO_82M), device="cpu").load_weights(list(synth.kokoro_weights(KOKORO_82M, seed=0).items()))
    pipe = model._get_pipeline("a")
    assert pipe.model.device == model.device and model._get_pipeline("a") is pipe
    ref = weakref.ref(model)
    gc.disable()
    try:
        del model, pipe
        assert ref() is None
    finally:
        gc.enable()
