from mlx_audio_b200.tts.models.soprano.text import *  # noqa: F401,F403
from mlx_audio_b200.tts.models.soprano.text import _num_to_words, _ordinal_to_words  # noqa: F401
