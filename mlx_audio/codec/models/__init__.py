from mlx_audio_b200.codec.models.dac import DAC  # noqa: F401
from mlx_audio_b200.codec.models.vocos import Vocos  # noqa: F401
from mlx_audio_b200.codec.models.encodec import Encodec  # noqa: F401
