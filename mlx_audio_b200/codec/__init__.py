from .models.bigvgan import BigVGAN, BigVGANConfig
from .models.dac import DAC, DACFile
from .models.encodec import Encodec, EncodecConfig
from .models.mimi import Mimi, MimiConfig, MimiStreamingDecoder, mimi_202407
from .models.snac import SNAC
from .models.vocos import Vocos, VocosBackbone

__all__ = ["Mimi", "MimiConfig", "MimiStreamingDecoder", "mimi_202407", "SNAC", "DAC", "DACFile", "BigVGAN", "BigVGANConfig", "Vocos", "VocosBackbone", "Encodec", "EncodecConfig"]
