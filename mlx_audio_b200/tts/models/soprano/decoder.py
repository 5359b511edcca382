"""reference: tts/models/soprano/decoder.py (``ISTFTHead`` is the Vocos head: the reference's returns [1, T])."""
from ....codec.models.vocos import ISTFTHead as _VocosHead
from .soprano import SopranoDecoder  # noqa: F401


class ISTFTHead(_VocosHead):
    """decoder.py:14-50: [B, L, dim] -> [B, (L - 1) hop]; the reference keeps the batch axis ([1, T]) and takes B = 1 only, equal-length
    B > 1 rows are accepted here."""

    def __call__(self, x):
        import torch
        with torch.no_grad():
            return self.waveform(torch.as_tensor(x).to(device=self.device, dtype=torch.float32).contiguous())
