"""Descript Audio Codec on H100 (reference: codec/models/descript/{dac,base}.py, nn/{layers,quantize}.py).

``DAC(**config).load_weights(...)`` with the reference's surface: ``encode`` / ``decode`` / ``__call__``, ``quantizer(z)`` /
``from_codes`` / ``from_latents``, ``compress`` / ``decompress`` and ``DACFile``.  Weight norm is folded once at load; every Snake,
bias, residual add and the final tanh is a conv prologue / epilogue (``ops.conv1d``); the residual quantiser is one kernel each way
(``b2a_dac_rvq_encode``, ``b2a_dac_from_codes``) for any number of code books.

Two quirks of the reference are kept, because its users' code lengths depend on them:

* ``WNConvTranspose1d.__call__`` (nn/layers.py:108-110) passes ``groups`` (= 1) in ``mx.conv_transpose1d``'s ``output_padding`` slot,
  so every up-sampling stage yields one extra sample: 250 frames decode to 80 043 samples at rates [8, 5, 4, 2].
* ``CodecMixin`` (base.py:62-121) looks for ``nn.Conv1d`` / ``nn.ConvTranspose1d`` instances, but DAC's layers are ``WNConv1d`` /
  ``WNConvTranspose1d``.  The list is empty: ``delay == 0``, ``get_output_length(n) == n``, and setting ``padding`` changes no layer.
  ``compress`` on audio longer than one window therefore cuts non-overlapping, zero-padded windows of
  ``ceil(win_duration * sample_rate / hop) * hop`` samples, and ``decompress`` returns the chunks' decodes back to back, untrimmed.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from pathlib import Path
from typing import Optional, Union

import numpy as np
import torch

from ... import ops
from ...ops import ACT
from .descript_layers import downsample, fold_wn, res_unit, res_units, snake, snapshot_dir, upsample, vq_level, wnconv

SUPPORTED_VERSIONS = ["1.0.0"]

# True: the residual quantiser runs as one launch (b2a_dac_rvq_encode).  False: the level-by-level host route -- per level a 1x1 conv,
# the single-level cosine search (rvq_encode mode 1), a one-level from_codes and a torch subtraction, as SNAC.encode does.  Both produce
# the same bits; the second is the comparison the tests and tools/dac_bench.py run against.
FUSED_RVQ = [True]


@dataclass
class DACFile:
    """base.py:13-52.  ``codes`` int64 [1, n_codebooks, T] (a tensor on any device); saved as uint16 with NumPy, host side."""
    codes: torch.Tensor
    chunk_length: int
    original_length: float
    input_db: float
    channels: int
    sample_rate: int
    padding: bool
    dac_version: str

    def save(self, path):
        artifacts = {
            "codes": self.codes.detach().cpu().numpy().astype(np.uint16),
            "metadata": {"input_db": self.input_db, "original_length": self.original_length, "sample_rate": self.sample_rate,
                         "chunk_length": self.chunk_length, "channels": self.channels, "padding": self.padding,
                         "dac_version": SUPPORTED_VERSIONS[-1]},
        }
        path = Path(path).with_suffix(".dac")
        with open(path, "wb") as f:
            np.save(f, artifacts)
        return path

    @classmethod
    def load(cls, path):
        artifacts = np.load(path, allow_pickle=True)[()]
        if artifacts["metadata"].get("dac_version", None) not in SUPPORTED_VERSIONS:
            raise RuntimeError(f"Given file {path} can't be loaded with this version of descript-audio-codec.")
        return cls(codes=torch.from_numpy(artifacts["codes"].astype(np.int64)), **artifacts["metadata"])


class ResidualVectorQuantize:
    """nn/quantize.py:66-151 on the GPU.  Tensors cross this interface in the reference's layout: z / z_q [B, D, T], codes [B, nq, T],
    latents / z_p [B, sum(codebook_dim), T]."""

    def __init__(self, input_dim, n_codebooks, codebook_size, codebook_dim, device):
        self.input_dim, self.n_codebooks, self.codebook_size = input_dim, n_codebooks, codebook_size
        self.codebook_dim = [codebook_dim] * n_codebooks if isinstance(codebook_dim, int) else list(codebook_dim)
        if len(self.codebook_dim) != n_codebooks or not all(1 <= c <= 16 for c in self.codebook_dim):
            raise NotImplementedError("DAC quantiser: one codebook_dim in [1, 16] per code book")
        self.device = torch.device(device)
        self._levels = None
        self._ensure = lambda: None       # DAC hooks its first-use random initialisation in here

    def _load(self, P):
        dev = self.device
        self._levels, self._in_proj = [], []
        for i in range(self.n_codebooks):
            lv = vq_level(P, f"quantizer.quantizers.{i}", dev)
            if "in_proj" in lv:
                lv.update(w_in=lv["in_proj"].w.reshape(self.input_dim, -1), b_in=lv["in_proj"].bias)
                self._in_proj.append(lv["in_proj"])
            self._levels.append(lv)
        self._table = ops.dac_levels(self._levels, dev)
        self._cum = np.cumsum([0] + self.codebook_dim)

    def _need_encoder(self):
        self._ensure()
        if not self._in_proj:
            raise ValueError("DAC quantiser: the loaded weights have no in_proj (quantizer.quantizers.*.in_proj.*)")

    @torch.no_grad()
    def quantize_cl(self, z_cl: torch.Tensor, n_quantizers: Optional[int] = None):
        """``__call__`` on the channels-last latent the encoder leaves: z [B, T, D] -> (z_q [B, T, D], codes, latents, loss)."""
        self._need_encoder()
        n = self.n_codebooks if n_quantizers is None else max(0, min(int(n_quantizers), self.n_codebooks))
        if n == 0:
            raise ValueError("DAC quantiser: n_quantizers must be at least 1")
        z_cl = z_cl.contiguous()
        if FUSED_RVQ[0]:
            codes, latents, zq, part = ops.dac_rvq_encode(z_cl, self._table, n, self.codebook_size, int(self._cum[n]), self.input_dim)
            return zq, codes, latents, part.sum().float()
        return self._quantize_levels(z_cl, n)

    def _quantize_levels(self, z_cl, n):
        B, T, D = z_cl.shape
        residual, zq, codes, latents, loss = z_cl, None, [], [], 0.0
        for i in range(n):
            lv = self._levels[i]
            if lv["cb"].shape[1] % 4:
                raise NotImplementedError("level-by-level DAC quantiser: codebook_dim must be a multiple of 4 (rvq_encode)")
            ze = ops.conv1d(residual, self._in_proj[i])                                                        # [B, T, cd]
            idx = ops.rvq_encode(ze.reshape(B * T, -1), lv["cbn"][None], lv["c2"][None], mode=1)[:, 0].reshape(B, T).contiguous()
            zqi = ops.snac_from_codes([idx], [1], [lv["cb"]], [lv["w_out"]], [lv["b_out"]], D, check=False)
            residual = residual - zqi
            zq = zqi if zq is None else zq + zqi
            codes.append(idx)
            latents.append(ze.transpose(1, 2))
            loss = loss + ((ze.double() - lv["cb"][idx].double()) ** 2).mean()
        return zq, torch.stack(codes, dim=1), torch.cat(latents, dim=1).contiguous(), loss.float()

    def __call__(self, z: torch.Tensor, n_quantizers: Optional[int] = None):
        """quantize.py:87-120: z [B, D, T] -> (z_q [B, D, T], codes [B, nq, T], latents, commitment_loss, codebook_loss); the two losses
        are the same number in a forward pass."""
        zq, codes, latents, loss = self.quantize_cl(z.to(device=self.device, dtype=torch.float32).transpose(1, 2), n_quantizers)
        return zq.transpose(1, 2), codes, latents, loss, loss

    @torch.no_grad()
    def from_codes_cl(self, codes: torch.Tensor, want_zp=False):
        self._ensure()
        codes = codes.to(device=self.device, dtype=torch.int64)
        if codes.dim() != 3 or not 1 <= codes.shape[1] <= self.n_codebooks:
            raise ValueError(f"DAC from_codes: codes must be [B, 1..{self.n_codebooks}, T], got {tuple(codes.shape)}")
        return ops.dac_from_codes(codes.contiguous(), self._table, self.codebook_size, int(self._cum[codes.shape[1]]), self.input_dim, want_zp=want_zp)

    def from_codes(self, codes: torch.Tensor):
        """quantize.py:122-131: the first codes.shape[1] code books -> (z_q [B, D, T], z_p [B, sum(cd), T], codes)."""
        zq, zp = self.from_codes_cl(codes, want_zp=True)
        return zq.transpose(1, 2), zp, codes

    @torch.no_grad()
    def from_latents(self, latents: torch.Tensor):
        """quantize.py:133-151: as many code books as latents.shape[1] covers -> (z_q [B, D, T], z_p, codes)."""
        self._need_encoder()
        latents = latents.to(device=self.device, dtype=torch.float32)
        n = int(np.where(self._cum <= latents.shape[1])[0].max())
        if n == 0:
            raise ValueError("DAC from_latents: fewer latent channels than the first code book's dimension")
        lat = latents[:, : int(self._cum[n])].contiguous()
        codes, _, zq, _ = ops.dac_rvq_encode(None, self._table, n, self.codebook_size, int(self._cum[n]), self.input_dim, latents=lat)
        zp = self.from_codes_cl(codes, want_zp=True)[1]
        return zq.transpose(1, 2), zp, codes


class DAC:
    def __init__(self, encoder_dim=64, encoder_rates=(2, 4, 5, 8), latent_dim=None, decoder_dim=1536, decoder_rates=(8, 5, 4, 2), n_codebooks=32,
                 codebook_size=1024, codebook_dim: Union[int, list] = 8, sample_rate=44100, device="cuda", **kwargs):
        self.encoder_dim, self.encoder_rates = encoder_dim, list(encoder_rates)
        self.decoder_dim, self.decoder_rates = decoder_dim, list(decoder_rates)
        self.latent_dim = latent_dim if latent_dim is not None else encoder_dim * (2 ** len(self.encoder_rates))
        self.hop_length = int(np.prod(self.encoder_rates))
        self.n_codebooks, self.codebook_size, self.codebook_dim, self.sample_rate = n_codebooks, codebook_size, codebook_dim, sample_rate
        self.device = torch.device(device)
        self.quantizer = ResidualVectorQuantize(self.latent_dim, n_codebooks, codebook_size, codebook_dim, self.device)
        self.quantizer._ensure = self._ensure_weights
        self.padding = True            # base.py:56-80: a flag only -- no layer reads it (module docstring)
        self.delay = 0                 # base.py:82-105 over an empty layer list
        self._dec = self._enc = None

    def _ensure_weights(self):
        """The reference's constructor leaves a randomly initialised, usable model (its own tests run one); here the random weights are
        made on first use, so that a model whose weights are loaded never pays for them."""
        if self._dec is None:
            from ... import synth
            cfg = {"encoder_dim": self.encoder_dim, "encoder_rates": self.encoder_rates, "latent_dim": self.latent_dim, "decoder_dim": self.decoder_dim,
                   "decoder_rates": self.decoder_rates, "n_codebooks": self.n_codebooks, "codebook_size": self.codebook_size,
                   "codebook_dim": self.codebook_dim}
            self.load_weights(synth.dac_weights(cfg, encoder=True))

    def get_output_length(self, input_length):
        """base.py:107-121 over an empty layer list."""
        return input_length

    @classmethod
    def from_pretrained(cls, repo_id, device="cuda"):
        """dac.py:251-272 for a LOCAL snapshot directory (config.json + model.safetensors); a hub id is resolved through
        huggingface_hub only when that package can reach it."""
        import json
        path = snapshot_dir(repo_id)
        from safetensors.torch import load_file
        with open(path / "config.json") as f:
            config = json.load(f)
        return cls(**config, device=device).load_weights(list(load_file(str(path / "model.safetensors")).items()))

    def load_weights(self, weights, strict=True):
        P = dict(weights)
        dev = self.device
        self.quantizer._load(P)
        pre = "decoder.model.layers"
        D = {"in": wnconv(P, f"{pre}.0", dev), "blocks": []}
        for i, stride in enumerate(self.decoder_rates):
            bp = f"{pre}.{i + 1}.block.layers"
            wt = fold_wn(P[f"{bp}.1.weight_v"], P[f"{bp}.1.weight_g"], except_dim=2)        # (out, K, in): norm per INPUT channel, layers.py:91
            D["blocks"].append({"stride": stride, "snake": snake(P, f"{bp}.0.alpha", dev), "up": ops.pack_conv(wt, P.get(f"{bp}.1.bias"), 1, dev),
                                "res": res_units(P, bp, 2, 1, dev)})
        n = len(self.decoder_rates)
        D["out_snake"], D["out"] = snake(P, f"{pre}.{n + 1}.alpha", dev), wnconv(P, f"{pre}.{n + 2}", dev)
        self._dec, self._enc = D, None
        if "encoder.block.layers.0.weight_v" in P:
            pre = "encoder.block.layers"
            E = {"in": wnconv(P, f"{pre}.0", dev), "blocks": []}
            for i, stride in enumerate(self.encoder_rates):
                bp = f"{pre}.{i + 1}.block.layers"
                E["blocks"].append({"stride": stride, "res": res_units(P, bp, 0, 1, dev), "snake": snake(P, f"{bp}.3.alpha", dev),
                                    "down": wnconv(P, f"{bp}.4", dev)})
            n = len(self.encoder_rates)
            E["out_snake"], E["out"] = snake(P, f"{pre}.{n + 1}.alpha", dev), wnconv(P, f"{pre}.{n + 2}", dev)
            self._enc = E
        return self

    def preprocess(self, audio_data: torch.Tensor, sample_rate=None) -> torch.Tensor:
        """dac.py:182-191: right-pad [B, 1, n] to a multiple of the hop."""
        if sample_rate is None:
            sample_rate = self.sample_rate
        assert sample_rate == self.sample_rate
        n = audio_data.shape[-1]
        return torch.nn.functional.pad(audio_data, (0, -n % self.hop_length))

    @torch.no_grad()
    def encode_latent(self, audio_data: torch.Tensor) -> torch.Tensor:
        """The encoder alone (dac.py:57-80): audio [B, 1, n] -> z [B, T, latent] channels-last, in front of the quantiser."""
        self._ensure_weights()
        if self._enc is None:
            raise ValueError("DAC.encode: the loaded weights have no encoder (encoder.block.layers.*)")
        E = self._enc
        x = audio_data.to(device=self.device, dtype=torch.float32)
        y = ops.conv1d(x.reshape(x.shape[0], -1, 1).contiguous(), E["in"], pad_left=3)              # [B, 1, n] -> [B, n, 1]: same memory
        for blk in E["blocks"]:
            y = downsample(y, blk)
        return ops.conv1d(y, E["out"], pad_left=1, pre=E["out_snake"])

    @torch.no_grad()
    def encode(self, audio_data: torch.Tensor, n_quantizers: Optional[int] = None):
        """dac.py:193-202: audio [B, 1, n] (n a multiple of the hop: see ``preprocess``) -> (z [B, D, T], codes [B, nq, T] int64,
        latents [B, sum(cd), T], commitment_loss, codebook_loss)."""
        zq, codes, latents, loss = self.quantizer.quantize_cl(self.encode_latent(audio_data), n_quantizers)
        return zq.transpose(1, 2), codes, latents, loss, loss

    @torch.no_grad()
    def decode_cl(self, z_cl: torch.Tensor) -> torch.Tensor:
        self._ensure_weights()
        W = self._dec
        x = ops.conv1d(z_cl, W["in"], pad_left=3)
        for blk in W["blocks"]:
            x = upsample(x, blk)
            for ru in blk["res"]:
                x = res_unit(x, ru)
        return ops.conv1d(x, W["out"], pad_left=3, pre=W["out_snake"], post_act=ACT["tanh"])

    def decode(self, z: torch.Tensor) -> torch.Tensor:
        """dac.py:204-205: z [B, D, T] -> audio [B, T_out, 1] -- channels-last, the reference does not move the axis back."""
        return self.decode_cl(z.to(device=self.device, dtype=torch.float32).transpose(1, 2).contiguous())

    def __call__(self, audio_data: torch.Tensor, sample_rate=None, n_quantizers=None, use_rvq=True):
        """dac.py:219-249.  ``audio`` is ``x[..., :length]`` of a [B, T_out, 1] tensor, i.e. untrimmed, as in the reference; without the
        quantiser the reference has no codes to return and fails, and so does this."""
        if not use_rvq:
            raise NotImplementedError("DAC.__call__(use_rvq=False): the reference raises UnboundLocalError on this path")
        length = audio_data.shape[-1]
        audio_data = self.preprocess(audio_data, sample_rate)
        z, codes, latents, commitment_loss, codebook_loss = self.encode(audio_data, n_quantizers)
        x = self.decode(z)
        return {"audio": x[..., :length], "z": z, "codes": codes, "latents": latents, "vq/commitment_loss": commitment_loss,
                "vq/codebook_loss": codebook_loss}

    @torch.no_grad()
    def compress(self, audio, win_duration: Optional[float] = 1.0, normalize_db: Optional[float] = -16, n_quantizers=None) -> DACFile:
        """base.py:123-196 for a 1-D float sample array / tensor at ``sample_rate`` (decoding a file is audio_io's job).  All windows go
        through the encoder and the quantiser as ONE batch; the reference encodes them one at a time."""
        if isinstance(audio, (str, Path)):
            raise NotImplementedError("DAC.compress takes samples; decode the file with mlx_audio.audio_io first")
        x = torch.as_tensor(np.asarray(audio) if not isinstance(audio, torch.Tensor) else audio).to(device=self.device, dtype=torch.float32).reshape(-1)
        nt = x.shape[0]
        signal_duration = nt / self.sample_rate
        input_db = float(20 * torch.log10(torch.sqrt((x.double() ** 2).mean() + 1e-12) + 1e-12))
        if normalize_db is not None:
            x = x * float(10.0 ** ((normalize_db - input_db) / 20))
        win_duration = signal_duration if win_duration is None else win_duration
        if signal_duration <= win_duration:
            padding, n_samples = True, nt
        else:
            padding = False
            n_samples = int(math.ceil(int(win_duration * self.sample_rate) / self.hop_length) * self.hop_length)
        n_win = -(-nt // n_samples)
        wins = torch.nn.functional.pad(x, (0, n_win * n_samples - nt)).reshape(n_win, 1, n_samples)
        codes = self.encode(self.preprocess(wins, self.sample_rate), n_quantizers)[1]                          # [W, nq, Tc]
        chunk_length = codes.shape[-1]
        codes = codes.permute(1, 0, 2).reshape(1, codes.shape[1], -1)
        return DACFile(codes=codes, chunk_length=chunk_length, original_length=signal_duration, input_db=input_db, channels=1,
                       sample_rate=self.sample_rate, padding=padding, dac_version=SUPPORTED_VERSIONS[-1])

    @torch.no_grad()
    def decompress(self, obj: Union[str, Path, DACFile]) -> torch.Tensor:
        """base.py:198-231: -> [1, n].  All full chunks decode as one batch (a shorter last chunk, which ``compress`` never writes, on its own)."""
        if isinstance(obj, (str, Path)):
            obj = DACFile.load(obj)
        if self.sample_rate != obj.sample_rate:
            raise ValueError(f"Sample rate of the audio signal ({obj.sample_rate}) does not match the sample rate of the model ({self.sample_rate}).")
        codes = obj.codes.to(device=self.device, dtype=torch.int64)
        _, nq, total = codes.shape
        cl = obj.chunk_length
        full = total // cl
        recons = []
        if full:
            batch = codes[0, :, : full * cl].reshape(nq, full, cl).permute(1, 0, 2).contiguous()
            recons.append(self.decode_cl(self.quantizer.from_codes_cl(batch)[0]).reshape(1, -1))
        if total % cl:
            recons.append(self.decode_cl(self.quantizer.from_codes_cl(codes[:, :, full * cl:].contiguous())[0]).reshape(1, -1))
        out = torch.cat(recons, dim=1)
        return out * float(10.0 ** ((obj.input_db - (-16)) / 20))
