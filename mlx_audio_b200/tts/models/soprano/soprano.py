"""Soprano text-to-speech on H100 (reference: tts/models/soprano/soprano.py, decoder.py).

A Qwen3 decoder LM turns ``[STOP][TEXT]{sentence}[START]`` into a stream of tokens; its final-normed hidden states (not the tokens) are
up-sampled x4 and decoded to 32 kHz audio by a Vocos backbone and an iSTFT head (n_fft 2048, hop 512, so 2048 samples per hidden state).

H100 mapping:
- LM: the Qwen3-TTS ``_DecoderStack`` (bf16 GEMVs at decode, q/k RMSNorm + RoPE + cache append, cache attention) with standard RoPE.
  Prefill runs the head on each row's last prompt position only.  One decode step -- embedding gather, the stack, the hidden-state store
  at a device-resident step index, the head GEMV over the vocabulary, ``b2a_lm_sample_mlx`` and the offset / step increments -- is one
  CUDA graph, captured once per (batch, sampler settings) and replayed across sentences and calls until the K/V cache is reallocated.
  The host reads the finished flags every 8th step.
- All sentences of a segment run as one batch: prompts are left-padded (masked keys, positions shifted per row), each row stops on its
  own stop ids and is decoded at its own length.
- Decoder: ``b2a_soprano_upsample`` writes the bf16 planes of the backbone's embed conv (or fp32 rows), then the Vocos backbone and the
  head linear (padded to a multiple of 64 columns) and ``b2a_vocos_istft_head``.

Kept from the reference: ``ModelConfig.__post_init__`` switches to the 512-wide, k3 decoder whenever ``model_path`` is set and does not
contain "soprano-1.1" (the generic loader sets it; ``from_pretrained`` does not, so it always builds the 768-wide decoder); the output
trim ``audio[-(n * 2048 - 2048):]`` keeps the whole waveform; a single hidden state gives an empty waveform; the sampler's top-p acts
on raw (unnormalised) logits.  Divergences: tied word embeddings raise ``NotImplementedError`` when the model is built (the reference
fails on its first forward); MLX-quantised (uint32) weights raise ``NotImplementedError``; ``from_pretrained`` reads local directories
only; the categorical draw is an inverse CDF driven by uniforms (``u=`` injects them) instead of MLX's PRNG; ``generate`` batches the
sentences of a segment.
"""
from __future__ import annotations

import json
import re
import time
import weakref
from dataclasses import dataclass
from pathlib import Path
from typing import List, Optional, Tuple

import numpy as np
import torch

from .... import ops
from ....codec.models.vocos import ISTFTHead, VocosBackbone
from ..base import BaseModelArgs, GenerationResult
from ..qwen3_tts.talker import _DecoderStack
from .text import clean_text

CHECK_EVERY = 8          # decode steps between reads of the finished flags


@dataclass
class DecoderConfig(BaseModelArgs):
    """soprano.py:26-41."""
    decoder_num_layers: int = 8
    decoder_dim: int = 768
    decoder_intermediate_dim: int = 2304
    hop_length: int = 512
    n_fft: int = 2048
    upscale: int = 4
    input_kernel: int = 1
    dw_kernel: int = 3
    token_size: int = 2048
    receptive_field: int = 4


@dataclass
class ModelConfig(BaseModelArgs):
    """The Qwen3 ``ModelArgs`` (lm/models/qwen3.py:16-30) plus soprano.py:44-58."""
    model_type: str = "qwen3"
    hidden_size: int = 512
    num_hidden_layers: int = 12
    intermediate_size: int = 1024
    num_attention_heads: int = 8
    rms_norm_eps: float = 1e-6
    vocab_size: int = 32000
    num_key_value_heads: int = 4
    max_position_embeddings: int = 4096
    rope_theta: float = 10000.0
    head_dim: int = 64
    tie_word_embeddings: bool = False
    rope_scaling: Optional[dict] = None
    sample_rate: int = 32000
    decoder_config: Optional[DecoderConfig] = None
    model_path: Optional[str] = None

    def __post_init__(self):
        if isinstance(self.decoder_config, dict):
            self.decoder_config = DecoderConfig.from_dict(self.decoder_config)
        if self.decoder_config is None:
            self.decoder_config = DecoderConfig()
        if self.model_path and "soprano-1.1" not in self.model_path.lower():
            self.decoder_config.decoder_dim = 512
            self.decoder_config.decoder_intermediate_dim = 1536
            self.decoder_config.input_kernel = 3


class SopranoModel:
    """The Qwen3 LM with its own ``lm_head`` (soprano.py:61-74) on the GPU: embedding table, ``_DecoderStack``, head."""

    def __init__(self, config: ModelConfig, device="cuda"):
        if config.tie_word_embeddings:
            raise NotImplementedError("Soprano: tied word embeddings are not supported (the reference's forward needs an lm_head)")
        self.config, self.device = config, torch.device(device)
        self.stack: Optional[_DecoderStack] = None
        self.embed = self.head = None

    def load(self, P: dict):
        c, dev = self.config, self.device
        self.stack = _DecoderStack(P, "language_model", c.num_hidden_layers, c.hidden_size, c.num_attention_heads, c.num_key_value_heads,
                                   c.head_dim, c.rms_norm_eps, c.rope_theta, (0, 0), dev)
        self.embed = P["language_model.embed_tokens.weight"].float().to(dev).contiguous()
        self.head = ops.pack_linear(P["language_model.lm_head.weight"].float(), None, dev)
        return self

    @property
    def layers(self):
        return self.stack.layers if self.stack is not None else [None] * self.config.num_hidden_layers


class SopranoDecoder:
    """decoder.py:53-119: up-sampling, ``VocosBackbone`` (input_kernel, dw_kernel, gamma 1 / num_layers), ``ISTFTHead``."""

    def __init__(self, num_input_channels=512, decoder_num_layers=8, decoder_dim=512, decoder_intermediate_dim=None, hop_length=512,
                 n_fft=2048, upscale=4, input_kernel=1, dw_kernel=3, device="cuda"):
        self.decoder_initial_channels, self.num_layers, self.dim = num_input_channels, decoder_num_layers, decoder_dim
        self.intermediate_dim = decoder_intermediate_dim if decoder_intermediate_dim else decoder_dim * 3
        self.hop_length, self.n_fft, self.upscale = hop_length, n_fft, upscale
        self.device = torch.device(device)
        self.decoder = VocosBackbone(num_input_channels, decoder_dim, self.intermediate_dim, decoder_num_layers,
                                     input_kernel_size=input_kernel, dw_kernel_size=dw_kernel, device=device)
        self.head = ISTFTHead(decoder_dim, n_fft, hop_length, device=device)

    def load(self, P: dict, prefix="decoder."):
        self.decoder.load(P, prefix + "decoder.")
        self.head.load(P, prefix + "head.")
        return self

    def waveform(self, x: torch.Tensor) -> torch.Tensor:
        """Hidden states [B, L, H] fp32 (CUDA) -> [B, 2048 (L - 1)]."""
        self.decoder._ensure_weights()
        self.head._ensure_weights()
        B, L, _ = x.shape
        if L == 1:
            return torch.empty(B, 0, device=self.device, dtype=torch.float32)
        embed = self.decoder._W["embed"]
        Lo = self.upscale * (L - 1) + 1
        use_planes = embed.w_tc is not None and not embed.f16 and ops._tc_eligible(embed, Lo, 1, False, 0)
        up = ops.soprano_upsample(x, self.upscale, planes_for=embed if use_planes else None)
        h = self.decoder.forward(up, planes_for=self.head._W["out"])
        return self.head.waveform(h)

    @torch.no_grad()
    def __call__(self, x) -> torch.Tensor:
        """decoder.py:92-119: [B, L, H] -> [B, 2048 (L - 1)] (the reference's head squeezes axis 0, so it takes B = 1 only)."""
        x = torch.as_tensor(x).to(device=self.device, dtype=torch.float32).contiguous()
        return self.waveform(x)


class _Session:
    """Device state of the decode loop for one batch size: step buffers, the per-row uniform table and histories, graphs."""

    def __init__(self, B: int, H: int, cap: int, dev):
        self.B, self.cap = B, cap
        self.offset = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step = torch.zeros(1, dtype=torch.int32, device=dev)
        self.kv_start = torch.zeros(B, dtype=torch.int32, device=dev)
        self.tok = torch.zeros(B, dtype=torch.int64, device=dev)
        self.finished = torch.zeros(B, dtype=torch.uint8, device=dev)
        self.x_in = torch.zeros(B, H, device=dev)
        self.last = torch.zeros(B, H, device=dev)
        self.u = torch.zeros(B, cap, device=dev)
        self.hist = torch.zeros(B, cap, dtype=torch.int64, device=dev)
        self.hidden = torch.zeros(B, cap, H, device=dev)
        self.graphs = {}


class Model:
    """soprano.py:77-493 on the GPU."""

    def __init__(self, config, tokenizer=None, device="cuda"):
        self.config = ModelConfig.from_dict(config) if isinstance(config, dict) else config
        self.tokenizer = tokenizer
        self._stop_token_id = None
        self.device = torch.device(device)
        c, d = self.config, self.config.decoder_config
        self.language_model = SopranoModel(c, device)
        self.decoder = SopranoDecoder(c.hidden_size, d.decoder_num_layers, d.decoder_dim, d.decoder_intermediate_dim, d.hop_length, d.n_fft,
                                      d.upscale, d.input_kernel, d.dw_kernel, device)
        self._sessions = {}
        self._rng = None

    # ------------------------------------------------------------------ weights
    @staticmethod
    def _check_dtypes(weights: dict):
        for k, v in weights.items():
            if getattr(v, "dtype", None) == torch.uint32 or str(getattr(v, "dtype", "")) in ("uint32", "torch.uint32"):
                raise NotImplementedError(f"Soprano: quantised checkpoints are not supported ({k} is uint32)")

    def sanitize(self, weights: dict) -> dict:
        """soprano.py:181-195: strip a leading ``model.``, keep ``decoder.*`` (cast to float32), prefix the rest with ``language_model.``."""
        self._check_dtypes(weights)
        out = {}
        for k, v in weights.items():
            if k.startswith("model."):
                k = k.replace("model.", "")
            if k.startswith("decoder."):
                v = v.float() if isinstance(v, torch.Tensor) else np.asarray(v, dtype=np.float32)
            elif not k.startswith("language_model."):
                k = "language_model." + k
            out[k] = v
        return out

    def load_weights(self, weights, strict: bool = False):
        P = {k: torch.as_tensor(v) for k, v in dict(weights).items()}
        self._check_dtypes(P)
        self.language_model.load(P)
        self.decoder.load(P)
        self._sessions = {}
        return self

    def eval(self):
        return self

    def post_load_hook(self, model_path) -> "Model":
        """soprano.py:108-124 with a local tokenizer: the stop id is ``pad_token_id`` if set, else the first id of "[STOP]"."""
        if self.tokenizer is None:
            from transformers import AutoTokenizer
            self.tokenizer = AutoTokenizer.from_pretrained(str(model_path))
        stop = self.tokenizer.encode("[STOP]", add_special_tokens=False)
        if self.tokenizer.pad_token_id is not None:
            self._stop_token_id = self.tokenizer.pad_token_id
        elif stop:
            self._stop_token_id = stop[0]
        else:
            raise ValueError("Stop token not found in tokenizer")
        return self

    @classmethod
    def from_pretrained(cls, model_name: str, device="cuda") -> "Model":
        """soprano.py:126-179 for a local directory (config.json, model.safetensors, tokenizer files).  ``model_path`` is not set, so the
        decoder is the 768-wide one whatever the directory's name, as in the reference."""
        from safetensors.torch import load_file
        path = Path(model_name)
        if not path.exists():
            raise FileNotFoundError(f"Soprano.from_pretrained: {model_name} is not a local directory (hub downloads are not supported)")
        with open(path / "config.json") as f:
            config = ModelConfig.from_dict(json.load(f))
        model = cls(config, device=device)
        model.post_load_hook(path)
        if (path / "model.safetensors").exists():
            model.load_weights(list(model.sanitize(load_file(str(path / "model.safetensors"))).items()))
        return model

    @property
    def sample_rate(self):
        return self.config.sample_rate

    @property
    def layers(self):
        return self.language_model.layers

    # ------------------------------------------------------------------ text
    def _preprocess_text(self, texts: List[str], min_length: int = 30) -> List[Tuple[str, int, int]]:
        """soprano.py:205-258: clean, split into sentences, fold sentences shorter than ``min_length`` into a neighbour, and wrap each as
        ``[STOP][TEXT]{sentence}[START]`` -> (prompt, text index, sentence index)."""
        res = []
        for ti, text in enumerate(texts):
            parts = re.split(r"(?<=[.!?])\s+", clean_text(text.strip()))
            if min_length > 0 and len(parts) > 1:
                kept = []
                for i, s in enumerate(parts):
                    if len(s) >= min_length:
                        kept.append(s)
                    elif kept:                                     # a short sentence joins the previous one ...
                        kept[-1] = (kept[-1] + " " + s).strip()
                    elif i + 1 < len(parts):                       # ... or, at the start, the next one
                        parts[i + 1] = (s + " " + parts[i + 1]).strip()
                    else:
                        kept.append(s)
                parts = kept
            res.extend((f"[STOP][TEXT]{s}[START]", ti, si) for si, s in enumerate(parts))
        return res

    def _tokenize(self, text: str) -> List[int]:
        if self.tokenizer is None:
            raise ValueError("Tokenizer not initialized. Use from_pretrained() to load the model.")
        return list(self.tokenizer.encode(text, add_special_tokens=False))

    def _stop_ids(self):
        eos = getattr(self.tokenizer, "eos_token_id", None) if self.tokenizer is not None else None
        return [i for i in (self._stop_token_id, eos) if i is not None]

    @staticmethod
    def _format_duration(seconds: float) -> str:
        hours, mins = int(seconds // 3600), int((seconds % 3600) // 60)
        return f"{hours:02d}:{mins:02d}:{int(seconds % 60):02d}.{int((seconds % 1) * 1000):03d}"

    # ------------------------------------------------------------------ LM loop
    def _session(self, B: int, need: int) -> _Session:
        s = self._sessions.get(B)
        if s is None or s.cap < need:
            s = self._sessions[B] = _Session(B, self.config.hidden_size, -(-need // 256) * 256, self.device)
        return s

    def _uniforms(self, rows: int, n: int, seed) -> torch.Tensor:
        """[rows, n] uniforms, one independent stream per row: row r of a call draws from ``seed + r`` (or from a base seed the model's own
        generator advances per call), so a row's draws do not depend on the rows it is batched with."""
        if seed is None:
            if self._rng is None:
                self._rng = torch.Generator()
                self._rng.seed()
            seed = int(torch.randint(0, 2 ** 62, (1,), generator=self._rng))
        return torch.stack([torch.rand(n, generator=torch.Generator().manual_seed(int(seed) + r)) for r in range(rows)])

    def _prefill(self, rows, temperature, top_p, max_tokens, u, seed) -> _Session:
        lm, stack = self.language_model, self.language_model.stack
        B, P = len(rows), max(len(r) for r in rows)
        if min(len(r) for r in rows) == 0:
            raise ValueError("Soprano: empty prompt")
        s = self._session(B, max_tokens + 2)
        kc, vc = weakref.ref(stack.kc) if stack.kc is not None else None, weakref.ref(stack.vc) if stack.vc is not None else None
        stack.alloc_cache(B, P + max_tokens + 1)
        if kc is None or kc() is not stack.kc or vc() is not stack.vc:
            # the K/V cache was reallocated (another batch size or a longer run): every captured graph holds the old buffers' addresses,
            # and a new buffer may land on an old address, so the graphs of every batch size go, not only those whose pointer moved
            for other in self._sessions.values():
                other.graphs = {}
        if u is None:
            u = self._uniforms(B, max_tokens, seed) if temperature > 0 else torch.zeros(B, max_tokens)
        u = torch.as_tensor(u, dtype=torch.float32)
        if u.shape != (B, max_tokens):
            raise ValueError(f"Soprano: u must be [{B}, {max_tokens}], got {tuple(u.shape)}")
        s.u.zero_()
        s.u[:, :max_tokens].copy_(u)
        s.offset.zero_()
        s.step.zero_()
        s.finished.zero_()
        s.hist.fill_(-1)
        s.kv_start.copy_(torch.tensor([P - len(r) for r in rows], dtype=torch.int32))
        ids = torch.tensor([[0] * (P - len(r)) + [int(t) for t in r] for r in rows], dtype=torch.int64, device=self.device)
        x = ops.gather_rows(lm.embed, ids.reshape(-1)).view(B, P, -1)
        h = stack.forward(x, base_dev=s.offset, kv_start=s.kv_start, pos_shift=s.kv_start, tail=lm.head)
        ops.incr_(s.offset, P)
        ops.copy2d(h[:, -1], s.last)
        ops.store_rows_at(s.last, s.hidden, s.step)
        if max_tokens > 0:
            logits = stack._proj(s.last, lm.head, nxt=stack.layers[0]["qkv"])
            self._sample(s, logits, temperature, top_p)
        return s

    def _sample(self, s: _Session, logits, temperature, top_p):
        ops.lm_sample_mlx(logits, temperature=temperature, top_p=top_p, u=s.u, step_dev=s.step, out=s.tok, hist=s.hist, finished=s.finished,
                          stop_ids=self._stop_ids())
        ops.incr_(s.step, 1)

    def _step_body(self, s: _Session, temperature, top_p):
        lm, stack = self.language_model, self.language_model.stack
        ops.gather_rows(lm.embed, s.tok, out=s.x_in)
        h = stack.forward(s.x_in.view(s.B, 1, -1), base_dev=s.offset, kv_start=s.kv_start, pos_shift=s.kv_start, tail=lm.head)
        h2 = h.view(s.B, -1)
        ops.store_rows_at(h2, s.hidden, s.step)
        logits = stack._proj(h2, lm.head, nxt=stack.layers[0]["qkv"])
        ops.incr_(s.offset, 1)
        self._sample(s, logits, temperature, top_p)

    def _step(self, s: _Session, temperature, top_p, use_graph: bool):
        if not use_graph:
            return self._step_body(s, temperature, top_p)
        key = (float(temperature), float(top_p), tuple(self._stop_ids()))     # graphs of reallocated caches are dropped in _prefill
        g = s.graphs.get(key)
        if g is None:
            self._step_body(s, temperature, top_p)                # eager first step: loads the S = 1 kernels before the capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._step_body(s, temperature, top_p)
            s.graphs[key] = g
            return
        g.replay()

    @torch.no_grad()
    def generate_from_ids(self, prompt_id_rows, *, temperature: float = 0.3, top_p: float = 0.95, max_tokens: int = 512, seed=None, u=None,
                          use_graph: bool = True):
        """The loop of ``stream_generate`` (soprano.py:304-361) for several prompts at once, each row at its own length.  ``u``
        [rows, max_tokens]: injected uniforms (row r's draw at step i is u[r, i]).  Returns (tokens, hidden): per row the int64 tokens it
        generated (the stop token excluded) and the fp32 hidden states it yielded [n + 1, H] (the prefill's last position first)."""
        rows = [list(r) for r in prompt_id_rows]
        s = self._prefill(rows, float(temperature), float(top_p), int(max_tokens), u, seed)
        if max_tokens > 0 and not bool(s.finished.all()):
            for k in range(1, max_tokens + 1):
                self._step(s, float(temperature), float(top_p), use_graph)
                if k % CHECK_EVERY == 0 and bool(s.finished.all()):
                    break
        hist = s.hist[:, :max_tokens].cpu()
        stops = torch.tensor(self._stop_ids() or [-2])
        tokens, hidden = [], []
        for b in range(len(rows)):
            hit = torch.nonzero(torch.isin(hist[b], stops)).flatten()
            n = int(hit[0]) if hit.numel() else max_tokens
            tokens.append(hist[b, :n].clone())
            hidden.append(s.hidden[b, :n + 1].clone())
        return tokens, hidden

    @torch.no_grad()
    def stream_generate(self, input_ids, max_tokens: int = 512, temperature: float = 0.3, top_p: float = 0.95, seed=None, u=None,
                        use_graph: bool = True, **kwargs):
        """soprano.py:304-361: yields (None, hidden [1, 1, H]) after the prefill, then (token [1, 1], hidden [1, 1, H]) per generated
        token until a stop id or ``max_tokens``.  Like the reference this reads every sampled token back to the host, one sync per token;
        ``generate`` and ``generate_from_ids`` read the finished flags every 8th step instead."""
        ids = torch.as_tensor(input_ids).reshape(-1).tolist()
        s = self._prefill([ids], float(temperature), float(top_p), int(max_tokens), None if u is None else torch.as_tensor(u).reshape(1, -1),
                          seed)
        yield None, s.hidden[:1, 0:1].clone()
        stops = set(self._stop_ids())
        for k in range(1, max_tokens + 1):
            tok = int(s.hist[0, k - 1])
            if tok in stops:
                return
            self._step(s, float(temperature), float(top_p), use_graph)
            yield torch.tensor([[tok]]), s.hidden[:1, k:k + 1].clone()

    # ------------------------------------------------------------------ audio
    def generate(self, text: str, voice: Optional[str] = None, temperature: float = 0.3, top_p: float = 0.95, split_pattern: str = "\n",
                 max_tokens: int = 512, verbose: bool = False, seed=None, **kwargs):
        """soprano.py:363-485: one ``GenerationResult`` per non-empty segment; the sentences of a segment are generated as one batch.
        ``seed``: the uniforms of the whole call come from one generator seeded with it, so every segment draws fresh values."""
        prompt = text.replace("\\n", "\n").replace("\\t", "\t")
        token_size = self.config.decoder_config.token_size
        seeds = None if seed is None else torch.Generator().manual_seed(int(seed))     # one stream per call, advanced per segment
        for segment_idx, segment in enumerate(prompt.split(split_pattern)):
            if not segment.strip():
                continue
            t0 = time.perf_counter()
            sentences = self._preprocess_text([segment])
            seg_seed = None if seeds is None else int(torch.randint(0, 2 ** 62, (1,), generator=seeds))
            _, hidden = self.generate_from_ids([self._tokenize(p) for p, _, _ in sentences], temperature=temperature, top_p=top_p,
                                               max_tokens=max_tokens, seed=seg_seed)
            parts, total = [], 0
            for h in hidden:
                n = h.shape[0]
                total += n
                if n >= max_tokens and verbose:
                    print("Warning: Generation hit max tokens, possible hallucination.")
                audio = self.decoder.waveform(h[None].contiguous())[0]
                keep = n * token_size - token_size
                parts.append(audio[-keep:] if keep > 0 else audio)
            audio = torch.cat(parts) if len(parts) > 1 else parts[0]
            torch.cuda.synchronize(self.device)
            elapsed = time.perf_counter() - t0
            samples = audio.shape[0]
            dur = samples / self.sample_rate
            yield GenerationResult(
                audio=audio, samples=samples, sample_rate=self.sample_rate, segment_idx=segment_idx, token_count=total,
                audio_duration=self._format_duration(dur), real_time_factor=elapsed / dur if dur > 0 else 0,
                prompt={"tokens": total, "tokens-per-sec": round(total / elapsed, 2) if elapsed > 0 else 0},
                audio_samples={"samples": samples, "samples-per-sec": round(samples / elapsed, 2) if elapsed > 0 else 0},
                processing_time_seconds=elapsed, peak_memory_usage=torch.cuda.max_memory_allocated(self.device) / 1e9)
