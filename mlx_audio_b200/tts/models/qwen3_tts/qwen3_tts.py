"""Qwen3-TTS generation loop on H100 (reference: tts/models/qwen3_tts/qwen3_tts.py).

Covers the base path of ``Model.generate`` (qwen3_tts.py:1122-1575): input assembly from token ids
(``_prepare_generation_inputs`` :326-484 after the host tokenizer, with x-vector cloning through ``speaker_encoder.py``), the per-frame
loop (:1323-1404) with ``_sample_token`` (:805-860), and ``_decode_chunk`` (:1017-1048) through the speech tokenizer; and in-context
voice cloning from reference audio + its transcript (``_generate_icl`` :2200-2510): the speech-tokenizer encoder turns the reference into
codes, one prompt row per reference frame (``_prepare_icl_generation_inputs`` :606-803), the same frame loop, and a joint decode of
[reference | generated] codes with the reference's share cut off (``_decode_icl_generated_codes`` :1085-1112).
``batch_generate`` (:1577-2060) routes a batch of texts to the continuous-batching session, to the static batch loop with one shared ICL
reference (per-row frame caps, joint decodes as one decoder batch), or to the batch stream (a chunk per row every interval).

One frame = talker step + first-codebook sample + 15 code-predictor sub-steps (each with its sampler) + next-input
embedding sum: ~700 small launches.  They are captured ONCE into a CUDA graph; every scalar that changes between frames
(KV length, trailing-text index, uniforms, seen-token set, codes, finished flags) lives in device memory, so the host only replays
the graph and tests whether every row has finished every 8th frame (the reference syncs once per frame, :1398-1400).  A single
sequence runs as a batch of one.
"""
from __future__ import annotations

import time
from pathlib import Path
from typing import Dict, List, Optional

import torch

from .... import ops
from ..base import BatchGenerationResult, GenerationResult
from .config import ModelConfig
from .speaker_encoder import Qwen3TTSSpeakerEncoder
from .speech_tokenizer import Qwen3TTSSpeechTokenizer
from .talker import Qwen3TTSTalkerForConditionalGeneration


def format_duration(seconds: float) -> str:
    """qwen3_tts.py:160-165."""
    hours = int(seconds // 3600)
    minutes = int((seconds % 3600) // 60)
    secs = int(seconds % 60)
    ms = int((seconds % 1) * 1000)
    return f"{hours:02d}:{minutes:02d}:{secs:02d}.{ms:03d}"


_MEL_CACHE = {}


def mel_spectrogram(audio, n_fft: int = 1024, num_mels: int = 128, sample_rate: int = 24000, hop_size: int = 256,
                    win_size: int = 1024, fmin: float = 0.0, fmax: float = 12000.0, device="cuda") -> torch.Tensor:
    """qwen3_tts.py:64-120 (speaker-encoder front end): manual reflect pad of (n_fft-hop)/2, STFT (center=False, Hann),
    sqrt(|X|^2 + 1e-9) @ slaney-mel^T, log(clip(., 1e-5)).  [n] or [B, n] -> [B, frames, num_mels]: one launch for the batch
    (``ops.spk_logmel``), which implements the speaker encoder's configuration (1024 / 256 / 1024) only."""
    from .... import dsp
    if (n_fft, hop_size, win_size) != (1024, 256, 1024):
        raise NotImplementedError("mel_spectrogram: the speaker log-mel kernel covers n_fft = win_size = 1024, hop_size = 256")
    on_dev = isinstance(audio, torch.Tensor) and audio.is_cuda
    a = (audio.float() if on_dev else torch.as_tensor(audio, dtype=torch.float32)).to(device)          # host samples: one copy in
    if a.dim() == 1:
        a = a[None]
    a = a.contiguous()
    key = (a.device, num_mels, sample_rate, float(fmin), float(fmax))
    if key not in _MEL_CACHE:
        basis = dsp.mel_filters(sample_rate=sample_rate, n_fft=n_fft, n_mels=num_mels, f_min=fmin, f_max=fmax, norm="slaney", mel_scale="slaney")
        window = dsp._resolve_window("hann", win_size)
        _MEL_CACHE[key] = (torch.as_tensor(window, dtype=torch.float32).to(a.device).contiguous(),
                           torch.as_tensor(basis, dtype=torch.float32).to(a.device).contiguous())
    window, basis = _MEL_CACHE[key]
    return ops.spk_logmel(a, window, basis)


class _FrameState:
    """The device buffers ``Model._frame`` reads and writes for B rows: ``trailing`` [B, n, H] text rows, ``pad`` [H], ``suppress`` [V].
    How the talker addresses its cache is the one difference between callers: a static loop appends at the talker's device offset,
    with ``_kv_start`` int32 [B] left-padding counts (None: none); a batch session sets ``_base_rows`` int32 [B] (each row's cache
    length) and ``_slot`` (its cache slot)."""

    def __init__(self, B: int, G: int, trailing: torch.Tensor, pad: torch.Tensor, suppress: torch.Tensor):
        dev, H = pad.device, pad.numel()
        self._kv_start = self._base_rows = self._slot = None
        self._trailing, self._pad, self._suppress = trailing, pad, suppress
        self._u = torch.zeros(G, B, device=dev)
        self._seen = torch.zeros(B, suppress.numel(), dtype=torch.uint8, device=dev)
        self._codes = torch.zeros(B, G, dtype=torch.int64, device=dev)
        self._finished = torch.zeros(B, dtype=torch.uint8, device=dev)
        self._tidx = torch.zeros(B, dtype=torch.int32, device=dev)
        self._x_in = torch.zeros(B, 1, H, device=dev)
        self._cp_in0 = torch.zeros(B, 2, H, device=dev)
        self._cp_in = torch.zeros(B, H, device=dev)
        self._err = torch.zeros(1, dtype=torch.int32, device=dev)


def _capture_frame(frame, bufs):
    """Capture ``frame()`` as a CUDA graph; returns (graph, launches per frame).  The frame first runs once eagerly, which loads the
    S = 1 kernels and counts its launches, and ``bufs`` (the device buffers a frame advances) are restored before the capture.  Capture
    records the kernels without running them, so the buffers still hold the pre-frame state afterwards; host-side mirrors (the
    talker's ``offset``) are the caller's to reset."""
    dev = bufs[0].device
    torch.cuda.synchronize(dev)
    saved = [b.clone() for b in bufs]
    l0 = ops.LAUNCHES[0]
    frame()
    launches = ops.LAUNCHES[0] - l0
    for b, s in zip(bufs, saved):
        b.copy_(s)
    torch.cuda.synchronize(dev)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        frame()
    return graph, launches


class Model:
    def __init__(self, config: ModelConfig, device="cuda"):
        self.config = config
        self.device = torch.device(device)
        self.talker = Qwen3TTSTalkerForConditionalGeneration(config.talker_config, device)
        # ECAPA-TDNN speaker encoder for x-vector voice cloning: base models only, as in the reference (qwen3_tts.py:178-182)
        self.speaker_encoder = Qwen3TTSSpeakerEncoder(config.speaker_encoder_config, device) \
            if getattr(config, "tts_model_type", "base") == "base" else None
        self.talker_dtype = torch.float32     # the talker checkpoint's dtype (weights are held in fp32; the x-vector is rounded to it)
        self.speech_tokenizer_has_encoder = False   # speech_tokenizer/config.json has an encoder_config (the ICL route's condition)
        self.speech_tokenizer: Optional[Qwen3TTSSpeechTokenizer] = None
        self.tokenizer = None
        self.generate_config = None
        tc = config.talker_config
        self.supported_speakers = list(tc.spk_id.keys()) if tc.spk_id else []
        self.supported_languages = ["auto"] + [l for l in (tc.codec_language_id or {}) if "dialect" not in l]
        self._graph = None
        self._icl_cache = {}        # (ref_text, (ref_audio size, ref_audio sum)) -> (ref codes [1, 16, T], ref ids) (qwen3_tts.py:639-664)

    def get_supported_speakers(self):
        return self.supported_speakers

    def get_supported_languages(self):
        return self.supported_languages

    @property
    def sample_rate(self) -> int:
        return self.config.sample_rate

    @property
    def model_type(self) -> str:
        return self.config.model_type

    def load_weights(self, weights, strict: bool = True):
        """``weights`` (dict or list of pairs) with the checkpoint's ``talker.`` prefix (stripped here, talker.py:825-839)."""
        weights = dict(weights)
        talker_w = self.talker.sanitize(weights)
        floats = [v.dtype for v in talker_w.values() if isinstance(v, torch.Tensor) and v.is_floating_point()]
        if floats:
            self.talker_dtype = floats[0]
        self.talker.load_weights(talker_w)
        spk = {k: v for k, v in weights.items() if k.startswith("speaker_encoder.")}
        if self.speaker_encoder is not None and spk:
            self.speaker_encoder.load_weights(self.speaker_encoder.sanitize(spk))
        t = self.talker
        self._tabs_all = ops.EmbedTables([t.codec_embedding] + t.code_predictor.codec_embedding)
        self._tab0 = ops.EmbedTables([t.codec_embedding])
        self._tab_cp = [ops.EmbedTables([e]) for e in t.code_predictor.codec_embedding]
        return self

    def load_speech_tokenizer(self, speech_tokenizer: Qwen3TTSSpeechTokenizer):
        self.speech_tokenizer = speech_tokenizer

    def load_generate_config(self, generate_config: dict):
        self.generate_config = generate_config

    def eval(self):
        return self

    @staticmethod
    def sanitize(weights):
        """qwen3_tts.py:2914-2935: drop ``position_ids``; conv weights [out, in, K] -> [out, K, in] unless already MLX-layout."""
        from .speech_tokenizer import check_array_shape_qwen3
        out = {}
        for k, v in weights.items():
            if "position_ids" in k:
                continue
            if ("conv" in k or "speaker_encoder.fc" in k) and "weight" in k and v.dim() == 3:
                v = v if check_array_shape_qwen3(v) else v.permute(0, 2, 1)
            out[k] = v
        return out

    @classmethod
    def post_load_hook(cls, model: "Model", model_path):
        """qwen3_tts.py:2818-2911: HF tokenizer (when its files are present), ``speech_tokenizer/`` sub-model, generation config."""
        import json
        from pathlib import Path
        from .config import Qwen3TTSTokenizerConfig, Qwen3TTSTokenizerDecoderConfig, Qwen3TTSTokenizerEncoderConfig, filter_dict_for_dataclass
        from .speech_tokenizer import Qwen3TTSSpeechTokenizerEncoder
        model_path = Path(model_path)
        try:
            from transformers import AutoTokenizer
            model.tokenizer = AutoTokenizer.from_pretrained(str(model_path))
        except Exception as e:                                           # same behaviour as the reference: warn and continue
            print(f"Warning: Could not load tokenizer: {e}")
        st_path = model_path / "speech_tokenizer"
        if st_path.exists():
            from safetensors.torch import load_file
            d = json.load(open(st_path / "config.json"))
            model.speech_tokenizer_has_encoder = "encoder_config" in d       # speech_tokenizer.py:1076-1097, read at qwen3_tts.py:2838-2854
            dec = Qwen3TTSTokenizerDecoderConfig(**filter_dict_for_dataclass(Qwen3TTSTokenizerDecoderConfig, d["decoder_config"])) \
                if "decoder_config" in d else None
            enc = Qwen3TTSTokenizerEncoderConfig(**filter_dict_for_dataclass(Qwen3TTSTokenizerEncoderConfig, d["encoder_config"])) \
                if "encoder_config" in d else None
            tc = Qwen3TTSTokenizerConfig(decoder_config=dec, encoder_config=enc)
            for k, v in d.items():
                if k not in ("decoder_config", "encoder_config") and hasattr(tc, k):
                    setattr(tc, k, v)
            w = {}
            for wf in sorted(st_path.glob("*.safetensors")):
                w.update(load_file(str(wf)))
            if w:
                st = Qwen3TTSSpeechTokenizer(tc, model.device).load_weights({**Qwen3TTSSpeechTokenizer.sanitize(w),
                                                                             **Qwen3TTSSpeechTokenizerEncoder.sanitize(w)})
                model.load_speech_tokenizer(st)
        gen = model_path / "generation_config.json"
        if gen.exists():
            model.load_generate_config(json.load(open(gen)))
        return model

    # ------------------------------------------------------------------ input assembly
    @torch.no_grad()
    def prepare_generation_inputs_from_ids(self, input_ids, language_id: Optional[int] = None, speaker_id=None, speaker_embed=None,
                                           instruct_ids=None):
        """qwen3_tts.py:326-484 after tokenisation: ``input_ids`` = tokenizer.encode("<|im_start|>assistant\\n{text}<|im_end|>\\n
        <|im_start|>assistant\\n").  Returns (input_embeds [1,P,H], trailing_text_hidden [1,n,H], tts_pad_embed [1,1,H])."""
        t, cfg, dev = self.talker, self.config.talker_config, self.device
        ids = torch.as_tensor(input_ids, dtype=torch.int64, device=dev).reshape(-1)
        text_embed = t.text_projection(ops.gather_rows(t.text_embedding, ids)[None])                          # [1,L,H]
        tts_bos, tts_eos, tts_pad = self._tts_embeds()
        combined = self._codec_prefix(language_id, speaker_id, speaker_embed, tts_pad, tts_bos)
        first_text = text_embed[:, 3:4] + self._codec_rows([cfg.codec_bos_id])
        parts = [text_embed[:, :3], combined, first_text]
        if instruct_ids is not None:                                      # "<|im_start|>user\n{instruct}<|im_end|>\n" (:452-458,473-476)
            iid = torch.as_tensor(instruct_ids, dtype=torch.int64, device=dev).reshape(-1)
            parts = [t.text_projection(ops.gather_rows(t.text_embedding, iid)[None])] + parts
        input_embeds = torch.cat(parts, dim=1).contiguous()
        trailing = torch.cat([text_embed[:, 4:-5], tts_eos], dim=1).contiguous()
        return input_embeds, trailing, tts_pad.contiguous()

    def _tts_embeds(self):
        """Projected (tts_bos, tts_eos, tts_pad) text embeddings, each [1, 1, H]."""
        t, dev = self.talker, self.device
        tts_ids = torch.tensor([self.config.tts_bos_token_id, self.config.tts_eos_token_id, self.config.tts_pad_token_id], device=dev)
        tts = t.text_projection(ops.gather_rows(t.text_embedding, tts_ids)[None])
        return tts[:, 0:1], tts[:, 1:2], tts[:, 2:3]

    def _codec_rows(self, ids) -> torch.Tensor:
        return ops.gather_rows(self.talker.codec_embedding, torch.tensor(ids, device=self.device))[None]

    def _codec_prefix(self, language_id, speaker_id, speaker_embed, tts_pad, tts_bos) -> torch.Tensor:
        """The rows between the role and the text (qwen3_tts.py:416-450, 748-796): think / language ids, speaker row, pad, overlaid with
        tts_pad ... tts_bos on the text side.  [1, n, H]"""
        t, cfg, dev = self.talker, self.config.talker_config, self.device
        if speaker_embed is None and speaker_id is not None:
            speaker_embed = ops.gather_rows(t.codec_embedding, torch.tensor([int(speaker_id)], device=dev))[None]
        elif speaker_embed is not None and self.talker_dtype != torch.float32:
            # the speaker encoder runs in fp32; the reference casts its output to the talker's dtype before the prefix (qwen3_tts.py:429-432)
            speaker_embed = torch.as_tensor(speaker_embed, device=dev).to(self.talker_dtype)
        if language_id is None:
            prefill = [cfg.codec_nothink_id, cfg.codec_think_bos_id, cfg.codec_think_eos_id]
        else:
            prefill = [cfg.codec_think_id, cfg.codec_think_bos_id, int(language_id), cfg.codec_think_eos_id]
        codec = self._codec_rows(prefill)
        suffix = self._codec_rows([cfg.codec_pad_id])
        parts = [codec] + ([speaker_embed.reshape(1, 1, -1).float()] if speaker_embed is not None else []) + [suffix]
        codec = torch.cat(parts, dim=1)
        return torch.cat([tts_pad.expand(1, codec.shape[1] - 1, -1), tts_bos], dim=1) + codec

    @torch.no_grad()
    def prepare_icl_generation_inputs_from_ids(self, target_ids, ref_ids, ref_codes, language_id: Optional[int] = None, speaker_embed=None):
        """_prepare_icl_generation_inputs (qwen3_tts.py:606-803) after tokenisation and reference encoding.  ``target_ids`` = ids of
        "<|im_start|>assistant\n{text}<|im_end|>\n<|im_start|>assistant\n", ``ref_ids`` = ids of "<|im_start|>assistant\n{ref_text}<|im_end|>\n",
        ``ref_codes`` [1, 16, T_ref] from the speech-tokenizer encoder, ``speaker_embed`` [1, H] (x-vector) or None.  Prompt = role,
        codec prefix, then every text row (reference transcript + target text + tts_eos, each + codec_pad), then the codec-bos row and one
        row per reference frame (tts_pad + sum_g table_g[code_g]).  Returns (input_embeds [1, P, H], trailing = tts_pad, tts_pad)."""
        t, cfg, dev = self.talker, self.config.talker_config, self.device
        target = torch.as_tensor(target_ids, dtype=torch.int64, device=dev).reshape(-1)
        ref = torch.as_tensor(ref_ids, dtype=torch.int64, device=dev).reshape(-1)
        tts_bos, tts_eos, tts_pad = self._tts_embeds()
        text = t.text_projection(ops.gather_rows(t.text_embedding, torch.cat([ref[3:-2], target[3:-5]]))[None])
        text = torch.cat([text, tts_eos], dim=1) + self._codec_rows([cfg.codec_pad_id])
        codes = torch.as_tensor(ref_codes, dtype=torch.int64).to(dev)[0].transpose(0, 1).contiguous()        # [T_ref, 16]
        ref_rows = ops.embed_sum(codes, self._tabs_all, pad=tts_pad.reshape(-1).contiguous())[None]          # tts_pad + sum_g table_g[code_g]
        bos = self._codec_rows([cfg.codec_bos_id]) + tts_pad
        role = t.text_projection(ops.gather_rows(t.text_embedding, target[:3])[None])
        combined = self._codec_prefix(language_id, None, speaker_embed, tts_pad, tts_bos)
        input_embeds = torch.cat([role, combined, text, bos, ref_rows], dim=1).contiguous()
        return input_embeds, tts_pad.contiguous(), tts_pad.contiguous()

    @torch.no_grad()
    def encode_reference(self, ref_audio) -> torch.Tensor:
        """24 kHz reference samples [n] (or [1, n], [1, 1, n]) -> its codes [1, 16, ceil(n / 1920)] (qwen3_tts.py:644-652)."""
        if self.speech_tokenizer is None or not self.speech_tokenizer.has_encoder:
            raise NotImplementedError("in-context (ICL) voice cloning needs the speech tokenizer's encoder weights, which are not loaded; "
                                      "pass ref_audio without ref_text for x-vector cloning")
        a = ref_audio if isinstance(ref_audio, torch.Tensor) else torch.as_tensor(ref_audio)
        return self.speech_tokenizer.encode(a.to(self.device).float().reshape(1, 1, -1))

    def extract_speaker_embedding(self, audio, sr: int = 24000) -> torch.Tensor:
        """qwen3_tts.py:285-324: 24 kHz samples [n] or [B, n] -> x-vector [B, enc_dim] (float32): log-mel front end + ECAPA-TDNN."""
        if sr != 24000:
            raise ValueError("Only 24kHz audio is supported for speaker embedding extraction")
        if self.speaker_encoder is None:
            raise ValueError("Speaker encoder not available for this model type")
        mels = mel_spectrogram(audio, n_fft=1024, num_mels=128, sample_rate=24000, hop_size=256, win_size=1024, fmin=0, fmax=12000,
                               device=self.device)
        return self.speaker_encoder(mels)

    def _prepare_generation_inputs(self, text: str, language: str = "auto", speaker: Optional[str] = None, instruct: Optional[str] = None,
                                   ref_audio=None):
        """qwen3_tts.py:326-484: tokenise with the chat template, resolve speaker / language / dialect ids from the config; with
        ``ref_audio`` (base models) the x-vector of the reference audio takes the speaker row (it wins over ``speaker``, whose dialect
        override still applies)."""
        if self.tokenizer is None:
            raise ValueError("Tokenizer not loaded. Call post_load_hook first.")
        cfg = self.config.talker_config
        ids = self.tokenizer.encode(f"<|im_start|>assistant\n{text}<|im_end|>\n<|im_start|>assistant\n")
        speaker_id = None
        if speaker and speaker.lower() in (cfg.spk_id or {}):
            sid = cfg.spk_id[speaker.lower()]
            speaker_id = sid[0] if isinstance(sid, (list, tuple)) else sid
        language_id = None
        if language.lower() != "auto" and cfg.codec_language_id and language.lower() in cfg.codec_language_id:
            language_id = cfg.codec_language_id[language.lower()]
        if language.lower() in ("chinese", "auto") and speaker and speaker.lower() in (cfg.spk_is_dialect or {}) \
                and cfg.spk_is_dialect[speaker.lower()]:
            dialect = cfg.spk_is_dialect[speaker.lower()]
            if dialect in (cfg.codec_language_id or {}):
                language_id = cfg.codec_language_id[dialect]
        instruct_ids = self.tokenizer.encode(f"<|im_start|>user\n{instruct}<|im_end|>\n") if instruct else None
        speaker_embed = None
        if ref_audio is not None and self.speaker_encoder is not None:
            speaker_embed = self.extract_speaker_embedding(ref_audio)
        return self.prepare_generation_inputs_from_ids(ids, language_id, speaker_id, speaker_embed=speaker_embed, instruct_ids=instruct_ids)

    def _suppress_codec_tokens(self, eos_token_id: int):
        """qwen3_tts.py:927-933."""
        cfg = self.config.talker_config
        return [i for i in range(cfg.vocab_size - 1024, cfg.vocab_size) if i != eos_token_id]

    # ------------------------------------------------------------------ frame loop
    def _frame(self, x_in: torch.Tensor, sp, st: _FrameState) -> None:
        """One pass of the loop body qwen3_tts.py:1323-1398 for every row of ``st``, with the batch loop's rules (qwen3_tts.py:1880-1912):
        a finished row samples EOS, and each row reads its own trailing-text row.  Results land in the buffers of ``st``."""
        t, cp = self.talker, self.talker.code_predictor
        g = self.config.talker_config.num_code_groups
        if st._base_rows is None:
            logits, hidden = t(x_in, use_device_offset=True, kv_start=st._kv_start)
        else:
            logits, hidden = t(x_in, base_rows=st._base_rows, slot=st._slot)
        ops.sample_token(logits[:, -1], temperature=sp["temperature"], top_k=sp["top_k"], top_p=sp["top_p"], u=st._u[0],
                         suppress_mask=st._suppress, seen=st._seen, repetition_penalty=sp["repetition_penalty"], mark_seen=True,
                         out=st._codes[:, 0], finished=st._finished, eos=sp["eos"])
        inp0 = st._cp_in0                                                                    # [B,2,H]: (hidden, embed(token 0))
        ops.copy2d(hidden[:, -1], inp0[:, 0])
        ops.embed_sum(st._codes[:, 0:1], self._tab0, out=inp0[:, 1], err=st._err)
        for ci in range(g - 1):
            if ci == 0:
                lg = cp(inp0, 0, 0)
            else:
                e = ops.embed_sum(st._codes[:, ci:ci + 1], self._tab_cp[ci - 1], out=st._cp_in, err=st._err)
                lg = cp(e[:, None], ci + 1, ci)
            ops.sample_token(lg[:, -1], temperature=sp["temperature"], top_k=sp["top_k"], top_p=sp["top_p"], u=st._u[ci + 1],
                             out=st._codes[:, ci + 1])
        # per-row trailing index, clamp-pad, advance unfinished rows (qwen3_tts.py:1903-1912)
        ops.embed_sum(st._codes, self._tabs_all, text=st._trailing, pad=st._pad, out=st._x_in[:, 0], err=st._err, tidx=st._tidx,
                      finished=st._finished)

    def _uniform_stream(self, seed):
        """Generator the sampler's uniforms are drawn from.  ``seed=None`` continues ONE stream owned by the model, so successive
        segments and calls see fresh draws the way the reference's global ``mx.random`` state advances (qwen3_tts.py:805-860);
        an integer starts a reproducible stream for this call only."""
        if seed is not None:
            return torch.Generator(device=self.device).manual_seed(int(seed))
        if getattr(self, "_rng", None) is None:
            self._rng = torch.Generator(device=self.device)
            self._rng.seed()
        return self._rng

    @torch.no_grad()
    def generate_codes(self, input_embeds, trailing_text_hidden, tts_pad_embed, *, batch_mode: bool = False,
                       trailing_rule: Optional[str] = None, **kw):
        """The generation loop of Model.generate for B prompts (a single sequence is a batch of one): int64 codes [B, n, 16], each
        row's frames up to (not including) its EOS or cap and code 0 after its end (the convention of batch_generate / batch_decode).
        ``u`` [max_tokens, 16, B] uniforms in [0,1) (drawn from ``seed`` when omitted; parity tests inject them).

        ``batch_mode`` (implied by ``left_padding`` or ``caps``) returns (codes, lengths [B]) and defaults to the loop of
        ``batch_generate``'s stream (qwen3_tts.py:1861-1935): ``left_padding`` [B] rows of zero embeddings in front of shorter prompts
        (masked keys, positions from cumsum(mask) - 1), ``trailing_text_hidden`` [B, n, H] right-padded with the pad embedding, the
        clamp-pad trailing rule.  ``trailing_rule="standard"``, the default otherwise, is the rule of Model.generate and of the default
        batch path, where every row behaves as a single sequence (continuous_batching.py:261-278: text while its index is inside the
        trailing text, pad afterwards)."""
        batch_mode = batch_mode or kw.get("left_padding") is not None or kw.get("caps") is not None
        codes, _, lengths, _ = next(self._frame_iter(input_embeds, trailing_text_hidden, tts_pad_embed,
                                                     trailing_rule=trailing_rule or ("clamp_pad" if batch_mode else "standard"), **kw))
        return (codes, lengths) if batch_mode else codes

    @torch.no_grad()
    def _frame_iter(self, input_embeds, trailing_text_hidden, tts_pad_embed, *, max_tokens: int = 4096, temperature: float = 0.9,
                    top_k: int = 50, top_p: float = 1.0, repetition_penalty: float = 1.05, u=None, seed: int = 0,
                    use_graph: bool = True, left_padding=None, trailing_rule: str = "clamp_pad", caps=None,
                    emit_every: Optional[int] = None):
        """The loop of ``generate_codes`` as a generator of (out, n, lengths [B] on the host, done); its last item, and without
        ``emit_every`` its only one, has ``done`` set and ``out`` = codes [B, n, 16] with n the longest row.  Finished rows are
        forced to EOS and masked on the device; ``trailing_rule="standard"`` appends one pad row to the trailing text so that the
        kernel's clamp lands on it.  ``caps`` [B] are per-row frame caps (the ICL rule of qwen3_tts.py:1818-1823, 1925-1932: a row that
        has recorded its cap is finished, and forced to EOS from the next frame on); rows without caps get ``max_tokens``.  With
        ``emit_every`` = k the loop also yields after every k-th frame -- ``out`` [B, max_tokens, 16] is the device buffer whose first
        n frames are final; rows advance in lockstep, so a row can only complete a stream chunk there -- unless every row has
        finished, in which case the reference breaks before emitting (:1913-1932)."""
        t, cfg, dev = self.talker, self.config.talker_config, self.device
        x = input_embeds.to(dev).float().contiguous()
        B, P, H = x.shape
        g, V = cfg.num_code_groups, cfg.vocab_size
        eos = cfg.codec_eos_token_id
        if trailing_rule not in ("clamp_pad", "standard"):
            raise ValueError(f"trailing_rule must be 'clamp_pad' or 'standard', got {trailing_rule!r}")
        capped = caps is not None
        caps = [min(int(c), max_tokens) for c in caps] if capped else [max_tokens] * B
        n_steps = max(caps)                                      # every row has finished by then: the cache needs no more rows
        if u is None:
            u = torch.rand(max_tokens, g, B, device=dev, generator=self._uniform_stream(seed))
        u = u.to(dev).float().contiguous()
        sp = {"temperature": float(temperature), "top_k": int(top_k), "top_p": float(top_p), "repetition_penalty": float(repetition_penalty),
              "eos": int(eos)}
        t.reset_cache(B, P + n_steps + 1)
        pad = tts_pad_embed.to(dev).float().reshape(-1).contiguous()
        trailing = trailing_text_hidden.to(dev).float().expand(B, -1, -1)
        if trailing_rule == "standard":
            trailing = torch.cat([trailing, pad.reshape(1, 1, H).expand(B, 1, H)], dim=1)
        suppress = torch.zeros(V, device=dev)
        suppress[torch.tensor(self._suppress_codec_tokens(eos), device=dev)] = float("-inf")
        st = _FrameState(B, g, trailing.contiguous(), pad, suppress)
        if left_padding is not None and any(int(v) for v in left_padding):
            st._kv_start = torch.tensor([int(v) for v in left_padding], dtype=torch.int32, device=dev)
        out = torch.zeros(B, max_tokens, g, dtype=torch.int64, device=dev)
        lengths = torch.zeros(B, dtype=torch.int64, device=dev)
        caps_dev = torch.tensor(caps, dtype=torch.int64, device=dev)
        cap_hit = torch.zeros(B, dtype=torch.bool, device=dev)
        frame = lambda: self._frame(st._x_in, sp, st)
        n = 0
        graph = None
        for step in range(n_steps):
            st._u.copy_(u[step])
            if step == 0:
                self._frame(x, sp, st)                                               # prefill frame (S = P rows), eager
            elif not use_graph:
                frame()
            else:
                if graph is None:
                    # warm-up on a side stream is not needed: every kernel has already run once in the prefill frame except
                    # the S = 1 GEMV variants, which the eager frame of the capture launches for the first time.
                    graph, launches = _capture_frame(frame, [t.offset_dev, st._seen, st._codes, st._x_in, st._finished, st._tidx])
                graph.replay()
                t.offset = P + step                                                  # the host mirror, which the capture advanced too
                ops.LAUNCHES[0] += launches
            # No per-frame host read: a finished row is masked on the device (its frame keeps the zeros `out` starts with, its length
            # stops growing) and the all-finished test is a sync every 8th frame only -- the frames replayed past the last EOS record
            # nothing.  (One .cpu() per frame held the loop at ~12 ms per frame; the graph itself replays in under 5.)
            fin = st._finished.bool()
            out[:, n] = torch.where(fin[:, None], out[:, n], st._codes)
            lengths += (~fin).to(torch.int64)
            st._finished.bitwise_or_(torch.ge(lengths, caps_dev, out=cap_hit))
            n += 1
            if emit_every and n % emit_every == 0:
                state = torch.cat([lengths, st._finished.to(torch.int64)]).cpu()          # the one read per chunk boundary
                # without caps a row is never finished by max_tokens in the reference: the last frame still emits
                if bool(state[B:].all()) and (capped or n < n_steps):
                    break
                yield out, n, state[:B], False
            elif (step & 7) == 7 and bool(st._finished.all()):
                break
        if int(st._err.item()) != 0:
            raise ValueError("generate_codes: a sampled code indexed outside its embedding table")
        self._graph = graph
        lengths = lengths.cpu()
        n = int(lengths.max()) if lengths.numel() else 0
        yield out[:, :n], n, lengths, True

    # ------------------------------------------------------------------ batch generation
    def supports_tts_batch(self, *, stream: bool = False, voice: Optional[str] = None, instruct: Optional[str] = None, ref_audio=None,
                           ref_text: Optional[str] = None, speed: Optional[float] = 1.0, pitch: Optional[float] = 1.0, **kwargs) -> bool:
        """qwen3_tts.py:215-251: whether a request with these settings may share a batch."""
        if stream or speed not in (None, 1.0) or pitch not in (None, 1.0):
            return False
        kind = getattr(self.config, "tts_model_type", "base")
        if ref_audio is not None or ref_text is not None:
            return (kind == "base" and ref_audio is not None and ref_text is not None and voice is None and instruct is None
                    and self.speech_tokenizer is not None and self.speech_tokenizer.has_encoder)
        if kind not in ("base", "custom_voice"):
            return False
        if kind == "base" and instruct:
            return False
        if kind == "custom_voice" and not voice:
            return False
        return True

    def supports_tts_continuous_batch(self, **kwargs) -> bool:
        """qwen3_tts.py:253-256: as ``supports_tts_batch``, but never for reference-audio requests."""
        if kwargs.get("ref_audio") is not None or kwargs.get("ref_text") is not None:
            return False
        return self.supports_tts_batch(**kwargs)

    def create_tts_batch_session(self, options):
        """qwen3_tts.py:1114-1120: a step-wise continuous-batching session (``continuous_batching.Qwen3TTSBatchSession``)."""
        from .continuous_batching import Qwen3TTSBatchSession
        return Qwen3TTSBatchSession(self, options)

    @torch.no_grad()
    def prepare_batch_inputs_from_ids(self, ids_list, language_id=None, speaker_ids=None, instruct_ids=None):
        """_prepare_batch_inputs (qwen3_tts.py:486-604) after tokenisation: left-pad the prompts with zero rows, right-pad the trailing
        text with the pad embedding.  Returns (input_embeds [B,P,H], trailing [B,n,H], tts_pad [1,1,H], left_padding [B])."""
        per = [self.prepare_generation_inputs_from_ids(ids, language_id, None if speaker_ids is None else speaker_ids[i],
                                                       instruct_ids=None if instruct_ids is None else instruct_ids[i])
               for i, ids in enumerate(ids_list)]
        return self._pad_batch(per)

    def _pad_batch(self, per):
        """Per-row (input_embeds [1,P_b,H], trailing [1,n_b,H], tts_pad [1,1,H]) -> the padded batch of ``_prepare_batch_inputs``."""
        pad = per[0][2]
        pmax = max(e.shape[1] for e, _, _ in per)
        tmax = max(tr.shape[1] for _, tr, _ in per)
        H = pad.shape[-1]
        x = torch.zeros(len(per), pmax, H, device=self.device)
        trailing = pad.reshape(1, 1, H).expand(len(per), tmax, H).clone()
        left = []
        for i, (e, tr, _) in enumerate(per):
            left.append(pmax - e.shape[1])
            x[i, pmax - e.shape[1]:] = e[0]
            trailing[i, : tr.shape[1]] = tr[0]
        return x, trailing, pad, left

    def batch_generate_from_ids(self, ids_list, *, language_id=None, speaker_ids=None, temperature: float = 0.9, max_tokens: int = 4096,
                                top_k: int = 50, top_p: float = 1.0, repetition_penalty: float = 1.05, seed: int = 0, u=None,
                                stream: bool = False, streaming_interval: float = 2.0, **kwargs):
        """``Model.batch_generate`` (qwen3_tts.py:1651-2060) for already-tokenised texts, one BatchGenerationResult per sequence.

        ``stream=False`` (the reference's default) follows its batch session (continuous_batching.py): every row generates exactly what it
        would generate alone from its own uniform stream (standard trailing-text rule), and is decoded by ``_decode_generated_codes`` --
        15-frame chunks with 5 frames of left context (qwen3_tts.py:1050-1083).  ``stream=True`` follows the streaming branch
        (qwen3_tts.py:1861-2029): finished rows forced to EOS, clamp-pad trailing rule, and a chunk per row every ``streaming_interval``
        seconds of frames, then each row's remainder as its final chunk (``_stream_batch``)."""
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        t0 = time.perf_counter()
        x, trailing, pad, left = self.prepare_batch_inputs_from_ids(ids_list, language_id, speaker_ids)
        gen = dict(max_tokens=max_tokens, temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty, seed=seed,
                   u=u, left_padding=left)
        if stream:
            yield from self._stream_batch(x, trailing, pad, gen, streaming_interval, t0)
            return
        codes, lengths = self.generate_codes(x, trailing, pad, batch_mode=True, trailing_rule="standard", **gen)
        seqs = [codes[b, : int(lengths[b])] for b in range(codes.shape[0])]
        # rows of equal length share their decode launches: the chunks of _decode_generated_codes do not interact, so chunk j of every
        # row goes through the vocoder as one batch (identical samples; 8 rows x 3 chunks: 24 decoder passes -> 2)
        live = [s_ for s_ in seqs if s_.shape[0] > 0]
        by_len: Dict[int, List[int]] = {}
        for i, s_ in enumerate(live):
            by_len.setdefault(int(s_.shape[0]), []).append(i)
        audios = [None] * len(live)
        for n_, idxs in by_len.items():
            wav = self.speech_tokenizer.decoder.chunked_decode(torch.stack([live[i] for i in idxs]).transpose(1, 2), chunk_size=15, left_context_size=5)
            for j, i in enumerate(idxs):
                audios[i] = wav[j, 0]
        torch.cuda.synchronize(self.device)
        dt = time.perf_counter() - t0
        it = iter(audios)
        for b, s_ in enumerate(seqs):
            if s_.shape[0] == 0:
                continue
            yield self._batch_result(next(it), b, int(s_.shape[0]), dt)

    def _stream_batch(self, x, trailing, pad, gen: dict, streaming_interval: float, t0: float):
        """The streaming branch of the static batch loop (qwen3_tts.py:1943-2029): once a row has ``max(1, int(streaming_interval * 12.5))``
        undecoded frames it emits them, decoded by ``chunked_decode`` behind up to 25 frames of context whose samples are dropped (the
        reference hard-codes the 25); after the loop every row with undecoded frames emits them as its final chunk.  The host reads the
        row lengths only at chunk boundaries (``_frame_iter(emit_every=...)``)."""
        chunk = max(1, int(streaming_interval * 12.5))
        decoded = [0] * x.shape[0]
        for out, n, lengths, done in self._frame_iter(x, trailing, pad, emit_every=chunk, **gen):
            # in the loop the rows still running (length n) emit; at the end every row with undecoded frames does
            ends = [int(v) for v in lengths]
            rows = [b for b, e in enumerate(ends) if e > decoded[b] and (done or e == n)]
            yield from self._emit_batch_chunks(out, rows, decoded, ends, done, t0)

    def _emit_batch_chunks(self, out, rows, decoded, ends, final: bool, t0: float):
        """One stream step of ``_stream_batch``: frames [decoded[b], ends[b]) of every row b in ``rows``, in row order.  Rows with equal
        context and chunk lengths go through one ``chunked_decode`` call (at an in-loop step that is every emitting row)."""
        up = self.speech_tokenizer.decode_upsample_rate
        groups: Dict[tuple, List[int]] = {}
        for b in rows:
            groups.setdefault((min(25, decoded[b]), ends[b] - decoded[b]), []).append(b)
        audio = {}
        for (ctx, new), members in groups.items():
            codes = torch.stack([out[b, decoded[b] - ctx: ends[b]] for b in members])                  # [R, ctx + new, G]
            wav = self.speech_tokenizer.decoder.chunked_decode(codes.transpose(1, 2))[:, 0]
            for i, b in enumerate(members):
                audio[b] = wav[i, ctx * up:] if ctx * up < wav.shape[1] else wav[i]
        torch.cuda.synchronize(self.device)
        for b in rows:
            new = ends[b] - decoded[b]
            decoded[b] = ends[b]
            yield self._batch_result(audio[b], b, new, time.perf_counter() - t0, is_streaming_chunk=True, is_final_chunk=final)

    def _batch_result(self, audio, sequence_idx: int, token_count: int, seconds: float, metadata=None, **flags):
        """The BatchGenerationResult of one row's audio; a session event's ``metadata`` overrides the duration, time and memory fields."""
        m = metadata or {}
        return BatchGenerationResult(audio=audio, sequence_idx=sequence_idx, samples=int(audio.shape[0]), sample_rate=self.sample_rate,
                                     token_count=token_count,
                                     audio_duration=m.get("audio_duration", format_duration(audio.shape[0] / self.sample_rate)),
                                     processing_time_seconds=m.get("processing_time_seconds", seconds),
                                     peak_memory_usage=m.get("peak_memory_usage", torch.cuda.max_memory_allocated(self.device) / 1e9), **flags)

    # ------------------------------------------------------------------ batch_generate: requests, routes, ICL
    @staticmethod
    def _same_shared_ref_value(left, right) -> bool:
        """qwen3_tts.py:1577-1580: paths are the same reference when their strings are; arrays only when they are the same object."""
        if isinstance(left, (str, Path)) and isinstance(right, (str, Path)):
            return str(left) == str(right)
        return left is right

    @staticmethod
    def _normalize_shared_batch_refs(batch_size: int, *, ref_audio=None, ref_text: Optional[str] = None, ref_audios=None, ref_texts=None):
        """qwen3_tts.py:1582-1649: resolve one shared in-context reference (audio, transcript) for the whole batch from the scalar and the
        per-text list arguments, with the reference's errors.  Returns (ref_audio, ref_text), both None without a reference."""
        def shared_from_list(name, values):
            if values is None:
                return None
            if len(values) != batch_size:
                raise ValueError(f"{name} length ({len(values)}) must match texts length ({batch_size})")
            present = [v for v in values if v is not None]
            if not present:
                return None
            if len(present) != batch_size:
                raise ValueError(f"Qwen3-TTS batch_generate requires {name} for every text when using reference cloning")
            shared = present[0]
            for v in present[1:]:
                if not Model._same_shared_ref_value(shared, v):
                    raise ValueError(f"Qwen3-TTS batch_generate currently supports only one shared {name[:-1]} across the whole batch")
            return shared

        list_audio = shared_from_list("ref_audios", ref_audios)
        list_text = shared_from_list("ref_texts", ref_texts)
        if list_audio is not None:
            if ref_audio is not None and not Model._same_shared_ref_value(ref_audio, list_audio):
                raise ValueError("ref_audio and ref_audios must refer to the same shared reference")
            ref_audio = list_audio
        if list_text is not None:
            if ref_text is not None and ref_text != list_text:
                raise ValueError("ref_text and ref_texts must refer to the same shared reference")
            ref_text = list_text
        if ref_audio is None and ref_text is None:
            return None, None
        if ref_audio is None or ref_text is None:
            raise ValueError("Qwen3-TTS batch reference cloning requires both ref_audio and ref_text")
        if isinstance(ref_audio, (str, Path)):
            raise NotImplementedError("batch_generate: file decoding (audio_io) is outside the accelerated path; pass 24 kHz samples")
        return ref_audio, ref_text

    @staticmethod
    def _batch_request(batch_size: int, voices=None, instructs=None, ref_audio=None, ref_text=None, ref_audios=None, ref_texts=None,
                       has_encoder: bool = False):
        """The request checks of batch_generate (qwen3_tts.py:1699-1739): per-text lists of the right length, one shared reference, and
        no voices / instructs / encoder-less speech tokenizer with it.  Returns (voices, instructs, ref_audio, ref_text, use_icl)."""
        if voices is None:
            voices = [None] * batch_size
        elif len(voices) != batch_size:
            raise ValueError(f"voices length ({len(voices)}) must match texts length ({batch_size})")
        if instructs is None:
            instructs = [None] * batch_size
        elif len(instructs) != batch_size:
            raise ValueError(f"instructs length ({len(instructs)}) must match texts length ({batch_size})")
        ref_audio, ref_text = Model._normalize_shared_batch_refs(batch_size, ref_audio=ref_audio, ref_text=ref_text, ref_audios=ref_audios,
                                                                 ref_texts=ref_texts)
        use_icl = ref_audio is not None and ref_text is not None
        if use_icl:
            if not has_encoder:
                raise ValueError("Qwen3-TTS batch reference cloning requires a speech tokenizer encoder")
            if any(v is not None for v in voices):
                raise ValueError("Qwen3-TTS batch reference cloning does not support voices")
            if any(i is not None for i in instructs):
                raise ValueError("Qwen3-TTS batch reference cloning does not support instructs")
        return voices, instructs, ref_audio, ref_text, use_icl

    def batch_generate_icl_from_ids(self, target_ids_list, ref_ids, *, ref_audio=None, ref_codes=None, speaker_embed=None, language_id=None,
                                    row_max_tokens=None, temperature: float = 0.9, max_tokens: int = 4096, top_k: int = 50, top_p: float = 1.0,
                                    repetition_penalty: float = 1.5, seed: int = 0, u=None, stream: bool = False,
                                    streaming_interval: float = 2.0, **kwargs):
        """The in-context branch of ``Model.batch_generate`` (qwen3_tts.py:1798-2060) for already-tokenised texts sharing one reference
        (ids as in ``prepare_icl_generation_inputs_from_ids``).  The reference is encoded (``ref_codes`` [1, 16, T_ref], unless given) and
        its x-vector computed once for the call; every row gets its own in-context prompt, the prompts are left-padded into one batch, and
        row b stops on EOS or after ``row_max_tokens[b]`` frames (default ``max_tokens``).  ``u`` [max_tokens, 16, B] injects the uniforms.
        Yields one BatchGenerationResult per row with frames: [ref | generated] decoded together (one decoder batch for all rows), trimmed
        to the valid length, the reference's share cut off; or with ``stream=True`` chunks of the generated codes (``_stream_batch``)."""
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        t0 = time.perf_counter()
        ref_codes, speaker_embed = self._resolve_icl_reference("batch_generate_icl_from_ids", ref_audio, ref_codes, speaker_embed)
        per = [self.prepare_icl_generation_inputs_from_ids(ids, ref_ids, ref_codes, language_id, speaker_embed) for ids in target_ids_list]
        x, trailing, pad, left = self._pad_batch(per)
        gen = dict(max_tokens=max_tokens, temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty, seed=seed,
                   u=u, left_padding=left, caps=row_max_tokens if row_max_tokens is not None else [max_tokens] * len(per))
        if stream:
            yield from self._stream_batch(x, trailing, pad, gen, streaming_interval, t0)
            return
        codes, lengths = self.generate_codes(x, trailing, pad, batch_mode=True, **gen)
        dt = time.perf_counter() - t0
        rows = [b for b in range(codes.shape[0]) if int(lengths[b]) > 0]
        audios = self._decode_icl_batch([codes[b, : int(lengths[b])] for b in rows], ref_codes)
        for b, a in zip(rows, audios):
            yield self._batch_result(a, b, int(lengths[b]), dt)

    def _resolve_icl_reference(self, caller: str, ref_audio, ref_codes, speaker_embed):
        """(ref_codes, speaker_embed) of an in-context call: the reference's codes are encoded from ``ref_audio`` unless given, and its
        x-vector takes the speaker row unless ``speaker_embed`` pins one (models with a speaker encoder)."""
        if ref_codes is None:
            if ref_audio is None:
                raise ValueError(f"{caller}: pass ref_audio or ref_codes")
            ref_codes = self.encode_reference(ref_audio)
        if speaker_embed is None and ref_audio is not None and self.speaker_encoder is not None:
            speaker_embed = self.extract_speaker_embedding(ref_audio)
        return ref_codes, speaker_embed

    def _icl_reference(self, ref_audio, ref_text):
        """(ref codes [1, 16, T], transcript ids) of a reference, cached on (ref_text, (size, sum) of ref_audio) (qwen3_tts.py:639-664)."""
        a = ref_audio if isinstance(ref_audio, torch.Tensor) else torch.as_tensor(ref_audio)
        key = (ref_text, (int(a.numel()), float(a.sum())))
        if key not in self._icl_cache:
            self._icl_cache[key] = (self.encode_reference(a), self.tokenizer.encode(f"<|im_start|>assistant\n{ref_text}<|im_end|>\n"))
        return a, self._icl_cache[key]

    def _language_id(self, lang_code: str):
        cfg = self.config.talker_config
        if lang_code.lower() != "auto" and cfg.codec_language_id and lang_code.lower() in cfg.codec_language_id:
            return cfg.codec_language_id[lang_code.lower()]
        return None

    def batch_generate(self, texts: List[str], voices: Optional[List[Optional[str]]] = None, instructs: Optional[List[Optional[str]]] = None,
                       ref_audio=None, ref_text: Optional[str] = None, ref_audios=None, ref_texts: Optional[List[Optional[str]]] = None,
                       temperature: float = 0.9, lang_code: str = "auto", max_tokens: int = 4096, top_k: int = 50, top_p: float = 1.0,
                       repetition_penalty: float = 1.05, stream: bool = False, streaming_interval: float = 2.0, streaming_context_size: int = 25,
                       verbose: bool = False, seed: Optional[int] = None, **kwargs):
        """Model.batch_generate (qwen3_tts.py:1651-2060): BatchGenerationResults for several texts generated as one batch.
        ``stream=False`` without a reference runs the continuous-batching session (:1741-1796); with one shared reference
        (``ref_audio`` + ``ref_text``, or the per-text aliases ``ref_audios`` / ``ref_texts`` naming the same reference) the in-context
        static batch (``batch_generate_icl_from_ids``), each row capped at ``min(max_tokens, max(75, 6 * len(encode(text))))`` frames and
        the repetition penalty raised to at least 1.5; ``stream=True`` the static batch with a chunk per row every ``streaming_interval``
        seconds.  ``streaming_context_size`` is accepted and, as in the reference, the stream context is 25 frames whatever it says."""
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        B = len(texts)
        if B == 0:
            return
        voices, instructs, ref_audio, ref_text, use_icl = self._batch_request(B, voices, instructs, ref_audio, ref_text, ref_audios, ref_texts,
                                                                              self.speech_tokenizer.has_encoder)
        if self.tokenizer is None:
            raise ValueError("Tokenizer not loaded. Call post_load_hook first.")
        gen = dict(temperature=temperature, max_tokens=max_tokens, top_k=top_k, top_p=top_p, seed=seed, stream=stream,
                   streaming_interval=streaming_interval)
        if use_icl:
            a, (ref_codes, ref_ids) = self._icl_reference(ref_audio, ref_text)
            target = [self.tokenizer.encode(f"<|im_start|>assistant\n{t}<|im_end|>\n<|im_start|>assistant\n") for t in texts]
            caps = [min(max_tokens, max(75, len(self.tokenizer.encode(t)) * 6)) for t in texts]      # raw text, no template (:1818-1823)
            yield from self.batch_generate_icl_from_ids(target, ref_ids, ref_audio=a, ref_codes=ref_codes, language_id=self._language_id(lang_code),
                                                        row_max_tokens=caps, repetition_penalty=max(repetition_penalty, 1.5), **gen)
            return
        if stream:
            per = [self._prepare_generation_inputs(t, language=lang_code, speaker=v, instruct=i) for t, v, i in zip(texts, voices, instructs)]
            x, trailing, pad, left = self._pad_batch(per)
            yield from self._stream_batch(x, trailing, pad, dict(max_tokens=max_tokens, temperature=temperature, top_k=top_k, top_p=top_p,
                                                                 repetition_penalty=repetition_penalty, seed=seed, left_padding=left),
                                          streaming_interval, time.perf_counter())
            return
        from ...continuous import TTSBatchItem, TTSBatchOptions
        session = self.create_tts_batch_session(TTSBatchOptions(temperature=temperature, top_p=top_p, top_k=top_k, repetition_penalty=repetition_penalty,
                                                                max_tokens=max_tokens, lang_code=lang_code, stream=False,
                                                                streaming_interval=streaming_interval, max_batch_size=B, verbose=verbose))
        session.add([TTSBatchItem(sequence_id=i, text=t, voice=voices[i], instruct=instructs[i]) for i, t in enumerate(texts)])
        t0 = time.perf_counter()
        while not session.idle:
            for ev in session.step():
                if ev.error is not None:
                    raise ev.error
                if ev.audio is None or ev.samples <= 0:
                    continue
                yield self._batch_result(ev.audio, ev.sequence_id, ev.token_count, time.perf_counter() - t0, ev.metadata,
                                         is_streaming_chunk=ev.is_streaming_chunk, is_final_chunk=ev.is_final_chunk)

    # ------------------------------------------------------------------ decode + public generate
    @torch.no_grad()
    def _decode_generated_codes(self, codes: torch.Tensor, *, decode_chunk: int = 15, decode_ctx: int = 5) -> torch.Tensor:
        """qwen3_tts.py:1050-1083: codes [n, G] of one sequence -> audio [1920 n], decoded in ``decode_chunk``-frame pieces with up to
        ``decode_ctx`` frames of left context whose samples are dropped."""
        if codes.shape[0] == 0:
            return torch.zeros(0, dtype=torch.float32, device=self.device)
        # the reference's loop is chunked_decode's loop with (15, 5) in place of (300, 25): same chunk boundaries, same "context only
        # when start > context" rule, context samples dropped (speech_tokenizer.py:932-954 vs qwen3_tts.py:1066-1078)
        return self.speech_tokenizer.decoder.chunked_decode(codes[None].transpose(1, 2), chunk_size=decode_chunk, left_context_size=decode_ctx)[0, 0]

    @torch.no_grad()
    def _decode_chunk(self, codes: torch.Tensor, chunk_tokens: int = 300) -> torch.Tensor:
        """qwen3_tts.py:1017-1048: codes [1, T, 16] -> audio [samples], trimmed to the frames whose first code is > 0."""
        chunks = list(self.speech_tokenizer.streaming_decode(codes, chunk_tokens=chunk_tokens))
        audio = torch.cat(chunks, dim=-1)[0]
        valid = int((codes[..., 0] > 0).sum().item()) * self.speech_tokenizer.decode_upsample_rate
        if 0 < valid < audio.shape[0]:
            audio = audio[:valid]
        return audio

    def _generation_result(self, audio, token_count: int, segment_idx: int, t0: float, is_streaming_chunk: bool = False,
                           is_final_chunk: bool = False, total_tokens: Optional[int] = None) -> GenerationResult:
        """The GenerationResult of ``audio`` decoded from ``token_count`` frames, timed from ``t0`` to the end of the work queued on the
        device; a stream chunk before the last also reports ``total_tokens``, the frames generated so far (qwen3_tts.py:1440-1571)."""
        torch.cuda.synchronize(self.device)
        dt = time.perf_counter() - t0
        samples = int(audio.shape[0])
        dur = samples / self.sample_rate
        audio_samples = {"samples": samples, "samples-per-sec": samples / dt if dt > 0 else 0}
        if total_tokens is not None:
            audio_samples["tokens"] = total_tokens
        return GenerationResult(audio=audio, samples=samples, sample_rate=self.sample_rate, segment_idx=segment_idx, token_count=token_count,
                                audio_duration=format_duration(dur), real_time_factor=dur / dt if dt > 0 else 0,
                                prompt={"tokens": token_count, "tokens-per-sec": token_count / dt if dt > 0 else 0}, audio_samples=audio_samples,
                                processing_time_seconds=dt, peak_memory_usage=torch.cuda.max_memory_allocated(self.device) / 1e9,
                                is_streaming_chunk=is_streaming_chunk, is_final_chunk=is_final_chunk)

    def _stream_segment(self, x, trailing, pad, segment_idx: int, streaming_interval: float, gen: dict):
        """The streaming branch of the generation loop (qwen3_tts.py:1316-1521, 2264-2446): once ``max(1, int(streaming_interval * 12.5))``
        frames are undecoded, decode them with the incremental decoder and yield a chunk; after EOS / ``max_tokens`` yield the rest (if
        any) as the final chunk.  The host reads the frame count only at chunk boundaries (``_frame_iter(emit_every=...)``).  Streamed
        audio is not trimmed to the valid length; each chunk is timed from the previous one."""
        dec = self.speech_tokenizer.decoder
        chunk = max(1, int(streaming_interval * 12.5))
        dec.reset_streaming_state()
        t0, decoded = time.perf_counter(), 0
        for out, n, lengths, done in self._frame_iter(x, trailing, pad, trailing_rule="standard", emit_every=chunk, **gen):
            end = int(lengths[0])
            if end > decoded and (done or end == n):             # in the loop only while the sequence is still running
                audio = dec.streaming_step(out[:1, decoded:end].transpose(1, 2))[0, 0]
                res = self._generation_result(audio, end - decoded, segment_idx, t0, is_streaming_chunk=True, is_final_chunk=done,
                                              total_tokens=None if done else end)
                t0, decoded = time.perf_counter(), end
                yield res
        dec.reset_streaming_state()

    def _run_segment(self, x, trailing, pad, segment_idx: int, t0: float, stream: bool, streaming_interval: float, gen: dict, decode):
        """One segment from its prepared inputs: streamed by ``_stream_segment``, or generated in full, decoded by ``decode`` (codes
        [1, n, 16] -> audio) and yielded as one GenerationResult timed from ``t0`` -- nothing when no frame was generated."""
        if stream:
            yield from self._stream_segment(x, trailing, pad, segment_idx, streaming_interval, gen)
            return
        codes = self.generate_codes(x, trailing, pad, **gen)
        if codes.shape[1] > 0:
            yield self._generation_result(decode(codes), int(codes.shape[1]), segment_idx, t0)

    def generate_from_ids(self, input_ids, *, language_id=None, speaker_id=None, temperature: float = 0.9, max_tokens: int = 4096,
                          top_k: int = 50, top_p: float = 1.0, repetition_penalty: float = 1.05, seed: int = 0, u=None,
                          stream: bool = False, streaming_interval: float = 2.0, ref_audio=None, speaker_embed=None, **kwargs):
        """``Model.generate`` (qwen3_tts.py:1122-1575) for one already-tokenised segment; yields one GenerationResult, or with
        ``stream=True`` one per ``streaming_interval`` seconds of generated frames (the last with ``is_final_chunk``).  ``ref_audio``
        (24 kHz samples, base models) = x-vector cloning: its speaker embedding takes the speaker row, as ``speaker_embed`` [1, H] does."""
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        t0 = time.perf_counter()
        if ref_audio is not None:
            if self.speaker_encoder is None:
                raise ValueError("Speaker encoder not available for this model type")
            speaker_embed = self.extract_speaker_embedding(ref_audio)
        x, trailing, pad = self.prepare_generation_inputs_from_ids(input_ids, language_id, speaker_id, speaker_embed=speaker_embed)
        gen = dict(max_tokens=max_tokens, temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty, seed=seed, u=u)
        yield from self._run_segment(x, trailing, pad, 0, t0, stream, streaming_interval, gen, self._decode_chunk)

    def generate_icl_from_ids(self, target_ids, ref_ids, *, ref_audio=None, ref_codes=None, speaker_embed=None, language_id=None,
                              temperature: float = 0.9, max_tokens: int = 4096, top_k: int = 50, top_p: float = 1.0,
                              repetition_penalty: float = 1.5, seed: int = 0, u=None, stream: bool = False, streaming_interval: float = 2.0,
                              **kwargs):
        """``_generate_icl`` (qwen3_tts.py:2200-2510) for already-tokenised texts (ids as in ``prepare_icl_generation_inputs_from_ids``).
        ``ref_codes`` [1, 16, T_ref] are the reference's codes, or encoded here from ``ref_audio``; the x-vector of ``ref_audio`` takes the
        speaker row (``speaker_embed`` [1, H] instead pins it).  Yields one GenerationResult: [ref | generated] codes decoded together,
        trimmed to the valid length and with the reference's proportional share cut off; or with ``stream=True`` one chunk per
        ``streaming_interval`` seconds of generated frames (segment 0, generated codes only)."""
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        t0 = time.perf_counter()
        ref_codes, speaker_embed = self._resolve_icl_reference("generate_icl_from_ids", ref_audio, ref_codes, speaker_embed)
        x, trailing, pad = self.prepare_icl_generation_inputs_from_ids(target_ids, ref_ids, ref_codes, language_id, speaker_embed)
        gen = dict(max_tokens=max_tokens, temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty, seed=seed, u=u)
        yield from self._run_segment(x, trailing, pad, 0, t0, stream, streaming_interval, gen,
                                     lambda codes: self._decode_icl_batch([codes[0]], ref_codes)[0])

    @torch.no_grad()
    def _decode_icl_batch(self, gen_list, ref_codes) -> List[torch.Tensor]:
        """qwen3_tts.py:1085-1112 for several rows [n_b, 16] of one reference: each row's audio is [ref | gen_b] decoded together, trimmed
        to the valid length (frames whose first code is > 0), then int(T_ref / total * samples) samples of reference cut off the front.
        The rows go through the decoder as one batch, right-padded with code 0.  Chunk boundaries count from frame 0 and the decoder is
        causal, so padding after a row's end does not reach its frames; the valid lengths and cuts are each row's own."""
        up = self.speech_tokenizer.decode_upsample_rate
        ref_t = torch.as_tensor(ref_codes, dtype=torch.int64).to(self.device)[0].transpose(0, 1)
        totals = [ref_t.shape[0] + int(c.shape[0]) for c in gen_list]
        full = torch.zeros(len(gen_list), max(totals), ref_t.shape[1], dtype=torch.int64, device=self.device)
        full[:, : ref_t.shape[0]] = ref_t
        for i, c in enumerate(gen_list):
            full[i, ref_t.shape[0]: totals[i]] = c.to(self.device)
        wav = self.speech_tokenizer.decoder.chunked_decode(full.transpose(1, 2))[:, 0]
        valid = ((full[..., 0] > 0).sum(dim=1) * up).tolist()             # padding is code 0: it never counts as valid
        audios = []
        for i, total in enumerate(totals):
            audio = wav[i, : total * up]
            if 0 < valid[i] < audio.shape[0]:
                audio = audio[: valid[i]]
            cut = int(ref_t.shape[0] / max(total, 1) * audio.shape[0])
            audios.append(audio[cut:] if 0 < cut < audio.shape[0] else audio)
        return audios

    def _generate_icl(self, text, ref_audio, ref_text, language, stream, streaming_interval, **gen):
        """_generate_icl (qwen3_tts.py:2200-2510): the text is one segment; the reference's codes (and transcript ids) are cached on
        (ref_text, (size, sum) of ref_audio), so a repeated reference does not run the encoder again (:639-664)."""
        if self.tokenizer is None:
            raise ValueError("Tokenizer not loaded. Call post_load_hook first.")
        a, (ref_codes, ref_ids) = self._icl_reference(ref_audio, ref_text)
        target_ids = self.tokenizer.encode(f"<|im_start|>assistant\n{text}<|im_end|>\n<|im_start|>assistant\n")
        yield from self.generate_icl_from_ids(target_ids, ref_ids, ref_audio=a, ref_codes=ref_codes, language_id=self._language_id(language),
                                              stream=stream, streaming_interval=streaming_interval, **gen)

    def _generate_segments(self, text, split_pattern, speaker, language, instruct, stream=False, streaming_interval=2.0, ref_audio=None, **gen):
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        # base path: segments are split AND stripped (qwen3_tts.py:1268-1271); the instruct paths pass split_pattern=None and the text as is
        segments = [t.strip() for t in text.split(split_pattern) if t.strip()] if split_pattern else [text]
        for idx, seg in enumerate(segments):
            t0 = time.perf_counter()
            x, trailing, pad = self._prepare_generation_inputs(seg, language=language, speaker=speaker, instruct=instruct, ref_audio=ref_audio)
            seg_gen = dict(gen)
            if seg_gen.get("seed") is not None:                       # a fixed seed still gives every segment its own draws
                seg_gen["seed"] = int(seg_gen["seed"]) + idx
            yield from self._run_segment(x, trailing, pad, idx, t0, stream, streaming_interval, seg_gen, self._decode_chunk)

    def generate(self, text: str, voice: Optional[str] = None, instruct: Optional[str] = None, temperature: float = 0.9, speed: float = 1.0,
                 lang_code: str = "auto", ref_audio=None, ref_text: Optional[str] = None, split_pattern: str = "\n", max_tokens: int = 4096,
                 verbose: bool = False, stream: bool = False, streaming_interval: float = 2.0, top_k: int = 50, top_p: float = 1.0,
                 repetition_penalty: float = 1.05, seed: Optional[int] = None, **kwargs):
        """Model.generate (qwen3_tts.py:1122-1575): routes on ``tts_model_type`` exactly as the reference (same errors)."""
        gen = dict(max_tokens=max_tokens, temperature=temperature, top_k=top_k, top_p=top_p, repetition_penalty=repetition_penalty, seed=seed)
        kind = getattr(self.config, "tts_model_type", "base")
        if kind == "voice_design":
            if not instruct:
                raise ValueError("VoiceDesign model requires 'instruct' to describe the voice "
                                 "(e.g., 'A cheerful young female voice with high pitch')")
            yield from self._generate_segments(text, None, None, lang_code, instruct, stream, streaming_interval, **gen)   # one utterance: no split
            return
        if kind == "custom_voice":
            if not voice:
                raise ValueError(f"CustomVoice model requires 'voice' (speaker name) (e.g., {self.supported_speakers})")
            if voice.lower() not in [s.lower() for s in self.supported_speakers]:
                raise ValueError(f"Speaker '{voice}' not supported. Available: {self.supported_speakers}")
            yield from self._generate_segments(text, None, voice, lang_code, instruct, stream, streaming_interval, **gen)
            return
        if self.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        if ref_audio is not None and ref_text is not None and (self.speech_tokenizer_has_encoder or self.speech_tokenizer.has_encoder):
            # in-context cloning (qwen3_tts.py:1227-1252) with a stronger repetition penalty; a checkpoint that declares an encoder whose
            # weights are missing raises (encode_reference) instead of silently synthesising another voice
            gen["repetition_penalty"] = max(repetition_penalty, 1.5)
            yield from self._generate_icl(text, ref_audio, ref_text, lang_code, stream, streaming_interval, **gen)
            return
        if voice is not None and voice.lower() not in [s.lower() for s in self.supported_speakers]:
            raise ValueError(f"Voice '{voice}' is not supported by this Base model. Base models have no built-in preset voices — "
                             "clone a voice by passing ref_audio and ref_text instead.")
        # ref_audio alone (or with ref_text when the speech tokenizer has no encoder): x-vector cloning on every segment (:381-383)
        yield from self._generate_segments(text, split_pattern, voice, lang_code, None, stream, streaming_interval, ref_audio=ref_audio, **gen)
