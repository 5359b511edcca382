"""Continuous batching for Qwen3-TTS on H100 (reference: tts/models/qwen3_tts/continuous_batching.py).

``Qwen3TTSBatchSession`` follows the reference session step for step: ``step()`` first advances every active request by one frame,
then admits up to ``available_slots`` pending requests (prefill + their first frame); a request finishes on EOS or after
``max_tokens`` frames and is decoded by ``Model._decode_generated_codes`` into one ``TTSBatchEvent(done=True)``.

H100 mapping.  The reference merges and re-extracts per-request KV caches every step (KVCache.merge / BatchKVCache.extract, :140,178,
309-324).  Here every request owns a SLOT: its KV rows in one talker cache [layers, slots, rows, kv], and per-slot device state
(cache length, code row, seen-token bitmap, trailing-text rows and index, finished flag, frame count and cap, uniforms).  The attention
and cache-append kernels take the per-slot lengths (``base_rows``), so one decode frame covers all slots, and ``ops.slot_advance``
records each live slot's codes and moves it on.  That frame is captured ONCE per session as a CUDA graph and replayed by every step;
empty slots are kept finished, so they run masked and never advance.  Admission runs eagerly: the pending prompts, left-padded, are
prefilled straight into their free slots (``base_rows = -left_pad``, ``slot`` = slot ids), and their first frame's results are
scattered into slot state.  The host reads the finished flags and frame counts once per step to build events.
"""
from __future__ import annotations

import contextlib
import time
from dataclasses import dataclass
from typing import List

import torch

from .... import ops
from ...continuous import TTSBatchEvent, TTSBatchItem, TTSBatchOptions
from .qwen3_tts import _capture_frame, _FrameState


def _format_duration(seconds: float) -> str:
    """continuous_batching.py:15-19."""
    hours = int(seconds // 3600)
    minutes = int((seconds % 3600) // 60)
    secs = seconds % 60
    return f"{hours:02d}:{minutes:02d}:{secs:06.3f}"


def _round_up(n: int, m: int) -> int:
    return -(-n // m) * m


@dataclass
class _ActiveRequest:
    sequence_id: int
    slot: int


class Qwen3TTSBatchSession:
    """Step-wise non-streaming Qwen3 TTS batch session over ``options.max_batch_size`` KV-cache slots.

    Uniforms for the sampler are drawn on the device from the session's own generator; ``TTSBatchItem.extra["u"]`` ([frames, 16]
    floats in [0, 1)) pins a request's uniforms instead, frame by frame (parity tests), and ``extra["max_tokens"]`` lowers its frame cap
    below ``options.max_tokens``.  The session owns its caches, so the model's other generation calls may run between steps.
    ``use_graph=False`` runs every frame eagerly instead of replaying the captured graph."""

    def __init__(self, model, options: TTSBatchOptions, use_graph: bool = True):
        if model.speech_tokenizer is None:
            raise ValueError("Speech tokenizer not loaded")
        self.model = model
        self.options = options
        self.config = model.config.talker_config
        self.eos_token_id = self.config.codec_eos_token_id
        self.suppress_tokens = model._suppress_codec_tokens(self.eos_token_id)
        self._pending: List[TTSBatchItem] = []
        self._active: List[_ActiveRequest] = []
        self._start_time = time.time()
        self.captures = 0                                   # CUDA graph captures of the frame (one per session unless a cache grows)
        self._graph = None
        self._use_graph = use_graph
        self._sp = {"temperature": float(options.temperature), "top_k": int(options.top_k), "top_p": float(options.top_p),
                    "repetition_penalty": float(options.repetition_penalty), "eos": int(self.eos_token_id)}
        if options.max_tokens <= 0:
            return
        dev, n, cfg = model.device, int(options.max_batch_size), self.config
        self._dev, self._n, self._G, self._V = dev, n, cfg.num_code_groups, cfg.vocab_size
        self._H = cfg.hidden_size
        self._rng = torch.Generator(device=dev)
        self._rng.seed()
        _, _, pad = model._tts_embeds()
        self._pad = pad.reshape(-1).contiguous()
        self._suppress = torch.zeros(self._V, device=dev)
        self._suppress[torch.tensor(self.suppress_tokens, device=dev)] = float("-inf")
        self._rows, self._T = 0, 0
        self._kc = self._vc = None
        cps = model.talker.code_predictor.stack
        shape = (len(cps.layers), n, _round_up(self._G + 1, 256), cps.n_kv * cps.hd)
        self._cp_kc, self._cp_vc = torch.zeros(shape, device=dev), torch.zeros(shape, device=dev)
        self._st = _FrameState(n, self._G, self._pad_rows(n, 1), self._pad, self._suppress)
        self._st._base_rows = torch.zeros(n, dtype=torch.int32, device=dev)
        self._st._finished.fill_(1)                         # empty slots are kept finished
        self._frames = torch.zeros(n, dtype=torch.int32, device=dev)
        self._cap = torch.full((n,), int(options.max_tokens), dtype=torch.int32, device=dev)
        self._out = torch.zeros(n, int(options.max_tokens), self._G, dtype=torch.int64, device=dev)
        self._utab = torch.zeros(n, int(options.max_tokens), self._G, device=dev)

    # ------------------------------------------------------------------ protocol
    @property
    def idle(self) -> bool:
        return not self._pending and not self._active

    @property
    def available_slots(self) -> int:
        return max(0, self.options.max_batch_size - len(self._active))

    def add(self, items: list[TTSBatchItem]) -> None:
        self._pending.extend(items)

    def cancel(self, sequence_id: int) -> None:
        self._pending = [item for item in self._pending if item.sequence_id != sequence_id]
        for a in [a for a in self._active if a.sequence_id == sequence_id]:
            self._st._finished[a.slot] = 1                  # the slot runs masked from the next frame on
            self._active.remove(a)

    @torch.no_grad()
    def step(self) -> list[TTSBatchEvent]:
        events: list[TTSBatchEvent] = []
        if self._active:
            events.extend(self._advance_active())
        if self.available_slots > 0 and self._pending:
            events.extend(self._admit_pending())
        return events

    # ------------------------------------------------------------------ device state
    @contextlib.contextmanager
    def _use_caches(self):
        """Point the talker's and the code predictor's stacks at the session's caches (restored on exit)."""
        t, cp = self.model.talker.stack, self.model.talker.code_predictor.stack
        saved = (t.kc, t.vc, cp.kc, cp.vc)
        t.kc, t.vc, cp.kc, cp.vc = self._kc, self._vc, self._cp_kc, self._cp_vc
        try:
            yield
        finally:
            t.kc, t.vc, cp.kc, cp.vc = saved

    def _ensure_capacity(self, rows: int, text_rows: int) -> None:
        """Grow the KV cache to ``rows`` rows (rounded to 256) and the trailing-text table to ``text_rows`` rows, keeping every live
        slot's contents; the frame graph holds the old buffers' addresses, so it is captured again."""
        if rows > self._rows:
            new = _round_up(rows, 256)
            st = self.model.talker.stack
            shape = (len(st.layers), self._n, new, st.n_kv * st.hd)
            kc, vc = torch.zeros(shape, device=self._dev), torch.zeros(shape, device=self._dev)
            if self._kc is not None:
                kc[:, :, : self._rows].copy_(self._kc)
                vc[:, :, : self._rows].copy_(self._vc)
            self._kc = self._vc = None
            self._kc, self._vc, self._rows, self._graph = kc, vc, new, None
        if text_rows > self._T:
            new = _round_up(text_rows, 64)
            tab = self._pad_rows(self._n, new)
            tab[:, : self._st._trailing.shape[1]].copy_(self._st._trailing)
            self._st._trailing, self._T, self._graph = tab, new, None

    def _pad_rows(self, B: int, T: int) -> torch.Tensor:
        """A trailing-text table [B, T, H] filled with the pad embedding: rows past a request's text read pad."""
        return self._pad.reshape(1, 1, -1).expand(B, T, self._H).contiguous()

    def _frame(self) -> None:
        self.model._frame(self._st._x_in, self._sp, self._st)
        ops.slot_advance(self._st._base_rows, self._frames, self._st._finished, self._cap, self._st._codes, self._out, self._utab, self._st._u)

    # ------------------------------------------------------------------ steps
    def _advance_active(self) -> list[TTSBatchEvent]:
        with self._use_caches():
            if not self._use_graph:
                self._frame()
            else:
                if self._graph is None:
                    st = self._st
                    self._graph, self._frame_launches = _capture_frame(self._frame, [st._base_rows, self._frames, st._finished, st._seen,
                                                                                     st._codes, st._x_in, st._tidx, st._u, st._err])
                    self.captures += 1
                self._graph.replay()
                ops.LAUNCHES[0] += self._frame_launches
        state = torch.cat([self._st._finished.int(), self._frames, self._st._err]).cpu()      # the step's one host read
        if int(state[-1]) != 0:
            raise ValueError("Qwen3TTSBatchSession: a sampled code indexed outside its embedding table")
        events, still = [], []
        for a in self._active:
            if int(state[a.slot]):
                events.append(self._decode(a.sequence_id, int(state[self._n + a.slot]), a.slot))
            else:
                still.append(a)
        self._active = still
        return events

    def _prepare(self, item: TTSBatchItem):
        return self.model._prepare_generation_inputs(item.text, language=self.options.lang_code, speaker=item.voice, instruct=item.instruct)

    def _admit_pending(self) -> list[TTSBatchEvent]:
        k = min(self.available_slots, len(self._pending))
        pending, self._pending = self._pending[:k], self._pending[k:]
        if not pending:
            return []
        if self.options.max_tokens <= 0:
            return [self._empty_event(item.sequence_id) for item in pending]
        model, dev, G, H = self.model, self._dev, self._G, self._H
        used = {a.slot for a in self._active}
        slots = [s for s in range(self._n) if s not in used][:k]
        prep = [self._prepare(item) for item in pending]
        pmax = max(int(e.shape[1]) for e, _, _ in prep)
        self._ensure_capacity(pmax + int(self.options.max_tokens) + 1, max(int(tr.shape[1]) for _, tr, _ in prep) + 1)
        # left-padded prompts [k, pmax, H]; row b's prompt lands at cache rows [0, P_b) of its slot
        x = torch.zeros(k, pmax, H, device=dev)
        a = _FrameState(k, G, self._pad_rows(k, self._T), self._pad, self._suppress)
        left = []
        for b, (e, tr, _) in enumerate(prep):
            left.append(pmax - int(e.shape[1]))
            x[b, left[-1]:] = e[0].float()
            a._trailing[b, : tr.shape[1]] = tr[0].float()
        sl = torch.tensor(slots, dtype=torch.int64, device=dev)
        a._base_rows = torch.tensor([-v for v in left], dtype=torch.int32, device=dev)
        a._slot = sl.to(torch.int32)
        mt = int(self.options.max_tokens)
        for b, item in enumerate(pending):
            u = item.extra.get("u") if item.extra else None
            row = torch.rand(mt, G, device=dev, generator=self._rng)
            if u is not None:
                u = torch.as_tensor(u, dtype=torch.float32).reshape(-1, G)[:mt].to(dev)
                row[: u.shape[0]] = u
            self._utab[slots[b]] = row
            self._cap[slots[b]] = min(mt, int(item.extra.get("max_tokens", mt))) if item.extra else mt
        a._u.copy_(self._utab[sl, 0].T)
        with self._use_caches():
            model._frame(x, self._sp, a)
        # scatter the first frame into slot state
        st = self._st
        fin = a._finished.bool()
        st._seen[sl] = a._seen
        st._codes[sl] = a._codes
        st._x_in[sl] = a._x_in
        st._tidx[sl] = a._tidx
        st._trailing[sl] = a._trailing
        st._base_rows[sl] = torch.tensor([int(e.shape[1]) for e, _, _ in prep], dtype=torch.int32, device=dev)
        self._out[sl, 0] = a._codes
        self._frames[sl] = (~fin).int()
        st._finished[sl] = (fin | (self._frames[sl] >= self._cap[sl])).to(torch.uint8)
        st._u[:, sl] = self._utab[sl, min(1, mt - 1)].T
        state = torch.cat([st._finished[sl].int(), self._frames[sl], a._err]).cpu()          # the admission's one host read
        if int(state[-1]) != 0:
            raise ValueError("Qwen3TTSBatchSession: a sampled code indexed outside its embedding table")
        events = []
        for b, item in enumerate(pending):
            if int(state[b]):
                events.append(self._decode(item.sequence_id, int(state[k + b]), slots[b]))
            else:
                self._active.append(_ActiveRequest(item.sequence_id, slots[b]))
        return events

    # ------------------------------------------------------------------ events
    def _decode(self, sequence_id: int, n: int, slot: int) -> TTSBatchEvent:
        """_decode_state (continuous_batching.py:326-344)."""
        if n == 0:
            return self._empty_event(sequence_id)
        audio = self.model._decode_generated_codes(self._out[slot, :n])
        return TTSBatchEvent(sequence_id=sequence_id, audio=audio, sample_rate=self.model.sample_rate, samples=int(audio.shape[0]), token_count=n,
                             done=True, metadata={"audio_duration": _format_duration(audio.shape[0] / self.model.sample_rate),
                                                  "processing_time_seconds": time.time() - self._start_time,
                                                  "peak_memory_usage": torch.cuda.max_memory_allocated(self.model.device) / 1e9})

    def _empty_event(self, sequence_id: int) -> TTSBatchEvent:
        """continuous_batching.py:346-360."""
        return TTSBatchEvent(sequence_id=sequence_id, audio=torch.zeros(0, dtype=torch.float32, device=self.model.device),
                             sample_rate=self.model.sample_rate, samples=0, token_count=0, done=True,
                             metadata={"audio_duration": _format_duration(0.0), "processing_time_seconds": time.time() - self._start_time,
                                       "peak_memory_usage": torch.cuda.max_memory_allocated(self.model.device) / 1e9})
