"""Oracle for the Qwen3-TTS continuous-batching session (reference: tts/models/qwen3_tts/continuous_batching.py), restated over the
single-sequence loop.

In the reference session every request generates exactly what it would generate alone from its own uniforms (its KV rows, seen tokens
and trailing-text index are its own; the batch only shares launches), so a request's codes are ``qwen3.generate_codes`` of its prompt.
What the session adds is WHEN each request finishes and in which order the events come:

- ``step()`` first advances the active requests by one frame (events in admission order), then admits up to ``max_batch_size -
  len(active)`` pending requests, whose prefill runs their frame 0 (events in pending order);
- a request with n recorded codes finishes on the frame that samples EOS (frame n) when n < max_tokens, else on frame max_tokens - 1;
- ``cancel`` drops a pending or active request without an event; ``max_tokens <= 0`` turns every admission into an empty event.
"""
from __future__ import annotations


def finish_frame(n_codes: int, max_tokens: int) -> int:
    """The frame (0 = the admission's) on which a request with ``n_codes`` recorded codes leaves the batch."""
    return n_codes if n_codes < max_tokens else n_codes - 1


def run_schedule(codes: dict, script: dict, max_batch_size: int, max_tokens: int, max_steps: int = 10_000):
    """``codes[seq_id]`` = the request's codes [n, G] (``qwen3.generate_codes`` with its uniforms and ``max_tokens``);
    ``script[step]`` = list of ("add", [seq_ids]) / ("cancel", seq_id) actions applied before that step.  Returns the events
    [(step, seq_id, token_count)] in the order the session emits them, and {seq_id: step it was cancelled while active}."""
    pending, active, events, cancelled = [], [], [], {}
    for step in range(max_steps):
        for kind, arg in script.get(step, []):
            if kind == "add":
                pending.extend(arg)
            else:
                pending = [s for s in pending if s != arg]
                if any(s == arg for s, _ in active):
                    cancelled[arg] = step
                active = [(s, t) for s, t in active if s != arg]
        if not pending and not active and step > max(script, default=0):
            break
        still = []
        for s, t0 in active:                                      # frame step - t0 of request s
            if max_tokens > 0 and step - t0 == finish_frame(codes[s].shape[0], max_tokens):
                events.append((step, s, codes[s].shape[0]))
            else:
                still.append((s, t0))
        active = still
        k = min(max_batch_size - len(active), len(pending))
        admitted, pending = pending[:k], pending[k:]
        for s in admitted:
            if max_tokens <= 0:
                events.append((step, s, 0))
            elif finish_frame(codes[s].shape[0], max_tokens) == 0:
                events.append((step, s, codes[s].shape[0]))
            else:
                active.append((s, step))
    return events, cancelled
