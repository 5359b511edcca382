"""Qwen3-TTS talker and code predictor on H100 (reference: tts/models/qwen3_tts/talker.py).

``Qwen3TTSTalkerForConditionalGeneration(cfg).load_weights(...)``; ``talker(inputs_embeds) -> (logits, hidden)`` with the
KV cache held inside the object (the reference passes ``mlx_lm`` ``KVCache`` lists; ``make_cache`` / ``cache.offset``
survive as ``reset_cache`` / ``offset``).

H100 mapping: a decode step is a chain of bf16 GEMVs that stream every weight once (b2a_gemv_bf16, RMSNorm / SwiGLU /
residual fused), one warp-per-head kernel for q/k RMSNorm + (M)RoPE + cache append, and a cache attention kernel; the KV
length lives in device memory so the whole frame (talker step + 15 code-predictor sub-steps + 16 sampler launches) is ONE
CUDA graph (see qwen3_tts.py).  Prefill (S >= 17 rows) runs the same layers on the wgmma conv kernel.
"""
from __future__ import annotations

from typing import Optional

import torch

from .... import ops
from .config import Qwen3TTSTalkerCodePredictorConfig, Qwen3TTSTalkerConfig

GEMV_MAX_ROWS = 16
PREFILL_TC_MIN_ROWS = 64          # prefills of at least this many rows run attention on b2a_attn_prefill (one full query tile)


def _interleave(gate: torch.Tensor, up: torch.Tensor) -> torch.Tensor:
    """(gate_0, up_0, gate_1, up_1, ...) row order: a GEMV CTA owns whole (gate, up) pairs and applies SwiGLU in its epilogue."""
    return torch.stack([gate, up], dim=1).reshape(-1, gate.shape[1])


class _DecoderStack:
    """N x (RMSNorm, attention with per-head q/k RMSNorm + rotary + KV cache, RMSNorm, SwiGLU MLP) + final RMSNorm
    (TalkerDecoderLayer talker.py:367-400 / CodePredictorDecoderLayer :603-632)."""

    def __init__(self, P, pre, n_layers, hidden, n_heads, n_kv, head_dim, eps, theta, mrope, device):
        f = lambda t: t.float().to(device).contiguous()
        self.n_heads, self.n_kv, self.hd, self.eps, self.theta, self.mrope = n_heads, n_kv, head_dim, eps, theta, mrope
        self.hidden, self.device = hidden, device
        self.layers = []
        for i in range(n_layers):
            L = f"{pre}.layers.{i}"
            A = L + ".self_attn"
            qkv = torch.cat([P[A + f".{n}_proj.weight"].float() for n in "qkv"], dim=0)
            gu = _interleave(P[L + ".mlp.gate_proj.weight"].float(), P[L + ".mlp.up_proj.weight"].float())
            self.layers.append({
                "n1": f(P[L + ".input_layernorm.weight"]), "n2": f(P[L + ".post_attention_layernorm.weight"]),
                "qkv": ops.pack_linear(qkv, None, device), "o": ops.pack_linear(P[A + ".o_proj.weight"].float(), None, device),
                "qn": f(P[A + ".q_norm.weight"]), "kn": f(P[A + ".k_norm.weight"]),
                "gu": ops.pack_linear(gu, None, device), "down": ops.pack_linear(P[L + ".mlp.down_proj.weight"].float(), None, device)})
        self.norm = f(P[pre + ".norm.weight"])
        self.kc = self.vc = None

    def alloc_cache(self, batch: int, max_len: int):
        """Pre-sized device cache [layer, B, rows, n_kv*hd].  The row capacity is rounded up to 256 and a buffer that is already
        large enough for this batch is reused: rows past the device-side length are never read (attn_decode stops at base + s),
        so a prompt of another length costs neither a ~1 GB reallocation nor a zero-fill."""
        rows = -(-max_len // 256) * 256
        if self.kc is None or self.kc.shape[1] != batch or self.kc.shape[2] < rows:
            shape = (len(self.layers), batch, rows, self.n_kv * self.hd)
            self.kc = self.vc = None                       # release before allocating the replacement
            self.kc = torch.zeros(shape, device=self.device, dtype=torch.float32)
            self.vc = torch.zeros(shape, device=self.device, dtype=torch.float32)

    def _proj(self, x2, cw, norm_w=None, swiglu=False, res=None, nxt=None):
        # nxt: the next projection, whose weights the GEMV pulls into L2 while it streams its own
        if x2.shape[0] <= GEMV_MAX_ROWS and ops.gemv_eligible(cw):
            return ops.gemv(x2, cw, norm_w=norm_w, norm_eps=self.eps, swiglu=swiglu, res=res, prefetch=nxt)
        h = ops.layernorm(x2, norm_w, None, eps=self.eps, rms=True) if norm_w is not None else x2
        y = ops.linear(h, cw, res=None if swiglu else res)
        return ops.swiglu(y, interleaved=True) if swiglu else y

    def forward(self, x: torch.Tensor, *, base_dev=None, base: int = 0, pos3=None, kv_start=None, final_norm: bool = True,
                tail=None, pos_shift=None, base_rows=None, slot=None) -> torch.Tensor:
        """x [B,S,H] -> final-normed hidden [B,S,H] (``final_norm=False``: the residual stream, for a consumer that fuses the
        norm); appends S rows to the cache at ``base`` (device scalar or host int).  ``tail``: the projection that follows the
        stack (head), prefetched into L2 by the last layer.  ``base_rows`` / ``slot`` int32 [B]: per-row cache positions and cache
        batch indices (continuous batching; see ops.qknorm_rope_cache)."""
        B, S, H = x.shape
        x2 = x.reshape(B * S, H)
        hq, hk, hd = self.n_heads, self.n_kv, self.hd
        max_k = self.kc.shape[2] if base_dev is not None or base_rows is not None else base + S
        rows = dict(base_rows=base_rows, slot=slot) if base_rows is not None or slot is not None else {}
        # long prefills (the in-context cloning prompt) on the tensor-core kernel; decode frames, the code predictor and short prompts
        # stay on attn_decode
        prefill_tc = S >= PREFILL_TC_MIN_ROWS and hd == 128 and hq == 2 * hk
        for li, lw in enumerate(self.layers):
            nxt_qkv = self.layers[li + 1]["qkv"] if li + 1 < len(self.layers) else tail
            qkv = self._proj(x2, lw["qkv"], norm_w=lw["n1"], nxt=lw["o"])
            q = ops.qknorm_rope_cache(qkv.view(B, S, -1), hq, hk, hd, self.kc[li], self.vc[li], q_norm=lw["qn"], k_norm=lw["kn"],
                                      eps=self.eps, pos3=pos3, base_dev=base_dev, base=base, mrope=self.mrope, theta=self.theta,
                                      pos_shift=pos_shift, **rows)
            attn = ops.attn_prefill if prefill_tc else ops.attn_decode
            a = attn(q, self.kc[li], self.vc[li], hq, hk, hd, scale=hd ** -0.5, base_dev=base_dev, base=base, kv_start=kv_start,
                     max_k=max_k, **rows)
            x2 = self._proj(a.view(B * S, hq * hd), lw["o"], res=x2, nxt=lw["gu"])
            m = self._proj(x2, lw["gu"], norm_w=lw["n2"], swiglu=True, nxt=lw["down"])
            x2 = self._proj(m, lw["down"], res=x2, nxt=nxt_qkv)
        if not final_norm:
            return x2.view(B, S, H)
        return ops.layernorm(x2, self.norm, None, eps=self.eps, rms=True).view(B, S, H)


class Qwen3TTSTalkerCodePredictor:
    """talker.py:706-764: 5-layer GQA transformer with standard RoPE, one lm_head and one embedding table per code group."""

    def __init__(self, P, config: Qwen3TTSTalkerCodePredictorConfig, talker_hidden_size: int, device):
        self.config = config
        self.num_code_groups = config.num_code_groups
        f = lambda t: t.float().to(device).contiguous()
        pre = "code_predictor"
        self.proj = None
        if pre + ".small_to_mtp_projection.weight" in P:
            self.proj = ops.pack_linear(P[pre + ".small_to_mtp_projection.weight"].float(), P[pre + ".small_to_mtp_projection.bias"].float(), device)
        self.stack = _DecoderStack(P, pre + ".model", config.num_hidden_layers, config.hidden_size, config.num_attention_heads,
                                   config.num_key_value_heads, config.head_dim, config.rms_norm_eps, config.rope_theta, (0, 0), device)
        self.codec_embedding = [f(P[f"{pre}.model.codec_embedding.{g}.weight"]) for g in range(config.num_code_groups - 1)]
        self.lm_head = [ops.pack_linear(P[f"{pre}.lm_head.{g}.weight"].float(), None, device) for g in range(config.num_code_groups - 1)]

    def reset_cache(self, batch: int):
        self.stack.alloc_cache(batch, self.num_code_groups + 1)

    def __call__(self, inputs_embeds: torch.Tensor, offset: int, generation_step: int) -> torch.Tensor:
        """inputs_embeds [B,S,H] at cache offset ``offset`` -> logits [B,S,vocab] of head ``generation_step``."""
        B, S, _ = inputs_embeds.shape
        if self.proj is not None:
            inputs_embeds = ops.linear(inputs_embeds, self.proj)
        head = self.lm_head[generation_step]
        h = self.stack.forward(inputs_embeds, base=offset, final_norm=False, tail=head)          # final RMSNorm fused into the head GEMV
        return self.stack._proj(h.reshape(B * S, -1), head, norm_w=self.stack.norm, nxt=self.stack.layers[0]["qkv"]).view(B, S, -1)


class Qwen3TTSTalkerForConditionalGeneration:
    """talker.py:767-840 (+ Qwen3TTSTalkerModel :403-500)."""

    def __init__(self, config: Qwen3TTSTalkerConfig, device="cuda"):
        self.config = config
        self.device = torch.device(device)
        self.stack: Optional[_DecoderStack] = None
        self.offset_dev = torch.zeros(1, dtype=torch.int32, device=self.device)     # KVCache.offset, device-resident
        self.offset = 0                                                              # host mirror (valid outside graph replays)

    def load_weights(self, weights):
        """``weights``: names after ``sanitize`` (``talker.`` prefix stripped), linear weights [out, in]."""
        P, cfg, dev = dict(weights), self.config, self.device
        f = lambda t: t.float().to(dev).contiguous()
        sec = (cfg.rope_scaling or {}).get("mrope_section", [24, 20, 20])
        self.stack = _DecoderStack(P, "model", cfg.num_hidden_layers, cfg.hidden_size, cfg.num_attention_heads, cfg.num_key_value_heads,
                                   cfg.head_dim, cfg.rms_norm_eps, cfg.rope_theta, (sec[1], sec[2]), dev)
        self.codec_embedding = f(P["model.codec_embedding.weight"])
        self.text_embedding = f(P["model.text_embedding.weight"]) if "model.text_embedding.weight" in P else None
        if "text_projection.linear_fc1.weight" in P:
            self.text_fc1 = ops.pack_linear(P["text_projection.linear_fc1.weight"].float(), P["text_projection.linear_fc1.bias"].float(), dev)
            self.text_fc2 = ops.pack_linear(P["text_projection.linear_fc2.weight"].float(), P["text_projection.linear_fc2.bias"].float(), dev)
        self.codec_head = ops.pack_linear(P["codec_head.weight"].float(), None, dev)
        self.code_predictor = Qwen3TTSTalkerCodePredictor(P, cfg.code_predictor_config, cfg.hidden_size, dev)
        return self

    @staticmethod
    def sanitize(weights):
        """talker.py:825-839: keep ``talker.*`` and strip the prefix."""
        return {k[len("talker."):]: v for k, v in weights.items() if k.startswith("talker.")}

    def get_input_embeddings(self):
        return self.codec_embedding

    def get_text_embeddings(self):
        return self.text_embedding

    def text_projection(self, x: torch.Tensor) -> torch.Tensor:
        """ResizeMLP (talker.py:339-364): fc2(silu(fc1(x)))."""
        return ops.linear(ops.linear(x, self.text_fc1, post_act=ops.ACT["silu"]), self.text_fc2)

    def reset_cache(self, batch: int, max_len: int):
        """make_cache (talker.py:498-500,820-822): pre-sized K/V (the reference grows them in 256-row blocks, cache.py:104-155)."""
        self.stack.alloc_cache(batch, max_len)
        self.code_predictor.reset_cache(batch)
        self.offset_dev.zero_()
        self.offset = 0

    def __call__(self, inputs_embeds: torch.Tensor, position_ids=None, kv_start=None, use_device_offset: bool = False, base_rows=None,
                 slot=None):
        """inputs_embeds [B,S,H] -> (logits [B,S,V], hidden [B,S,H]); appends to the cache (talker.py:799-818).  ``kv_start`` int32 [B]
        = left-padding count per row: the ``attention_mask`` path of talker.py:449-476 (keys before it are masked, rotary positions are
        cumsum(mask) - 1 = cache row - kv_start, clamped at 0).  ``base_rows`` int32 [B] (with an optional ``slot`` map) = per-row cache
        lengths of a continuous batch: row b appends at cache row base_rows[b] of cache batch slot[b] and sees the rows before it; a
        negative base left-pads the row.  The caller owns those lengths: ``offset`` is not touched."""
        B, S, _ = inputs_embeds.shape
        if base_rows is not None:
            h = self.stack.forward(inputs_embeds, base_rows=base_rows, slot=slot, tail=self.codec_head)
            logits = self.stack._proj(h.reshape(B * S, -1), self.codec_head, nxt=self.code_predictor.stack.layers[0]["qkv"]).view(B, S, -1)
            return logits, h
        pos3 = None
        if position_ids is not None:
            pos3 = position_ids.to(device=self.device, dtype=torch.int32)
            if pos3.dim() == 2:
                pos3 = pos3[None].expand(3, -1, -1)
            pos3 = pos3.contiguous()
        if use_device_offset:
            h = self.stack.forward(inputs_embeds, base_dev=self.offset_dev, pos3=pos3, kv_start=kv_start, tail=self.codec_head,
                                   pos_shift=kv_start if pos3 is None else None)
            ops.incr_(self.offset_dev, S)
        else:
            h = self.stack.forward(inputs_embeds, base=self.offset, pos3=pos3, kv_start=kv_start, tail=self.codec_head,
                                   pos_shift=kv_start if pos3 is None else None)
            ops.incr_(self.offset_dev, S)
        self.offset += S
        logits = self.stack._proj(h.reshape(B * S, -1), self.codec_head, nxt=self.code_predictor.stack.layers[0]["qkv"]).view(B, S, -1)
        return logits, h
