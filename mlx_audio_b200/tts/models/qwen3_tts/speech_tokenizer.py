"""Qwen3-TTS 12.5 Hz speech tokenizer on H100 (reference: tts/models/qwen3_tts/speech_tokenizer.py).

``Qwen3TTSSpeechTokenizer(cfg).load_weights(...)``; ``decode(audio_codes[B,T,16]) -> (wav[B,samples], lengths)``
(speech_tokenizer.py:1099-1118), ``batch_decode`` (:1120-1179), ``streaming_decode`` (:1181-1217) and the decoder's
``__call__`` / ``chunked_decode`` (:843-880, 932-954) and the incremental ``streaming_step`` / ``reset_streaming_state`` (:882-930).  ``encode(audio[B,1,n]) -> codes[B,16,ceil(n/1920)]``
(:1082-1093) through ``Qwen3TTSSpeechTokenizerEncoder`` (:957-1058) when the checkpoint has encoder weights: Mimi's encode chain
(codec/models/mimi.py), with a full causal mask and half-split RoPE in its transformer.

H100 mapping: RVQ gather-sum in one kernel; every dense conv / linear runs on the wgmma conv kernel with the SnakeBeta /
LayerScale / gamma / residual / clip fused as prologue or epilogue; the 300-frame chunks of ``chunked_decode`` are
independent, so equal-length chunks are decoded as one batch instead of one after another.
"""
from __future__ import annotations

from typing import Dict, List

import numpy as np
import torch

from .... import ops
from ....codec.models import mimi
from ....ops import ACT, Pre
from .config import Qwen3TTSTokenizerConfig, Qwen3TTSTokenizerDecoderConfig, Qwen3TTSTokenizerEncoderConfig


def check_array_shape_qwen3(arr) -> bool:
    """True when a 3-D conv weight already is MLX-layout (out, K, in) (qwen3_tts.py:123-157)."""
    shape = tuple(arr.shape)
    if len(shape) != 3:
        return False
    _, dim2, dim3 = shape
    if dim2 == 1:
        return dim3 > 64
    if dim3 == 1:
        return not dim2 > 64
    return dim2 < dim3


class Qwen3TTSSpeechTokenizerDecoder:
    def __init__(self, config: Qwen3TTSTokenizerDecoderConfig, device="cuda"):
        self.config = config
        self.device = torch.device(device)
        self.total_upsample = int(np.prod(list(config.upsample_rates) + list(config.upsampling_ratios)))
        self._w = None
        self._st = None                 # streaming state (streaming_step); None = no stream in progress

    # ------------------------------------------------------------------ weights
    def load_weights(self, weights, prefix="decoder."):
        """``weights``: MLX-side names (after ``Qwen3TTSSpeechTokenizer.sanitize``), conv weights [Cout, K, Cin/g]."""
        P, cfg, dev = {k[len(prefix):]: v for k, v in dict(weights).items() if k.startswith(prefix)}, self.config, self.device
        f = lambda t: t.float().to(dev).contiguous()
        conv = lambda pre, groups=1: ops.pack_conv(P[pre + ".weight"].float(), P.get(pre + ".bias"), groups, dev)
        lin = lambda pre: ops.pack_linear(P[pre + ".weight"].float(), P.get(pre + ".bias"), dev)

        def snake(pre):                                                 # SnakeBeta constants (speech_tokenizer.py:123-126)
            a, b = torch.exp(P[pre + ".alpha"].float()), torch.exp(P[pre + ".beta"].float())
            return Pre(act=ACT["snake"], a=f(a), b=f(1.0 / (b + 1e-9)))

        W = {}
        nsem, nq = cfg.num_semantic_quantizers, cfg.num_quantizers
        W["cb_first"] = f(torch.stack([P[f"quantizer.rvq_first.vq.layers.{i}.codebook.embed.weight"].float() for i in range(nsem)]))
        W["cb_rest"] = f(torch.stack([P[f"quantizer.rvq_rest.vq.layers.{i}.codebook.embed.weight"].float() for i in range(nq - nsem)]))
        W["proj_first"] = conv("quantizer.rvq_first.output_proj")
        W["proj_rest"] = conv("quantizer.rvq_rest.output_proj")
        W["pre_conv"] = conv("pre_conv.conv")
        T = "pre_transformer"
        W["in_proj"], W["out_proj"], W["norm"] = lin(T + ".input_proj"), lin(T + ".output_proj"), f(P[T + ".norm.weight"])
        W["layers"] = []
        for i in range(cfg.num_hidden_layers):
            L = f"{T}.layers.{i}"
            qkv = torch.cat([P[L + f".self_attn.{n}_proj.weight"].float() for n in "qkv"], dim=0)
            gu = torch.cat([P[L + ".mlp.gate_proj.weight"].float(), P[L + ".mlp.up_proj.weight"].float()], dim=0)
            W["layers"].append({
                "n1": f(P[L + ".input_layernorm.weight"]), "n2": f(P[L + ".post_attention_layernorm.weight"]),
                "qkv": ops.pack_linear(qkv, None, dev), "o": lin(L + ".self_attn.o_proj"),
                "gu": ops.pack_linear(gu, None, dev), "down": lin(L + ".mlp.down_proj"),
                "ls1": f(P[L + ".self_attn_layer_scale.scale"]), "ls2": f(P[L + ".mlp_layer_scale.scale"])})
        W["upsample"] = []
        for i, _ in enumerate(cfg.upsampling_ratios):
            U = f"upsample.{i}"
            W["upsample"].append({"up": conv(U + ".0.conv"), "dw": conv(U + ".1.dwconv.conv", cfg.latent_dim),
                                  "ln": (f(P[U + ".1.norm.weight"]), f(P[U + ".1.norm.bias"])),
                                  "pw1": lin(U + ".1.pwconv1"), "pw2": lin(U + ".1.pwconv2"), "gamma": f(P[U + ".1.gamma"])})
        W["init"] = conv("decoder.0.conv")
        W["blocks"] = []
        for bi, r in enumerate(cfg.upsample_rates):
            B_ = f"decoder.{bi + 1}.block"
            units = []
            for ui, d in enumerate((1, 3, 9)):
                U = f"{B_}.{ui + 2}"
                units.append({"d": d, "s1": snake(U + ".act1"), "c1": conv(U + ".conv1.conv"), "s2": snake(U + ".act2"), "c2": conv(U + ".conv2.conv")})
            W["blocks"].append({"r": r, "snake": snake(B_ + ".0"), "up": conv(B_ + ".1.conv"), "units": units})
        W["out_snake"] = snake(f"decoder.{len(cfg.upsample_rates) + 1}")
        W["out_conv"] = conv(f"decoder.{len(cfg.upsample_rates) + 2}.conv")
        self._w = W
        return self

    # ------------------------------------------------------------------ forward
    @torch.no_grad()
    def __call__(self, codes: torch.Tensor, taps=None) -> torch.Tensor:
        """codes int [B, num_quantizers, T] -> audio [B, 1, 1920 T] clipped to [-1, 1] (speech_tokenizer.py:843-880)."""
        W, cfg, dev = self._w, self.config, self.device
        if codes.shape[1] != cfg.num_quantizers:
            raise ValueError(f"Expected {cfg.num_quantizers} layers of codes, got {codes.shape[1]}")
        codes = codes.to(device=dev, dtype=torch.int64).contiguous()
        B, nq, T = codes.shape
        nsem = cfg.num_semantic_quantizers
        x = ops.conv1d(ops.rvq_decode(codes[:, :nsem], W["cb_first"]), W["proj_first"])
        if nq > nsem:
            x = ops.conv1d(ops.rvq_decode(codes[:, nsem:], W["cb_rest"]), W["proj_rest"], res=x)
        h = ops.conv1d(x, W["pre_conv"], pad_left=2, lout=T)                                   # CausalConv1d k3
        if taps is not None:
            taps["pre_conv"] = h
        # ---- pre_transformer (speech_tokenizer.py:383-413): RMSNorm, RoPE (rotate_half), full causal, SwiGLU, LayerScale
        nh, hd, eps = cfg.num_attention_heads, cfg.head_dim, cfg.rms_norm_eps
        d = nh * hd
        x = ops.linear(h, W["in_proj"])
        for lw in W["layers"]:
            n = ops.layernorm(x, lw["n1"], None, eps=eps, rms=True)
            qkv = ops.linear(n, lw["qkv"])
            ops.rope_(qkv[:, :, :d], nh, offset=0, base=cfg.rope_theta, traditional=False)
            ops.rope_(qkv[:, :, d:2 * d], nh, offset=0, base=cfg.rope_theta, traditional=False)
            att = ops.attention(qkv[:, :, :d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:], n_heads=nh, scale=hd ** -0.5, causal=True)
            x = ops.linear(att, lw["o"], cscale=lw["ls1"], res=x)
            n = ops.layernorm(x, lw["n2"], None, eps=eps, rms=True)
            m = ops.swiglu(ops.linear(n, lw["gu"]))
            x = ops.linear(m, lw["down"], cscale=lw["ls2"], res=x)
        h = ops.linear(ops.layernorm(x, W["norm"], None, eps=eps, rms=True), W["out_proj"])
        if taps is not None:
            taps["transformer"] = h
        # ---- 2 x (CausalTransposeConv1d k=s=2, ConvNeXtBlock) (speech_tokenizer.py:86-159)
        for (uw, fct) in zip(W["upsample"], cfg.upsampling_ratios):
            h = ops.conv1d(h, uw["up"], stride=fct, pad_left=0, lout=h.shape[1] * fct, transpose=True)
            t = ops.conv1d(h, uw["dw"], pad_left=6, lout=h.shape[1])
            t = ops.layernorm(t, *uw["ln"], eps=1e-6)
            t = ops.linear(t, uw["pw1"], post_act=ACT["gelu"])
            h = ops.linear(t, uw["pw2"], cscale=uw["gamma"], res=h)
        if taps is not None:
            taps["upsample"] = h
        # ---- decoder: conv k7, 4 x (SnakeBeta, ConvT, 3 residual units), SnakeBeta, conv k7 -> 1, clip
        w = ops.conv1d(h, W["init"], pad_left=6, lout=h.shape[1])
        for bi, bw in enumerate(W["blocks"]):
            r = bw["r"]
            w = ops.conv1d(w, bw["up"], stride=r, pad_left=0, lout=w.shape[1] * r, pre=bw["snake"], transpose=True)
            for u in bw["units"]:
                t = ops.conv1d(w, u["c1"], dilation=u["d"], pad_left=6 * u["d"], lout=w.shape[1], pre=u["s1"])
                w = ops.conv1d(t, u["c2"], pre=u["s2"], res=w)
            if taps is not None:
                taps[f"block{bi}"] = w
        wav = ops.conv1d(w, W["out_conv"], pad_left=6, lout=w.shape[1], pre=W["out_snake"], post_act=ACT["clip1"])   # [B, L, 1]
        return wav.reshape(B, 1, -1)

    @torch.no_grad()
    def chunked_decode(self, codes: torch.Tensor, chunk_size: int = 300, left_context_size: int = 25) -> torch.Tensor:
        """speech_tokenizer.py:932-954, with chunks of equal length decoded as one batch (they do not interact)."""
        codes = codes.to(device=self.device, dtype=torch.int64)
        B, nq, T = codes.shape
        up = self.total_upsample
        spans, start = [], 0
        while start < T:
            end = min(start + chunk_size, T)
            ctx = left_context_size if start - left_context_size > 0 else start
            spans.append((start, end, ctx))
            start = end
        out = torch.empty(B, 1, T * up, device=self.device, dtype=torch.float32)
        groups: Dict[tuple, List[tuple]] = {}
        for sp in spans:
            groups.setdefault((sp[1] - sp[0] + sp[2], sp[2]), []).append(sp)
        for (length, ctx), members in groups.items():
            batch = torch.cat([codes[:, :, s - c: e] for (s, e, c) in members], dim=0)          # [n*B, nq, length]
            wav = self(batch)
            for i, (s, e, c) in enumerate(members):
                out[:, :, s * up: e * up] = wav[i * B: (i + 1) * B, :, c * up:]
        return out

    # ------------------------------------------------------------------ incremental (streaming) decode
    # speech_tokenizer.py:882-930.  Every stateful layer reads one [B, H + rows, C] buffer: H history rows, then the rows of this call,
    # which their producer writes in place (out= views), so the conv runs with pad_left = 0 over the whole buffer.  History rows hold
    # pre-activation values (Snake stays in the conv prologue; it is elementwise, so this equals the reference's post-activation
    # buffers).  Each buffer exists twice (ping-pong): the carry of the last H rows into the other copy's head is one launch for all
    # layers, and stays race-free when the history is longer than a call's rows.  A decoder block's transposed conv writes its r-row
    # overflow (bias included) past the rows of this call; the next call adds it, from the other copy, into its head rows -- the
    # reference's overlap-add (DecoderBlockUpsample.step, :645-656), which counts the bias twice there.  The KV cache of the transformer
    # is each layer's qkv buffer: the projection writes rows [offset, offset + L), RoPE and causal attention continue from offset.
    kv_step = 256          # KV-cache capacity grows in steps of this many frames (the reference's KVCache step)

    def reset_streaming_state(self):
        """Start a new stream: the next ``streaming_step`` begins with empty conv history, KV cache and overlap buffers."""
        self._st = None

    def _stream_layers(self):
        """(history rows, channels, rows per frame, overflow rows) of every buffered layer input, in the carry's order."""
        W, cfg = self._w, self.config
        layers = [(W["pre_conv"].K - 1, W["pre_conv"].cin, 1, 0)]
        rpf = 1
        for uw, f in zip(W["upsample"], cfg.upsampling_ratios):
            if uw["up"].K != f:
                raise NotImplementedError("streaming_step: an upsampling transposed conv with kernel != stride has no overlap buffer")
            rpf *= f
            layers.append((uw["dw"].K - 1, uw["dw"].cin, rpf, 0))
        layers.append((W["init"].K - 1, W["init"].cin, rpf, 0))
        for bw in W["blocks"]:
            r = bw["r"]
            if bw["up"].K != 2 * r:
                raise NotImplementedError("streaming_step: decoder-block transposed convs must have kernel 2 * stride")
            rpf *= r
            for ui, u in enumerate(bw["units"]):
                layers.append(((u["c1"].K - 1) * u["d"], u["c1"].cin, rpf, r if ui == 0 else 0))
        layers.append((W["out_conv"].K - 1, W["out_conv"].cin, rpf, 0))
        return layers

    def _stream_buffers(self, B, cap):
        layers = self._stream_layers()
        return [[torch.zeros(B, H + cap * rpf + extra, C, device=self.device) for _ in range(2)] for (H, C, rpf, extra) in layers]

    def _stream_grow(self, S, B, L):
        """Make room for L new frames: conv buffers for chunks of L frames, KV capacity for offset + L (steps of ``kv_step``).  History,
        overflow and cached K/V move to the new buffers in one launch each."""
        layers = self._stream_layers()
        if L > S["cap"]:
            new = self._stream_buffers(B, L)
            if S["off"] > 0:
                p, q, moves = S["p"], 1 - S["p"], []
                for (H, C, rpf, extra), old, nb in zip(layers, S["bufs"], new):
                    moves.append((old[p][:, :H], nb[p][:, :H], False))
                    if extra:
                        t0 = H + S["prev"] * rpf
                        moves.append((old[q][:, t0:t0 + extra], nb[q][:, t0:t0 + extra], False))
                ops.stream_rows(moves)
            S["bufs"], S["cap"] = new, L
        need = S["off"] + L
        if need > S["kv_cap"]:
            cap = -(-need // self.kv_step) * self.kv_step
            d3 = 3 * self.config.num_attention_heads * self.config.head_dim
            new = [torch.empty(B, cap, d3, device=self.device) for _ in self._w["layers"]]
            ops.stream_rows([(old[:, :S["off"]], nb[:, :S["off"]], False) for old, nb in zip(S["kv"], new)])
            S["kv"], S["kv_cap"] = new, cap

    @torch.no_grad()
    def streaming_step(self, codes: torch.Tensor) -> torch.Tensor:
        """codes int [B, num_quantizers, n_new] (only the new frames) -> audio [B, 1, 1920 n_new] clipped to [-1, 1], continuing the
        stream begun by the last ``reset_streaming_state()`` (speech_tokenizer.py:889-930)."""
        W, cfg, dev = self._w, self.config, self.device
        if codes.shape[1] != cfg.num_quantizers:
            raise ValueError(f"Expected {cfg.num_quantizers} layers of codes, got {codes.shape[1]}")
        codes = codes.to(device=dev, dtype=torch.int64).contiguous()
        B, nq, L = codes.shape
        S = getattr(self, "_st", None)
        if S is not None and S["B"] != B:
            raise ValueError(f"streaming_step: batch size changed from {S['B']} to {B} within a stream (call reset_streaming_state first)")
        if L == 0:
            return torch.empty(B, 1, 0, device=dev)
        if S is None:
            S = self._st = {"B": B, "off": 0, "p": 0, "prev": 0, "cap": 0, "kv_cap": 0, "kv": [],
                            "err": torch.zeros(1, dtype=torch.int32, device=dev)}
        self._stream_grow(S, B, L)
        layers = self._stream_layers()
        p, off = S["p"], S["off"]
        X = [b[p] for b in S["bufs"]]
        prev = [b[1 - p] for b in S["bufs"]]
        nsem = cfg.num_semantic_quantizers
        H0 = layers[0][0]
        pc_in = X[0][:, H0:H0 + L]
        x = ops.conv1d(ops.rvq_decode(codes[:, :nsem], W["cb_first"], err=S["err"]), W["proj_first"], out=None if nq > nsem else pc_in)
        if nq > nsem:
            ops.conv1d(ops.rvq_decode(codes[:, nsem:], W["cb_rest"], err=S["err"]), W["proj_rest"], res=x, out=pc_in)
        h = ops.conv1d(X[0][:, :H0 + L], W["pre_conv"], lout=L)
        # ---- transformer with the KV cache (rows [0, off) of every layer's qkv buffer)
        nh, hd, eps = cfg.num_attention_heads, cfg.head_dim, cfg.rms_norm_eps
        d = nh * hd
        x = ops.linear(h, W["in_proj"])
        for lw, kv in zip(W["layers"], S["kv"]):
            n = ops.layernorm(x, lw["n1"], None, eps=eps, rms=True)
            new = kv[:, off:off + L]
            ops.linear(n, lw["qkv"], out=new)
            ops.rope_(new[:, :, :d], nh, offset=off, base=cfg.rope_theta, traditional=False)
            ops.rope_(new[:, :, d:2 * d], nh, offset=off, base=cfg.rope_theta, traditional=False)
            att = ops.attention(new[:, :, :d], kv[:, :off + L, d:2 * d], kv[:, :off + L, 2 * d:], n_heads=nh, scale=hd ** -0.5,
                                causal=True, q_offset=off)
            x = ops.linear(att, lw["o"], cscale=lw["ls1"], res=x)
            n = ops.layernorm(x, lw["n2"], None, eps=eps, rms=True)
            m = ops.swiglu(ops.linear(n, lw["gu"]))
            x = ops.linear(m, lw["down"], cscale=lw["ls2"], res=x)
        h = ops.linear(ops.layernorm(x, W["norm"], None, eps=eps, rms=True), W["out_proj"])
        # ---- upsampling: transposed conv (k = s, no overlap) into the ConvNeXt buffer; pwconv2 writes the next buffered input
        li = 1
        for i, (uw, f) in enumerate(zip(W["upsample"], cfg.upsampling_ratios)):
            Hh, rows = layers[li][0], h.shape[1] * f
            cur = X[li][:, Hh:Hh + rows]
            ops.conv1d(h, uw["up"], stride=f, pad_left=0, lout=rows, transpose=True, out=cur)
            t = ops.conv1d(X[li][:, :Hh + rows], uw["dw"], lout=rows)
            t = ops.layernorm(t, *uw["ln"], eps=1e-6)
            t = ops.linear(t, uw["pw1"], post_act=ACT["gelu"])
            nxt = X[li + 1][:, layers[li + 1][0]:layers[li + 1][0] + rows]
            h = ops.linear(t, uw["pw2"], cscale=uw["gamma"], res=cur, out=nxt if i == len(W["upsample"]) - 1 else None)
            li += 1
        # ---- decoder: conv k7, 4 x (SnakeBeta, ConvT + overlap-add, 3 residual units), SnakeBeta, conv k7 -> 1, clip
        Hh, rows = layers[li][0], h.shape[1]
        w = ops.conv1d(X[li][:, :Hh + rows], W["init"], lout=rows)
        li += 1
        for bw in W["blocks"]:
            r = bw["r"]
            rows = w.shape[1] * r
            H_, rpf = layers[li][0], layers[li][2]
            ops.conv1d(w, bw["up"], stride=r, pad_left=0, lout=rows + r, pre=bw["snake"], transpose=True, out=X[li][:, H_:H_ + rows + r])
            if off > 0:
                t0 = H_ + S["prev"] * rpf
                ops.stream_rows([(prev[li][:, t0:t0 + r], X[li][:, H_:H_ + r], True)])
            for ui, u in enumerate(bw["units"]):
                Hu = layers[li][0]
                t = ops.conv1d(X[li][:, :Hu + rows], u["c1"], dilation=u["d"], lout=rows, pre=u["s1"])
                Hn = layers[li + 1][0]
                last_unit = ui == len(bw["units"]) - 1
                out = X[li + 1][:, Hn:Hn + rows] if (not last_unit or bw is W["blocks"][-1]) else None
                w = ops.conv1d(t, u["c2"], pre=u["s2"], res=X[li][:, Hu:Hu + rows], out=out)
                li += 1
        Hh, rows = layers[li][0], w.shape[1]
        wav = ops.conv1d(X[li][:, :Hh + rows], W["out_conv"], lout=rows, pre=W["out_snake"], post_act=ACT["clip1"])
        # ---- carry: the last H rows of every buffered input become the other copy's history head (one launch)
        carry = []
        for (H, C, rpf, extra), buf, nb in zip(layers, X, prev):
            end = H + L * rpf
            carry.append((buf[:, end - H:end], nb[:, :H], False))
        ops.stream_rows(carry)
        S["p"], S["off"], S["prev"] = 1 - p, off + L, L
        return wav.reshape(B, 1, -1)


class Qwen3TTSSpeechTokenizerEncoder:
    """speech_tokenizer.py:957-1058: SEANet encoder -> encoder transformer -> stride-2 ConvDownsample1d -> split RVQ, keeping the first
    ``valid_num_quantizers`` code books.  The launch sequence is Mimi's encode (codec/models/mimi.py: ``encode_latent`` /
    ``encode_codes``) with the two switches the reference sets here: a full causal mask (no ``context`` window, :1050-1055) and half-split
    RoPE (``rope_traditional=False``, :1009).  The residual chain is sequential, so only the kept books are searched."""

    def __init__(self, config: Qwen3TTSTokenizerEncoderConfig, valid_num_quantizers: int = 16, device="cuda"):
        c = config
        if c.num_key_value_heads != c.num_attention_heads or c.num_residual_layers != 1 or c.use_conv_shortcut or not c.use_causal_conv:
            raise NotImplementedError("Qwen3TTSSpeechTokenizerEncoder: the encode chain covers causal convs, one identity-shortcut residual "
                                      "layer per block and one KV head per attention head")
        self.config = config
        self.device = torch.device(device)
        self.valid_num_quantizers = min(int(valid_num_quantizers), c.num_quantizers)
        encoder_frame_rate = c.sampling_rate / float(np.prod(c.upsampling_ratios))
        self.mimi_config = mimi.MimiConfig(
            dimension=c.hidden_size, nfilters=c.num_filters, ratios=list(c.upsampling_ratios), ksize=c.kernel_size,
            residual_ksize=c.residual_kernel_size, last_ksize=c.last_kernel_size, compress=c.compress, num_heads=c.num_attention_heads,
            num_layers=c.num_hidden_layers, dim_feedforward=c.intermediate_size, context=c.sliding_window, max_period=float(int(c.rope_theta)),
            nq=c.num_quantizers, bins=c.codebook_size, qdim=c.codebook_dim, upsample_stride=int(encoder_frame_rate / c.frame_rate),
            sample_rate=float(c.sampling_rate), frame_rate=c.frame_rate)
        self._enc = None

    def load_weights(self, weights, prefix: str = "encoder_model."):
        """``weights``: names and layouts of ``Qwen3TTSSpeechTokenizerEncoder.sanitize`` (``encoder_model.`` prefix), codebooks as
        (embedding_sum, cluster_usage) -> embedding_sum / max(cluster_usage, 1e-5) (quantization.py:26-30)."""
        P, cfg, dev = {k[len(prefix):]: v for k, v in dict(weights).items() if k.startswith(prefix)}, self.mimi_config, self.device

        def emb(pre):
            return P[pre + ".embedding_sum"].float() / torch.clamp(P[pre + ".cluster_usage"].float(), min=1e-5)[:, None]
        cb_first = torch.stack([emb("quantizer.rvq_first.vq.layers.0.codebook")]).to(dev).contiguous()
        cb_rest = torch.stack([emb(f"quantizer.rvq_rest.vq.layers.{i}.codebook") for i in range(cfg.nq - 1)]).to(dev).contiguous() \
            if cfg.nq > 1 else None
        self._enc = mimi.load_encoder(P, cfg, dev, cb_first, cb_rest)
        return self

    @torch.no_grad()
    def encode_latent(self, audio: torch.Tensor) -> torch.Tensor:
        """audio [B, 1, n] at 24 kHz -> the 12.5 Hz latent [B, ceil(n / 1920), hidden_size] in front of the quantiser."""
        return mimi.encode_latent(self._enc, self.mimi_config, audio, self.device, rope_traditional=False, window=0)

    @torch.no_grad()
    def encode(self, audio: torch.Tensor) -> torch.Tensor:
        """audio [B, 1, n] at 24 kHz -> int64 codes [B, valid_num_quantizers, ceil(n / 1920)] (:1037-1058)."""
        return mimi.encode_codes(self._enc, self.encode_latent(audio), self.valid_num_quantizers)

    @staticmethod
    def sanitize(weights):
        """Encoder half of speech_tokenizer.py:1220-1447: the checkpoint's ``encoder.*`` keys (transformers' Mimi state-dict names) ->
        the reference's ``encoder_model.*`` module tree.  SEANet layer indices -> init / residual / downsample / final convs, q / k / v ->
        one ``in_proj``, conv weights (out, in, K) -> (out, K, in), codebooks kept as (embedding_sum, cluster_usage)."""
        conv_map = {0: "encoder.init_conv1d", 3: "encoder.layers.0.downsample", 6: "encoder.layers.1.downsample",
                    9: "encoder.layers.2.downsample", 12: "encoder.layers.3.downsample", 14: "encoder.final_conv1d"}
        res_map, blk_map = {1: 0, 4: 1, 7: 2, 10: 3}, {1: 0, 3: 1}
        tr = {"self_attn.o_proj.weight": "self_attn.out_proj.weight", "mlp.fc1.weight": "gating.linear1.weight",
              "mlp.fc2.weight": "gating.linear2.weight", "input_layernorm.weight": "norm1.weight", "input_layernorm.bias": "norm1.bias",
              "post_attention_layernorm.weight": "norm2.weight", "post_attention_layernorm.bias": "norm2.bias",
              "self_attn_layer_scale.scale": "layer_scale_1.scale", "mlp_layer_scale.scale": "layer_scale_2.scale"}
        sw = lambda v: v.transpose(-1, -2) if v.dim() == 3 else v                                  # noqa: E731
        out, qkv = {}, {}
        for k, v in weights.items():
            if not k.startswith("encoder."):
                continue
            v = torch.as_tensor(v)
            parts = k.split(".")
            if k.startswith("encoder.encoder.layers."):
                n = int(parts[3])
                if "block" in k:
                    if n not in res_map or int(parts[5]) not in blk_map:
                        continue
                    base, suffix = f"encoder.layers.{res_map[n]}.residuals.0.block.{blk_map[int(parts[5])]}", ".".join(parts[6:])
                else:
                    if n not in conv_map:
                        continue
                    base, suffix = conv_map[n], ".".join(parts[4:])
                out[f"encoder_model.{base}.conv.{suffix}"] = sw(v) if "weight" in suffix else v
            elif k.startswith("encoder.encoder_transformer.layers."):
                li, rest = int(parts[3]), ".".join(parts[4:])
                if rest in ("self_attn.q_proj.weight", "self_attn.k_proj.weight", "self_attn.v_proj.weight"):
                    qkv.setdefault(li, {})[rest.split(".")[1][0]] = v
                elif rest in tr:
                    out[f"encoder_model.encoder_transformer.transformer.layers.{li}.{tr[rest]}"] = v
            elif k.startswith("encoder.downsample."):
                suffix = k[len("encoder.downsample."):]
                out[f"encoder_model.downsample.conv.conv.{suffix}"] = sw(v) if "weight" in suffix else v
            elif k.startswith("encoder.quantizer."):
                rest = k[len("encoder.quantizer."):]
                which = "rvq_first" if "semantic_residual_vector_quantizer" in rest else "rvq_rest"
                if ".codebook.cluster_usage" in rest or ".codebook.embed_sum" in rest:
                    li = int(rest.split("layers.")[1].split(".")[0])
                    name = "cluster_usage" if "cluster_usage" in rest else "embedding_sum"
                    out[f"encoder_model.quantizer.{which}.vq.layers.{li}.codebook.{name}"] = v
                elif "input_proj.weight" in rest or "output_proj.weight" in rest:
                    out[f"encoder_model.quantizer.{which}.{'input_proj' if 'input_proj' in rest else 'output_proj'}.weight"] = sw(v)
        for li, d in qkv.items():
            if len(d) == 3:
                out[f"encoder_model.encoder_transformer.transformer.layers.{li}.self_attn.in_proj.weight"] = torch.cat([d["q"], d["k"], d["v"]], 0)
        return out


class Qwen3TTSSpeechTokenizer:
    """speech_tokenizer.py:1061-1217."""

    def __init__(self, config: Qwen3TTSTokenizerConfig, device="cuda"):
        self.config = config
        self.encoder_valid_num_quantizers = config.encoder_valid_num_quantizers
        self.input_sample_rate = config.input_sample_rate
        self.output_sample_rate = config.output_sample_rate
        self.decode_upsample_rate = config.decode_upsample_rate
        self.encode_downsample_rate = config.encode_downsample_rate
        self.decoder = Qwen3TTSSpeechTokenizerDecoder(config.decoder_config, device)
        self.encoder_model = None
        self.device = torch.device(device)

    @property
    def has_encoder(self) -> bool:
        return self.encoder_model is not None

    def load_weights(self, weights):
        """Decoder weights (``decoder.*``, after ``sanitize``) and, when the config has an ``encoder_config`` and the dict holds
        ``encoder_model.*`` weights (after ``Qwen3TTSSpeechTokenizerEncoder.sanitize``), the encoder."""
        weights = dict(weights)
        self.decoder.load_weights(weights, prefix="decoder.")
        if self.config.encoder_config is not None and any(k.startswith("encoder_model.") for k in weights):
            self.encoder_model = Qwen3TTSSpeechTokenizerEncoder(self.config.encoder_config, self.encoder_valid_num_quantizers,
                                                                self.device).load_weights(weights)
        return self

    def encode(self, audio):
        """audio [B, 1, samples] at 24 kHz -> codes [B, 16, ceil(samples / 1920)] (speech_tokenizer.py:1082-1093)."""
        if self.encoder_model is None:
            raise ValueError("Encoder not available for this speech tokenizer")      # same error as speech_tokenizer.py:1092-1093
        return self.encoder_model.encode(audio)

    def decode(self, audio_codes: torch.Tensor):
        """audio_codes [B, T, 16] -> (wav [B, samples], audio_lengths [B])."""
        audio_codes = audio_codes.to(self.device)
        wav = self.decoder.chunked_decode(audio_codes.transpose(1, 2)).squeeze(1)
        lengths = (audio_codes[..., 0] > 0).sum(dim=1) * self.decode_upsample_rate
        return wav, lengths

    def batch_decode(self, codes_list):
        """speech_tokenizer.py:1120-1179: pad to the longest with code 0, decode as one batch, trim per sequence."""
        if not codes_list:
            return [], []
        normed = [c[None] if c.dim() == 2 else c for c in codes_list]
        seq_lens = [c.shape[1] for c in normed]
        max_len, nq = max(seq_lens), normed[0].shape[2]
        batch = torch.zeros(len(normed), max_len, nq, dtype=torch.int64, device=self.device)
        for i, c in enumerate(normed):
            batch[i, : c.shape[1]] = c[0].to(self.device)
        wav = self.decoder.chunked_decode(batch.transpose(1, 2)).squeeze(1)
        lengths = [int(sl) * self.decode_upsample_rate for sl in seq_lens]
        audios = []
        for b, n in enumerate(lengths):
            a = wav[b]
            audios.append(a[:n] if 0 < n < a.shape[0] else a)
        return audios, lengths

    def streaming_decode(self, audio_codes: torch.Tensor, chunk_tokens: int = 100):
        """speech_tokenizer.py:1181-1217: yields [B, samples] per chunk of ``chunk_tokens`` frames (25 frames left context)."""
        codes = audio_codes.to(self.device).transpose(1, 2)
        total, start = codes.shape[-1], 0
        while start < total:
            end = min(start + chunk_tokens, total)
            ctx = 25 if start - 25 > 0 else start
            wav = self.decoder(codes[..., start - ctx: end])[..., ctx * self.decode_upsample_rate:]
            yield wav.squeeze(1)
            start = end

    @staticmethod
    def sanitize(weights):
        """Decoder half of speech_tokenizer.py:1220-1447: PyTorch conv layouts -> [out, K, in], transposed convs
        [in, out, K] -> [out, K, in], codebooks = embedding_sum / clip(cluster_usage, 1e-5)."""
        out, codebook = {}, {}
        for k, v in weights.items():
            if k.startswith("encoder."):
                continue                                                # encode side: Qwen3TTSSpeechTokenizerEncoder.sanitize
            if "_codebook.cluster_usage" in k or "_codebook.embedding_sum" in k:
                base = k.rsplit("._codebook.", 1)[0]
                codebook.setdefault(base, {})["cluster_usage" if "cluster_usage" in k else "embedding_sum"] = v
                continue
            is_tr = ("upsample" in k and ".0.conv.weight" in k) or ("decoder.decoder" in k and "block.1.conv.weight" in k)
            if is_tr and v.dim() == 3:
                v = v if check_array_shape_qwen3(v) else v.permute(1, 2, 0)
            elif ("conv.weight" in k or "_proj.weight" in k) and v.dim() == 3:
                v = v if check_array_shape_qwen3(v) else v.permute(0, 2, 1)
            out[k] = v
        for base, d in codebook.items():
            if "cluster_usage" in d and "embedding_sum" in d:
                out[f"{base}.codebook.embed.weight"] = d["embedding_sum"] / torch.clamp(d["cluster_usage"][:, None], min=1e-5)
        return out
