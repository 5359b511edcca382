"""Kyutai Mimi codec, decode side, on H100 (reference: codec/models/mimi/mimi.py + modules/*).

``Mimi(mimi_202407(nq)).load_weights(...)``, ``decode(codes[B,nq,T]) -> [B,1,1920 T]`` (mimi.py:155-162).
RVQ gather-sum in one kernel, windowed causal attention (context 250) without materialising the
O(T^2) mask the reference builds (transformer.py:98-107), ELU / LayerScale / residual adds fused into
the neighbouring convs.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import math

import torch

from ... import ops
from ...ops import ACT, Pre


@dataclass
class MimiConfig:
    """Flat restatement of MimiConfig / SeanetConfig / TransformerConfig (mimi.py:35-96)."""
    dimension: int = 512
    nfilters: int = 64
    ratios: list = field(default_factory=lambda: [8, 6, 5, 4])
    ksize: int = 7
    residual_ksize: int = 3
    last_ksize: int = 3
    compress: int = 2
    num_heads: int = 8
    num_layers: int = 8
    dim_feedforward: int = 2048
    context: int = 250
    max_period: float = 10000.0
    nq: int = 32
    bins: int = 2048
    qdim: int = 256
    upsample_stride: int = 2
    sample_rate: float = 24000.0
    frame_rate: float = 12.5


def mimi_202407(num_codebooks: int) -> MimiConfig:
    return MimiConfig(nq=num_codebooks)


class Mimi:
    def __init__(self, cfg: MimiConfig, device="cuda"):
        self.cfg = cfg
        self.device = torch.device(device)
        self._w = None
        self._enc = None
        self._states = {}
        self._dec_state = None
        self._enc_state = None

    @property
    def frame_rate(self):
        return self.cfg.frame_rate

    @property
    def sample_rate(self):
        return self.cfg.sample_rate

    def reset_state(self):
        """mimi.py:138-144: forget the streaming state of both directions."""
        self._dec_state = None
        self._enc_state = None

    @torch.no_grad()
    def decode_step(self, xs: torch.Tensor) -> torch.Tensor:
        """mimi.py:171-176: the next ``T_new`` code frames [B, nq, T_new] -> their samples [B, 1, 1920 T_new], exactly the matching slice of a
        one-shot ``decode`` of the whole stream for any chunking.  Incremental: every causal conv carries its unconsumed input rows, every
        transposed conv its held-back tail, the transformer a ring KV cache of ``context`` + chunk positions -- the cost of a call does not
        depend on how far into the stream it is and memory stays bounded.  Single-frame steps replay a CUDA graph captured once per batch
        size.  ``reset_state()`` / ``decode()`` start a new stream; the batch size is fixed at the first step after that."""
        xs = xs.to(device=self.device, dtype=torch.int64)
        if xs.dim() != 3 or not 1 <= xs.shape[1] <= self.cfg.nq:
            raise ValueError(f"decode_step: expected codes [B, <= {self.cfg.nq}, T], got {tuple(xs.shape)}")
        st = self._dec_state
        if st is None:
            st = self._dec_state = self._state("dec", xs.shape[0])
        elif xs.shape[0] != st.B:
            raise ValueError(f"decode_step: batch size {xs.shape[0]} differs from the stream's {st.B} (reset_state() starts a new stream)")
        return st.decode(xs)

    @torch.no_grad()
    def encode_step(self, xs: torch.Tensor) -> torch.Tensor:
        """mimi.py:164-169: the next ``n`` samples pcm [B, 1, n] -> int64 codes [B, nq, F] of the F frames this call completes (possibly 0);
        leftover samples are carried.  Over a stream the codes equal ``encode`` of the concatenated audio (for audio ending on a frame
        boundary).  ``reset_state()`` / ``encode()`` start a new stream; the batch size is fixed at the first step after that."""
        if self._enc is None:
            raise ValueError("Mimi.encode_step: the loaded weights have no encoder (encoder.*, encoder_transformer.*, downsample.*)")
        xs = xs.to(device=self.device, dtype=torch.float32)
        if xs.dim() != 3 or xs.shape[1] != 1:
            raise ValueError(f"encode_step: expected pcm [B, 1, n], got {tuple(xs.shape)}")
        st = self._enc_state
        if st is None:
            st = self._enc_state = self._state("enc", xs.shape[0])
        elif xs.shape[0] != st.B:
            raise ValueError(f"encode_step: batch size {xs.shape[0]} differs from the stream's {st.B} (reset_state() starts a new stream)")
        return st.encode(xs)

    def _state(self, direction: str, B: int) -> "MimiStreamState":
        """The (B, direction) state: allocated once, zeroed in place for every new stream (a captured graph keeps its buffers)."""
        key = (direction, B)
        st = self._states.get(key)
        if st is None:
            st = self._states[key] = MimiStreamState(self, direction, B)
        st.reset()
        return st

    @property
    def span_halo(self) -> int:
        """Left context (code frames) that makes a span decode exact: the stack is causal; each of the transformer's layers looks back
        ``context`` positions (at ``upsample_stride`` positions per frame), so the receptive field of the stack is num_layers * context
        positions, plus a few frames for the causal convolutions either side of it."""
        c = self.cfg
        return -(-(c.num_layers * c.context) // c.upsample_stride) + 16

    @torch.no_grad()
    def decode_span(self, codes: torch.Tensor, start: int, end: int, halo=None) -> torch.Tensor:
        """Samples of code frames [start, end) -- equal to that slice of ``decode(codes)`` -- from the frames themselves plus ``halo``
        frames of left context (SURVEY.md section 8e: one stream sharded across GPUs).  Returns [B, 1, (end - start) * 1920]."""
        halo = self.span_halo if halo is None else halo
        T = codes.shape[-1]
        if not 0 <= start < end <= T:
            raise ValueError(f"decode_span: need 0 <= start < end <= {T}")
        rs = max(0, start - halo)
        pcm = self.decode(codes[:, :, rs:end])
        hop = pcm.shape[-1] // (end - rs)
        return pcm[..., (start - rs) * hop:]

    @staticmethod
    def sanitize_pytorch_weights(weights: dict) -> dict:
        """The key / layout mapping of ``Mimi.load_pytorch_weights`` (mimi.py:196-249): kyutai's PyTorch checkpoint names -> the reference's
        module tree (leading underscores dropped, SEANet ``model.N`` indices -> ``layers.i.{upsample,downsample,residuals.0}``, transformer
        ``in_proj_weight`` / ``linearN`` renames), conv weights (out, in, K) -> (out, K, in), transposed-conv weights (in, out/g, K) ->
        (out, K, in/g)."""
        out = {}
        for k, v in weights.items():
            k = ".".join(s.removeprefix("_") for s in k.split("."))
            if k.startswith("encoder.model."):
                k = k.replace("encoder.model.", "encoder.")
            if k.startswith("decoder.model."):
                k = k.replace("decoder.model.", "decoder.")
            if k.endswith(".in_proj_weight"):
                k = k.replace(".in_proj_weight", ".in_proj.weight")
            if k.endswith(".linear1.weight"):
                k = k.replace(".linear1.weight", ".gating.linear1.weight")
            if k.endswith(".linear2.weight"):
                k = k.replace(".linear2.weight", ".gating.linear2.weight")
            for li, di in enumerate((2, 5, 8, 11)):
                k = k.replace(f"decoder.{di}.", f"decoder.layers.{li}.upsample.")
                k = k.replace(f"decoder.{di + 1}.", f"decoder.layers.{li}.residuals.0.")
            for li, ei in enumerate((1, 4, 7, 10)):
                k = k.replace(f"encoder.{ei}.", f"encoder.layers.{li}.residuals.0.")
                k = k.replace(f"encoder.{ei + 2}.", f"encoder.layers.{li}.downsample.")
            k = k.replace("decoder.0.", "decoder.init_conv1d.").replace("decoder.14.", "decoder.final_conv1d.")
            k = k.replace("encoder.0.", "encoder.init_conv1d.").replace("encoder.14.", "encoder.final_conv1d.")
            k = k.replace(".block.1.", ".block.0.").replace(".block.3.", ".block.1.")
            if k.endswith((".conv.weight", ".output_proj.weight", ".input_proj.weight")):
                v = v.transpose(-1, -2)
            if k.endswith(".convtr.weight"):
                v = v.permute(0, 2, 1) if (v.dim() == 3 and v.shape[1] == 1) else v.permute(1, 2, 0)
            out[k] = v.contiguous()
        return out

    @classmethod
    def from_pretrained(cls, repo_id, filename: str = "tokenizer-e351c8d8-checkpoint125.safetensors", device="cuda"):
        """mimi.py:264-275: the 32-codebook 2024-07 configuration from kyutai's checkpoint; ``repo_id`` may be a local directory."""
        from pathlib import Path
        f = Path(repo_id) / filename
        if not f.exists():
            from huggingface_hub import hf_hub_download
            f = Path(hf_hub_download(repo_id, filename))
        return cls(mimi_202407(32), device=device).load_pytorch_weights(f, strict=True)

    def load_pytorch_weights(self, file, strict: bool = True):
        """mimi.py:192-262: ``file`` = path of kyutai's safetensors checkpoint (or an already loaded dict)."""
        if not isinstance(file, dict):
            from safetensors.torch import load_file
            file = load_file(str(file))
        return self.load_weights(self.sanitize_pytorch_weights(file), strict=strict)

    def load_weights(self, weights, strict=True):
        P, cfg, dev = dict(weights), self.cfg, self.device
        f = lambda t: t.float().to(dev).contiguous()
        bf = lambda t: t.float().to(torch.bfloat16).float()

        def emb(pre):                                                   # quantization.py:26-30
            usage = torch.clamp(P[pre + ".cluster_usage"].float(), min=1e-5)[:, None]
            return P[pre + ".embedding_sum"].float() / usage

        W = {}
        W["cb_first"] = f(torch.stack([emb("quantizer.rvq_first.vq.layers.0.codebook")]))
        W["cb_rest"] = f(torch.stack([emb(f"quantizer.rvq_rest.vq.layers.{i}.codebook") for i in range(cfg.nq - 1)])) if cfg.nq > 1 else None
        W["proj_first"] = ops.pack_conv(P["quantizer.rvq_first.output_proj.weight"].float(), None, 1, dev)
        W["proj_rest"] = ops.pack_conv(P["quantizer.rvq_rest.output_proj.weight"].float(), None, 1, dev) if cfg.nq > 1 else None
        W["upsample"] = ops.pack_conv(P["upsample.convtr.convtr.convtr.weight"].float(), None, cfg.dimension, dev)
        W["layers"] = []
        for li in range(cfg.num_layers):
            L = f"decoder_transformer.transformer.layers.{li}"
            W["layers"].append({
                "n1": (f(P[L + ".norm1.weight"]), f(P[L + ".norm1.bias"])), "n2": (f(P[L + ".norm2.weight"]), f(P[L + ".norm2.bias"])),
                "in_proj": ops.pack_linear(P[L + ".self_attn.in_proj.weight"].float(), None, dev),
                "out_proj": ops.pack_linear(P[L + ".self_attn.out_proj.weight"].float(), None, dev),
                "l1": ops.pack_linear(P[L + ".gating.linear1.weight"].float(), None, dev),
                "l2": ops.pack_linear(P[L + ".gating.linear2.weight"].float(), None, dev),
                "ls1": f(P[L + ".layer_scale_1.scale"]), "ls2": f(P[L + ".layer_scale_2.scale"])})
        cw = lambda pre: ops.pack_conv(P[pre + ".weight"].float(), P.get(pre + ".bias"), 1, dev)
        W["init"] = cw("decoder.init_conv1d.conv.conv")
        W["dec"] = []
        for li, r in enumerate(cfg.ratios):
            L = f"decoder.layers.{li}"
            W["dec"].append({"r": r, "up": cw(L + ".upsample.convtr.convtr"), "c0": cw(L + ".residuals.0.block.0.conv.conv"),
                             "c1": cw(L + ".residuals.0.block.1.conv.conv")})
        W["final"] = cw("decoder.final_conv1d.conv.conv")
        del bf
        self._w = W
        self._enc = None
        self._states = {}
        self.reset_state()
        if "encoder.init_conv1d.conv.conv.weight" in P:                 # encode side (seanet.py:194-199, mimi.py:146-153, quantization.py:178-185)
            self._enc = load_encoder(P, cfg, dev, W["cb_first"], W["cb_rest"])
        return self

    @torch.no_grad()
    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        """codes int64 [B, nq, T] -> pcm [B, 1, 1920 T]."""
        W, cfg, dev = self._w, self.cfg, self.device
        self._dec_state = None                                          # decode() resets the decode stream (mimi.py:156-158)
        codes = codes.to(device=dev, dtype=torch.int64).contiguous()
        B, nq, T = codes.shape
        q = ops.rvq_decode(codes[:, :1], W["cb_first"])
        x = ops.conv1d(q, W["proj_first"])
        if nq > 1:
            q2 = ops.rvq_decode(codes[:, 1:], W["cb_rest"][: nq - 1])
            x = ops.conv1d(q2, W["proj_rest"], res=x)
        s = cfg.upsample_stride
        x = ops.conv1d(x, W["upsample"], stride=s, pad_left=0, lout=T * s, transpose=True)         # causal: trim k-s on the right
        x = self._transformer(x, W["layers"])
        elu = Pre(act=ACT["elu"])
        x = ops.conv1d(x, W["init"], pad_left=cfg.ksize - 1, lout=x.shape[1])
        for lw in W["dec"]:
            r = lw["r"]
            y = ops.conv1d(x, lw["up"], stride=r, pad_left=0, lout=x.shape[1] * r, pre=elu, transpose=True)
            t = ops.conv1d(y, lw["c0"], pad_left=cfg.residual_ksize - 1, lout=y.shape[1], pre=elu)
            x = ops.conv1d(t, lw["c1"], pre=elu, res=y)
        pcm = ops.conv1d(x, W["final"], pad_left=cfg.last_ksize - 1, lout=x.shape[1], pre=elu)      # [B, L, 1]
        return pcm.reshape(B, 1, -1)

    def _transformer(self, x: torch.Tensor, layers) -> torch.Tensor:
        return _transformer(x, layers, self.cfg)

    @torch.no_grad()
    def encode_latent(self, xs: torch.Tensor) -> torch.Tensor:
        """pcm [B, 1, n] -> the 12.5 Hz latent [B, ceil(n / 1920), 512] in front of the quantiser (mimi.py:146-152)."""
        if self._enc is None:
            raise ValueError("Mimi.encode: the loaded weights have no encoder (encoder.*, encoder_transformer.*, downsample.*)")
        return encode_latent(self._enc, self.cfg, xs, self.device)

    @torch.no_grad()
    def encode(self, xs: torch.Tensor) -> torch.Tensor:
        """mimi.py:146-153: pcm [B, 1, n] -> int64 codes [B, nq, ceil(n / 1920)]: SEANet encoder, encoder transformer, stride-2 replicate-padded
        down-sampling conv, then the split residual quantiser (quantization.py:178-185): the first codebook on its own projection, the other
        nq - 1 as a residual chain on theirs -- `rvq_encode_kernel` runs the chain (argmin |e|^2 / 2 - x.e, first index on ties)."""
        self._enc_state = None                                          # encode() resets the encode stream (mimi.py:147-149)
        return encode_codes(self._enc, self.encode_latent(xs))


# ------------------------------------------------------------------------------------------------------------------- encode side
# Shared by Mimi.encode and the Qwen3-TTS speech-tokenizer encoder (speech_tokenizer.py:957-1058), which is Mimi's encoder with a full
# causal mask, half-split RoPE and only its first code books kept.
def _transformer(x: torch.Tensor, layers, cfg: MimiConfig, rope_traditional: bool = True, window=None) -> torch.Tensor:
    """ProjectedTransformer (mimi/modules/transformer.py:63-261), fresh cache: pre-norm layers, RoPE (``rope_traditional``: interleaved
    pairs, else rotate_half), causal attention inside a ``window``-position window (None: ``cfg.context``; 0: full causal), LayerScale on
    both residual branches."""
    d, nh = cfg.dimension, cfg.num_heads
    win = cfg.context if window is None else window
    for lw in layers:
        n1 = ops.layernorm(x, *lw["n1"], eps=1e-5)
        qkv = ops.linear(n1, lw["in_proj"])
        ops.rope_(qkv[:, :, :d], nh, offset=0, base=cfg.max_period, traditional=rope_traditional)
        ops.rope_(qkv[:, :, d:2 * d], nh, offset=0, base=cfg.max_period, traditional=rope_traditional)
        att = ops.attention(qkv[:, :, :d], qkv[:, :, d:2 * d], qkv[:, :, 2 * d:], n_heads=nh, scale=(d // nh) ** -0.5,
                            causal=True, window=win)
        x = ops.linear(att, lw["out_proj"], cscale=lw["ls1"], res=x)
        n2 = ops.layernorm(x, *lw["n2"], eps=1e-5)
        m = ops.linear(n2, lw["l1"], post_act=ACT["gelu_tanh"])
        x = ops.linear(m, lw["l2"], cscale=lw["ls2"], res=x)
    return x


def _cconv(x, cw, ksize, stride=1, pre=None, pad_mode=0, res=None):
    """StreamableConv1d (mimi/modules/conv.py:224-243), causal: k - stride samples of left padding, the right edge padded up to a whole
    last frame (zeros, or the edge sample for ``pad_mode=1``)."""
    L = x.shape[1]
    pad_total = ksize - stride
    lout = int(math.ceil(max(L + pad_total - ksize, 0) / stride + 1.0))
    return ops.conv1d(x, cw, stride=stride, pad_left=pad_total, lout=lout, pad_mode=pad_mode, pre=pre, res=res)


def load_encoder(P, cfg: MimiConfig, dev, cb_first: torch.Tensor, cb_rest) -> dict:
    """Encode-side weights from the reference's names (``encoder.*``, ``encoder_transformer.*``, ``downsample.*``, the quantiser's
    ``input_proj``s) and the quantiser's codebooks ``cb_first`` [1, bins, qdim] / ``cb_rest`` [nq - 1, bins, qdim] (or None)."""
    f = lambda t: t.float().to(dev).contiguous()
    cw = lambda pre: ops.pack_conv(P[pre + ".weight"].float(), P.get(pre + ".bias"), 1, dev)
    tr = []
    for li in range(cfg.num_layers):
        L = f"encoder_transformer.transformer.layers.{li}"
        tr.append({
            "n1": (f(P[L + ".norm1.weight"]), f(P[L + ".norm1.bias"])), "n2": (f(P[L + ".norm2.weight"]), f(P[L + ".norm2.bias"])),
            "in_proj": ops.pack_linear(P[L + ".self_attn.in_proj.weight"].float(), None, dev),
            "out_proj": ops.pack_linear(P[L + ".self_attn.out_proj.weight"].float(), None, dev),
            "l1": ops.pack_linear(P[L + ".gating.linear1.weight"].float(), None, dev),
            "l2": ops.pack_linear(P[L + ".gating.linear2.weight"].float(), None, dev),
            "ls1": f(P[L + ".layer_scale_1.scale"]), "ls2": f(P[L + ".layer_scale_2.scale"])})
    E = {"init": cw("encoder.init_conv1d.conv.conv"), "layers": [], "final": cw("encoder.final_conv1d.conv.conv"), "tr": tr,
         "down": cw("downsample.conv.conv.conv"), "cb_first": cb_first, "cb_rest": cb_rest}
    for li, r in enumerate(reversed(cfg.ratios)):
        L = f"encoder.layers.{li}"
        E["layers"].append({"r": r, "c0": cw(L + ".residuals.0.block.0.conv.conv"), "c1": cw(L + ".residuals.0.block.1.conv.conv"),
                            "down": cw(L + ".downsample.conv.conv")})
    for name, cb in (("first", cb_first), ("rest", cb_rest)):
        if cb is None:
            continue
        E["in_" + name] = ops.pack_conv(P[f"quantizer.rvq_{name}.input_proj.weight"].float(), None, 1, dev)
        E["c2_" + name] = ((cb.double() ** 2).sum(-1) / 2).contiguous()             # |e|^2 / 2 of argmin(|e|^2 / 2 - x.e)
    return E


def encode_latent(E: dict, cfg: MimiConfig, xs: torch.Tensor, device, *, rope_traditional: bool = True, window=None) -> torch.Tensor:
    """pcm [B, 1, n] -> latent [B, ceil(n / 1920), dimension]: SEANet encoder, encoder transformer (switches as in ``_transformer``),
    stride-2 replicate-padded down-sampling conv."""
    x = xs.to(device=device, dtype=torch.float32)
    x = x.reshape(x.shape[0], -1, 1)                                 # [B, 1, n] -> [B, n, 1] (one channel: same memory)
    elu = Pre(act=ACT["elu"])
    x = _cconv(x, E["init"], cfg.ksize)
    for lw in E["layers"]:
        t = _cconv(x, lw["c0"], cfg.residual_ksize, pre=elu)
        y = _cconv(t, lw["c1"], 1, pre=elu, res=x)                   # block(x) + x  (seanet.py:61-66)
        x = _cconv(y, lw["down"], 2 * lw["r"], stride=lw["r"], pre=elu)
    x = _cconv(x, E["final"], cfg.last_ksize, pre=elu)
    x = _transformer(x, E["tr"], cfg, rope_traditional, window)
    s = cfg.upsample_stride
    return _cconv(x, E["down"], 2 * s, stride=s, pad_mode=1)


def encode_codes(E: dict, z: torch.Tensor, n_books=None) -> torch.Tensor:
    """Split residual quantiser (quantization.py:178-185): latent [B, T, dimension] -> int64 codes [B, n_books, T] (default: every book).
    The residual chain is sequential, so running only the first ``n_books`` gives exactly the first ``n_books`` codes of the full chain."""
    B, T, _ = z.shape
    r1 = ops.conv1d(z, E["in_first"])
    codes = [ops.rvq_encode(r1.reshape(B * T, -1), E["cb_first"], E["c2_first"]).reshape(B, T, 1)]
    n_rest = 0 if E["cb_rest"] is None else E["cb_rest"].shape[0]
    if n_books is not None:
        n_rest = min(n_rest, n_books - 1)
    if n_rest > 0:
        r2 = ops.conv1d(z, E["in_rest"])
        codes.append(ops.rvq_encode(r2.reshape(B * T, -1), E["cb_rest"][:n_rest], E["c2_rest"][:n_rest]).reshape(B, T, -1))
    return torch.cat(codes, dim=2).transpose(1, 2).contiguous()


# ------------------------------------------------------------------------------------------------------------------- streaming
STREAM_PIECE_FRAMES = 128     # a longer call runs in pieces of this many frames: bounds the ring (context + 2 x 128 positions) and activations


def _stream_transformer(x: torch.Tensor, layers, cfg: MimiConfig, k_ring, v_ring, ctr: torch.Tensor) -> torch.Tensor:
    """``_transformer`` for the next positions of a stream: RoPE at the absolute positions ctr[0] + t, k / v into each layer's ring, the
    ``cfg.context`` window over the ring (transformer.py:79-112 with a growing KVCache)."""
    d, nh = cfg.dimension, cfg.num_heads
    for lw, kr, vr in zip(layers, k_ring, v_ring):
        n1 = ops.layernorm(x, *lw["n1"], eps=1e-5)
        qkv = ops.linear(n1, lw["in_proj"])
        ops.ring_rope_kv(qkv, nh, kr, vr, ctr, base=cfg.max_period)
        att = ops.ring_attn(qkv[:, :, :d], kr, vr, ctr, n_heads=nh, scale=(d // nh) ** -0.5, window=cfg.context)
        x = ops.linear(att, lw["out_proj"], cscale=lw["ls1"], res=x)
        n2 = ops.layernorm(x, *lw["n2"], eps=1e-5)
        m = ops.linear(n2, lw["l1"], post_act=ACT["gelu_tanh"])
        x = ops.linear(m, lw["l2"], cscale=lw["ls2"], res=x)
    return x


class MimiStreamState:
    """Device state of one streaming direction ("dec" or "enc") at batch size B, allocated once and zeroed in place by ``reset``:
    ``ctr`` int32 [ring position, history parity counter], per causal conv a two-slot history [2, B, keff - 1, Cin], per transposed conv
    its held-back tail [B, K - stride, Cout], per transformer layer a k and a v ring [B, context + 2 x STREAM_PIECE_FRAMES + 2, 512].
    Decode: single-frame steps replay a CUDA graph captured at the second such step (the first runs eagerly and creates any workspaces).
    Encode: the histories of the strided convs vary in length (tracked here); transformer positions are processed in whole frames, an odd
    one waits in ``pend``."""

    def __init__(self, mimi: "Mimi", direction: str, B: int):
        cfg, dev = mimi.cfg, mimi.device
        self.m, self.dir, self.B = mimi, direction, B
        z = lambda *shape: torch.zeros(*shape, device=dev, dtype=torch.float32)
        hist = lambda cw: z(2, B, max(cw.K - 1, 1), cw.cin)
        s, d = cfg.upsample_stride, cfg.dimension
        self.ctr = torch.zeros(2, device=dev, dtype=torch.int32)
        self.err = torch.zeros(1, device=dev, dtype=torch.int32)
        self.cap = cfg.context + s * STREAM_PIECE_FRAMES + s
        self.k_ring = [z(B, self.cap, d) for _ in range(cfg.num_layers)]
        self.v_ring = [z(B, self.cap, d) for _ in range(cfg.num_layers)]
        self.bufs = [self.ctr, self.err]
        if direction == "dec":
            W = mimi._w
            self.up_tail = z(B, W["upsample"].K - s, d)
            self.h_init, self.h_final = hist(W["init"]), hist(W["final"])
            self.dec = [{"tail": z(B, lw["up"].K - lw["r"], lw["up"].cout), "h0": hist(lw["c0"])} for lw in W["dec"]]
            self.bufs += [self.up_tail, self.h_init, self.h_final] + [t for sl in self.dec for t in sl.values()]
            self.graphs = {}              # nq -> (graph, static codes [B, nq, 1], static pcm)
            self.eager_single = 0
        else:
            E = mimi._enc
            self.convs = {"init": (E["init"], 1)}
            for i, lw in enumerate(E["layers"]):
                self.convs[f"c0_{i}"] = (lw["c0"], 1)
                self.convs[f"down_{i}"] = (lw["down"], lw["r"])
            self.convs["final"] = (E["final"], 1)
            self.convs["ds"] = (E["down"], s)
            self.hist = {k: hist(cw) for k, (cw, _) in self.convs.items()}
            self.pend = z(B, s, d)
            self.bufs += list(self.hist.values()) + [self.pend]

    def reset(self):
        for t in self.bufs:
            t.zero_()
        if self.dir == "enc":
            self.H = {k: cw.K - st for k, (cw, st) in self.convs.items()}        # the causal left padding (fresh: zeros / edge rows)
            self.fresh = {k: True for k in self.convs}
            self.npend = 0

    def _check(self):
        if int(self.err.item()) != 0:
            raise ValueError(f"decode_step: code index out of range [0, {self.m.cfg.bins})")

    # ---- decode
    def _decode_piece(self, codes: torch.Tensor) -> torch.Tensor:
        W, cfg = self.m._w, self.m.cfg
        B, nq, T = codes.shape
        q = ops.rvq_decode(codes[:, :1], W["cb_first"], check=False, err=self.err)
        x = ops.conv1d(q, W["proj_first"])
        if nq > 1:
            q2 = ops.rvq_decode(codes[:, 1:], W["cb_rest"][: nq - 1], check=False, err=self.err)
            x = ops.conv1d(q2, W["proj_rest"], res=x)
        s = cfg.upsample_stride
        x = ops.convtr1d_stream(x, W["upsample"], self.up_tail, stride=s)
        x = _stream_transformer(x, W["layers"], cfg, self.k_ring, self.v_ring, self.ctr)
        elu, step = Pre(act=ACT["elu"]), self.ctr[1:]
        x = ops.conv1d_stream(x, W["init"], self.h_init, cfg.ksize - 1, step)
        for lw, sl in zip(W["dec"], self.dec):
            y = ops.convtr1d_stream(x, lw["up"], sl["tail"], stride=lw["r"], pre=elu)
            t = ops.conv1d_stream(y, lw["c0"], sl["h0"], cfg.residual_ksize - 1, step, pre=elu)
            x = ops.conv1d(t, lw["c1"], pre=elu, res=y)
        pcm = ops.conv1d_stream(x, W["final"], self.h_final, cfg.last_ksize - 1, step, pre=elu)
        ops.stream_advance(self.ctr, s * T)
        return pcm.reshape(B, 1, -1)

    def decode(self, codes: torch.Tensor) -> torch.Tensor:
        B, nq, T = codes.shape
        if T == 0:
            return torch.zeros(B, 1, 0, device=codes.device, dtype=torch.float32)
        if T == 1 and GRAPH_SINGLE_FRAME[0]:
            ent = self.graphs.get(nq)
            if ent is None and self.eager_single > 0:
                cin = codes.contiguous().clone()
                torch.cuda.synchronize(codes.device)
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    out = self._decode_piece(cin)
                ent = self.graphs[nq] = (g, cin, out)
            if ent is not None:
                g, cin, out = ent
                cin.copy_(codes)
                g.replay()
                self._check()
                return out.clone()
            self.eager_single += 1
        codes = codes.contiguous()
        parts = [self._decode_piece(codes[:, :, a:a + STREAM_PIECE_FRAMES].contiguous()) for a in range(0, T, STREAM_PIECE_FRAMES)]
        self._check()
        return parts[0] if len(parts) == 1 else torch.cat(parts, dim=-1)

    # ---- encode
    def _conv(self, name: str, x, pre=None, res=None, pad_mode=0):
        cw, stride = self.convs[name]
        L = 0 if x is None else x.shape[1]
        y = ops.conv1d_stream(x if L else None, cw, self.hist[name], self.H[name], self.ctr[1:], B=self.B, stride=stride, pad_mode=pad_mode,
                              fresh=self.fresh[name], pre=pre, res=res)
        if not (self.fresh[name] and L == 0):
            self.H[name] += L - y.shape[1] * stride
            self.fresh[name] = False
        return y

    def _encode_piece(self, pcm: torch.Tensor) -> torch.Tensor:
        E, cfg, B = self.m._enc, self.m.cfg, self.B
        elu, s = Pre(act=ACT["elu"]), cfg.upsample_stride
        x = self._conv("init", pcm.reshape(B, -1, 1).contiguous())
        for i, lw in enumerate(E["layers"]):
            t = self._conv(f"c0_{i}", x, pre=elu)
            y = ops.conv1d(t, lw["c1"], pre=elu, res=x) if t.shape[1] else t.new_zeros(B, 0, x.shape[2])   # block(x) + x (seanet.py:61-66)
            x = self._conv(f"down_{i}", y, pre=elu)
        x = self._conv("final", x, pre=elu)
        n = self.npend + x.shape[1]
        run = n - n % s                                               # positions that complete frames
        if run == 0:                                                  # no frame: keep the positions, no transformer launch
            if x.shape[1]:
                self.pend[:, self.npend:n].copy_(x)
            self.npend = n
            self._conv("ds", None, pad_mode=1)                        # carries the down-sampler's history to the next parity slot
            ops.stream_advance(self.ctr, 0)
            return torch.zeros(B, cfg.nq, 0, device=x.device, dtype=torch.int64)
        z = torch.cat([self.pend[:, :self.npend], x], dim=1) if self.npend else x
        if n > run:
            self.pend[:, :n - run].copy_(z[:, run:])
        self.npend = n - run
        z = _stream_transformer(z[:, :run].contiguous(), E["tr"], cfg, self.k_ring, self.v_ring, self.ctr)
        lat = self._conv("ds", z, pad_mode=1)
        ops.stream_advance(self.ctr, run)
        return encode_codes(E, lat)

    def encode(self, pcm: torch.Tensor) -> torch.Tensor:
        n, hop = pcm.shape[-1], STREAM_PIECE_FRAMES * int(round(self.m.cfg.sample_rate / self.m.cfg.frame_rate))
        parts = [self._encode_piece(pcm[:, :, a:a + hop]) for a in range(0, max(n, 1), hop)] if n else [self._encode_piece(pcm)]
        return parts[0] if len(parts) == 1 else torch.cat(parts, dim=2)


GRAPH_SINGLE_FRAME = [True]      # single-frame decode steps through a captured CUDA graph (False: always eager)


class MimiStreamingDecoder:
    """mimi.py:278-320: keeps the codec's streaming state across calls.  The reference decodes frame by frame with ``decode_step``; since
    every step returns the matching slice of a one-shot decode, a block of frames is decoded here with a single ``decode_step``."""

    def __init__(self, mimi: Mimi) -> None:
        self._mimi = mimi
        self.reset()

    def reset(self) -> None:
        self._mimi.reset_state()

    def decode_frames(self, tokens: torch.Tensor) -> torch.Tensor:
        """tokens [B, C, T] or [C, T] -> waveform [B, 1, 1920 T] for these frames (continuing the stream)."""
        if tokens.dim() == 2:
            tokens = tokens[None]
        return self._mimi.decode_step(tokens)
