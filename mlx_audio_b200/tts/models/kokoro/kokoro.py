"""Kokoro-82M on H100: ``Model(config)`` / ``load_weights`` / ``__call__`` / ``generate`` with the
reference's signatures (tts/models/kokoro/kokoro.py:57-370) over our CUDA kernels.

GPU-first structure (not a translation of the MLX graph):
  * one device-resident weight set, weight-norm folded once at load (the reference recomputes
    g*v/||v|| every forward, istftnet.py:130) and rounded to the checkpoint's bf16 grid;
  * activations channels-last fp32; "concatenations" are channel-slice views of one buffer;
  * InstanceNorm/AdaIN statistics -> per-(batch,channel) scale/shift that the consuming conv applies
    in its prologue together with Snake / LeakyReLU; residuals, 1/sqrt(2), the 1/3 resblock average
    are conv epilogues -- every conv reads its input once and writes its output once;
  * all 49 AdaIN / AdaLayerNorm style projections are ONE batched GEMV per utterance;
  * the 6 BiLSTMs run as 8-CTA-cluster persistent recurrences (csrc/lstm.cu);
  * the alignment matrix of kokoro.py:148-170 is a device prefix sum + row gather (one host read of
    the frame count instead of one sync per phoneme).
"""
from __future__ import annotations

import functools
import math
import time
import weakref
from dataclasses import dataclass
from numbers import Number
from typing import Dict, Optional

import torch

from .... import ops
from ....ops import ACT, ConvW, Pre
from ..base import BaseModelArgs, GenerationResult, check_array_shape


def _fused_layers(fn):
    """Kokoro's single layers (text-encoder convs, asr_res, the LSTM input projections) take the fused conv kernel; see ops.FUSED_DISPATCH."""
    @functools.wraps(fn)
    def wrapped(*a, **k):
        with ops.fused_dispatch(True):
            return fn(*a, **k)
    return wrapped


@dataclass
class ModelConfig(BaseModelArgs):
    """Reference: kokoro.py:39-54."""
    istftnet: dict
    dim_in: int
    dropout: float
    hidden_dim: int
    max_conv_dim: int
    max_dur: int
    multispeaker: bool
    n_layer: int
    n_mels: int
    n_token: int
    style_dim: int
    text_encoder_kernel_size: int
    plbert: dict
    vocab: Dict[str, int] = None
    sample_rate: int = 24000


def _bf16(x: torch.Tensor) -> torch.Tensor:
    return x.to(torch.bfloat16).to(torch.float32)


def fold_weight_norm(v: torch.Tensor, g: torch.Tensor) -> torch.Tensor:
    """w = g * v / (||v|| + 1e-7) over all axes but 0 (istftnet.py:53-93), evaluated once in fp32 and
    rounded to bf16 -- the dtype in which the reference's bf16 checkpoint evaluates it every forward."""
    v32, g32 = v.float(), g.float()
    nrm = torch.sqrt((v32 * v32).sum(dim=tuple(range(1, v.dim())), keepdim=True))
    return _bf16(v32 / (nrm + 1e-7) * g32)


class _AdaSlots:
    """Collects every style->(gamma|beta) Linear so one GEMV serves the whole utterance."""

    def __init__(self):
        self.ws, self.bs, self.slices, self.off = [], [], {}, 0

    def add(self, name, w, b):
        n = w.shape[0]
        self.ws.append(w.float())
        self.bs.append(b.float())
        self.slices[name] = (self.off, n)
        self.off += n


class Model:
    """Drop-in for ``mlx_audio.tts.models.kokoro.Model`` (duck-typed protocol of utils.py:387-414)."""

    REPO_ID = "prince-canuma/Kokoro-82M"

    @dataclass
    class Output:
        audio: torch.Tensor
        pred_dur: Optional[torch.Tensor] = None

    def __init__(self, config: ModelConfig, repo_id: str = None, device="cuda"):
        self.config = config
        self.repo_id = repo_id
        self.vocab = config.vocab or {}
        self.device = torch.device(device)
        self.context_length = config.plbert["max_position_embeddings"]
        self._w = None
        self._pipelines = {}
        self.tap = None            # set to a dict to capture intermediates (parity tests)
        self.concurrent = True     # independent sub-graphs (text encoder, F0/N heads, source path, resblocks) on parallel streams
        self.use_graphs = True     # __call__ / generate replay cached CUDA graphs (synthesize_ids); False -> eager forward_ids
        self.max_graphs = 32
        self.share_graph_pool = True
        self._graphs, self._graph_pool, self._rng_state, self._warm_stream = {}, None, None, None
        self._stats_pool = None

    # ------------------------------------------------------------------ protocol
    @property
    def sample_rate(self):
        return self.config.sample_rate

    def eval(self):
        return self

    def parameters(self):
        return self._raw

    def sanitize(self, weights: dict) -> dict:
        """PyTorch-checkpoint -> reference parameter tree (kokoro.py:179-276, istftnet.py:999-1011)."""
        lstm_map = {"weight_ih_l0_reverse": "Wx_backward", "weight_hh_l0_reverse": "Wh_backward",
                    "bias_ih_l0_reverse": "bias_ih_backward", "bias_hh_l0_reverse": "bias_hh_backward",
                    "weight_ih_l0": "Wx_forward", "weight_hh_l0": "Wh_forward",
                    "bias_ih_l0": "bias_ih_forward", "bias_hh_l0": "bias_hh_forward"}
        out = {}
        for key, val in weights.items():
            if key.startswith("bert"):
                if "position_ids" in key:
                    continue
                out[key] = val
                continue
            base, _, leaf = key.rpartition(".")
            if leaf in lstm_map and (key.startswith("text_encoder") or key.startswith("predictor")):
                out[f"{base}.{lstm_map[leaf]}"] = val
            elif key.startswith("text_encoder") and leaf in ("gamma", "beta"):
                out[f"{base}.{'weight' if leaf == 'gamma' else 'bias'}"] = val
            elif "F0_proj.weight" in key or "N_proj.weight" in key:
                out[key] = val.transpose(1, 2)
            elif "noise_convs" in key and key.endswith(".weight"):
                out[key] = val.transpose(1, 2)
            elif "weight_v" in key:
                out[key] = val if check_array_shape(val) else val.transpose(1, 2)
            else:
                out[key] = val
        return out

    def load_weights(self, weights, strict: bool = True):
        """weights: list of (name, tensor) pairs or a dict, names = the reference's parameter tree."""
        P = dict(weights)
        self._raw = P
        self._prepare(P, strict)
        return self

    # ------------------------------------------------------------------ weight preparation
    def _cw(self, P, pre, *, groups=1, transpose_layout=False, bias=True) -> ConvW:
        w = fold_weight_norm(P[pre + ".weight_v"], P[pre + ".weight_g"])
        if transpose_layout:                       # ConvWeighted's `weight.T` branch (istftnet.py:159-166)
            w = w.permute(2, 1, 0)
        b = P.get(pre + ".bias") if bias else None
        return ops.pack_conv(w, b, groups, self.device)

    def _lin(self, P, pre, bias=True) -> ConvW:
        return ops.pack_linear(P[pre + ".weight"].float(), P.get(pre + ".bias") if bias else None, self.device)

    def _lstm(self, P, pre):
        wx = torch.cat([P[f"{pre}.Wx_forward"], P[f"{pre}.Wx_backward"]], 0).float()               # [2*4H, In]
        b = torch.cat([P[f"{pre}.bias_ih_forward"] + P[f"{pre}.bias_hh_forward"],
                       P[f"{pre}.bias_ih_backward"] + P[f"{pre}.bias_hh_backward"]], 0).float()
        wh = torch.stack([P[f"{pre}.Wh_forward"], P[f"{pre}.Wh_backward"]], 0).float().contiguous().to(self.device)
        return ops.pack_linear(wx, b, self.device), wh

    def _resblk1d(self, P, pre, ada, upsample=False):
        blk = {"conv1": self._cw(P, pre + ".conv1"), "conv2": self._cw(P, pre + ".conv2"), "up": upsample, "name": pre}
        ada.add(pre + ".norm1", P[pre + ".norm1.fc.weight"], P[pre + ".norm1.fc.bias"])
        ada.add(pre + ".norm2", P[pre + ".norm2.fc.weight"], P[pre + ".norm2.fc.bias"])
        if (pre + ".conv1x1.weight_v") in P:
            blk["sc"] = self._cw(P, pre + ".conv1x1", bias=False)
        if upsample:
            blk["pool"] = self._cw(P, pre + ".pool", groups=P[pre + ".pool.weight_v"].shape[0])
        return blk

    def _resblock1(self, P, pre, ada, k, dils):
        blk = {"k": k, "dils": dils, "name": pre, "c1": [], "c2": [], "a1": [], "a2": []}
        for j in range(3):
            blk["c1"].append(self._cw(P, f"{pre}.convs1.{j}"))
            blk["c2"].append(self._cw(P, f"{pre}.convs2.{j}"))
            ada.add(f"{pre}.adain1.{j}", P[f"{pre}.adain1.{j}.fc.weight"], P[f"{pre}.adain1.{j}.fc.bias"])
            ada.add(f"{pre}.adain2.{j}", P[f"{pre}.adain2.{j}.fc.weight"], P[f"{pre}.adain2.{j}.fc.bias"])
            for nm, lst in (("alpha1", "a1"), ("alpha2", "a2")):
                a = P[f"{pre}.{nm}.{j}"].float().reshape(-1).to(self.device)
                blk[lst].append((a.contiguous(), (1.0 / a).contiguous()))          # Snake: x + (1/a) sin^2(a x)
        return blk

    def _prepare(self, P, strict):
        cfg, dev = self.config, self.device
        W = {}
        ada = _AdaSlots()
        f = lambda t: t.float().to(dev).contiguous()
        # --- ALBERT (modules.py:434-645)
        B = "bert."
        W["word_emb"] = f(P[B + "embeddings.word_embeddings.weight"])
        W["pos_type"] = f(P[B + "embeddings.position_embeddings.weight"].float()
                          + P[B + "embeddings.token_type_embeddings.weight"][0].float()[None])
        W["emb_ln"] = (f(P[B + "embeddings.LayerNorm.weight"]), f(P[B + "embeddings.LayerNorm.bias"]))
        W["map_in"] = self._lin(P, B + "encoder.embedding_hidden_mapping_in")
        L = B + "encoder.albert_layer_groups.0.albert_layers.0."
        wqkv = torch.cat([P[L + f"attention.{n}.weight"].float() for n in ("query", "key", "value")], 0)
        bqkv = torch.cat([P[L + f"attention.{n}.bias"].float() for n in ("query", "key", "value")], 0)
        W["qkv"] = ops.pack_linear(wqkv, bqkv, dev)
        W["attn_out"] = self._lin(P, L + "attention.dense")
        W["attn_ln"] = (f(P[L + "attention.LayerNorm.weight"]), f(P[L + "attention.LayerNorm.bias"]))
        W["ffn"] = self._lin(P, L + "ffn")
        W["ffn_out"] = self._lin(P, L + "ffn_output")
        W["full_ln"] = (f(P[L + "full_layer_layer_norm.weight"]), f(P[L + "full_layer_layer_norm.bias"]))
        W["bert_encoder"] = self._lin(P, "bert_encoder")
        # --- prosody predictor (modules.py:288-411)
        W["dur_lstms"] = []
        for i in range(cfg.n_layer):
            W["dur_lstms"].append(self._lstm(P, f"predictor.text_encoder.lstms.{2 * i}"))
            ada.add(f"adaln.{i}", P[f"predictor.text_encoder.lstms.{2 * i + 1}.fc.weight"], P[f"predictor.text_encoder.lstms.{2 * i + 1}.fc.bias"])
        W["pred_lstm"] = self._lstm(P, "predictor.lstm")
        # duration head: Linear(512 -> max_dur = 50) -> sigmoid -> sum.  50 outputs miss the tensor-core kernels' Cout % 32 rule and the
        # CUDA-core tile kernel needs 170 us for it on the text side's critical path; zero-padded to 64 outputs it is one small GEMM, and
        # the padded columns (sigmoid(0) = 0.5) get weight 0 in the sum.
        dpad = -cfg.max_dur % 32
        dw, db = P["predictor.duration_proj.linear_layer.weight"].float(), P["predictor.duration_proj.linear_layer.bias"].float()
        W["dur_proj"] = ops.pack_linear(torch.cat([dw, dw.new_zeros(dpad, dw.shape[1])], 0), torch.cat([db, db.new_zeros(dpad)], 0), dev)
        W["dur_sum"] = ops.pack_linear(torch.cat([torch.ones(1, cfg.max_dur), torch.zeros(1, dpad)], 1), None, dev)
        W["shared"] = self._lstm(P, "predictor.shared")
        for name in ("F0", "N"):
            W[name] = [self._resblk1d(P, f"predictor.{name}.0", ada), self._resblk1d(P, f"predictor.{name}.1", ada, True),
                       self._resblk1d(P, f"predictor.{name}.2", ada)]
            W[name + "_proj"] = ops.pack_conv(P[f"predictor.{name}_proj.weight"].float(), P[f"predictor.{name}_proj.bias"], 1, dev)
        # --- text encoder (modules.py:21-68)
        W["te_emb"] = f(P["text_encoder.embedding.weight"])
        W["te_cnn"] = [(self._cw(P, f"text_encoder.cnn.{i}.0"), f(P[f"text_encoder.cnn.{i}.1.weight"]), f(P[f"text_encoder.cnn.{i}.1.bias"]))
                       for i in range(cfg.n_layer)]
        W["te_lstm"] = self._lstm(P, "text_encoder.lstm")
        # --- decoder (istftnet.py:936-997)
        W["encode"] = self._resblk1d(P, "decoder.encode", ada)
        W["decode"] = [self._resblk1d(P, f"decoder.decode.{i}", ada, (f"decoder.decode.{i}.pool.weight_v") in P) for i in range(4)]
        W["F0_conv"] = self._cw(P, "decoder.F0_conv")
        W["N_conv"] = self._cw(P, "decoder.N_conv")
        W["asr_res"] = self._cw(P, "decoder.asr_res.0")
        # --- generator (istftnet.py:725-835)
        ist = cfg.istftnet
        G = "decoder.generator"
        W["src_lin"] = (f(P[G + ".m_source.l_linear.weight"]).reshape(-1), f(P[G + ".m_source.l_linear.bias"]).reshape(-1))
        rates, ks, rk, rd = ist["upsample_rates"], ist["upsample_kernel_sizes"], ist["resblock_kernel_sizes"], ist["resblock_dilation_sizes"]
        W["ups"], W["noise_convs"], W["noise_res"], W["resblocks"] = [], [], [], []
        for i in range(len(rates)):
            W["ups"].append(self._cw(P, f"{G}.ups.{i}", transpose_layout=True))
            W["noise_convs"].append(ops.pack_conv(P[f"{G}.noise_convs.{i}.weight"].float(), P[f"{G}.noise_convs.{i}.bias"], 1, dev))
            W["noise_res"].append(self._resblock1(P, f"{G}.noise_res.{i}", ada, 7 if i + 1 < len(rates) else 11, (1, 3, 5)))
            for j in range(len(rk)):
                W["resblocks"].append(self._resblock1(P, f"{G}.resblocks.{i * len(rk) + j}", ada, rk[j], tuple(rd[j])))
        # conv_post (128 -> 22, k7, the last layer before the iSTFT head, on the critical path): Cout padded 22 -> 32 with zero filters so
        # that it runs on the tensor-core conv instead of the CUDA-core tile (150 us -> ~30 us); the head reads 22 of the 32 columns.
        wp = fold_weight_norm(P[G + ".conv_post.weight_v"], P[G + ".conv_post.weight_g"])
        bp = P[G + ".conv_post.bias"].float()
        n_post = wp.shape[0]
        if n_post % 32:
            padn = -(-n_post // 32) * 32 - n_post
            wp = torch.cat([wp, torch.zeros(padn, *wp.shape[1:], dtype=wp.dtype)], 0)
            bp = torch.cat([bp, torch.zeros(padn, dtype=bp.dtype)], 0)
        W["conv_post"] = ops.pack_conv(wp, bp, 1, self.device)
        W["n_post"] = n_post
        # --- one batched style projection
        W["ada_all"] = ops.pack_linear(torch.cat(ada.ws, 0), torch.cat(ada.bs, 0), dev)
        self._ada_slices = ada.slices
        self._ada_pred = [k for k in ada.slices if k.startswith("adaln.") or k.startswith("predictor.")]
        self._w = W

    def _tap(self, name, t):
        if self.tap is not None:
            self.tap[name] = t.detach().clone()

    # ------------------------------------------------------------------ building blocks
    def _gb(self, name):
        off, n = self._ada_slices[name]
        src = self._gb_pred if name in self._pred_set else self._gb_dec
        return src[:, off:off + n]

    def _lstm_run(self, x2d, lw, out=None):
        xproj = ops.linear(x2d, lw[0])                           # [T, 2*4H]
        return ops.lstm_bidir(xproj[None], lw[1], out=None if out is None else out[None])[0]

    def _adain_resblk1d(self, x, blk, out=None):
        """AdainResBlk1d (istftnet.py:853-933) on x [1,L,Cin] -> [1,L or 2L,Cout]."""
        s1, h1 = ops.adain_coeffs(x, self._gb(blk["name"] + ".norm1").contiguous())
        pre1 = Pre(s1, h1, ACT["lrelu"], 0.2)
        L = x.shape[1]
        if blk["up"]:
            r = ops.conv1d(x, blk["pool"], stride=2, pad_left=1, lout=2 * L, pre=pre1, transpose=True)
            r = ops.conv1d(r, blk["conv1"], pad_left=1)
        else:
            r = ops.conv1d(x, blk["conv1"], pad_left=1, pre=pre1)
        s2, h2 = ops.adain_coeffs(r, self._gb(blk["name"] + ".norm2").contiguous())
        sc = ops.conv1d(x, blk["sc"]) if "sc" in blk else x
        return ops.conv1d(r, blk["conv2"], pad_left=1, pre=Pre(s2, h2, ACT["lrelu"], 0.2), res=sc,
                          res_div=2 if blk["up"] else 1, out_scale=1.0 / math.sqrt(2.0), out=out)

    def _adain_resblock1(self, x, blk, out=None, out_scale=1.0, accumulate=False, defer_last=False):
        """AdaINResBlock1 (istftnet.py:341-396) on x [1,L,C].  ``defer_last`` returns a closure issuing the final conv
        (the one that writes / accumulates into ``out``) so parallel branches can serialise only that step."""
        k = blk["k"]
        for j, d in enumerate(blk["dils"]):
            s1, h1 = ops.adain_coeffs(x, self._gb(f"{blk['name']}.adain1.{j}").contiguous())
            a, ia = blk["a1"][j]
            xt = ops.conv1d(x, blk["c1"][j], dilation=d, pad_left=(k * d - d) // 2, pre=Pre(s1, h1, ACT["snake"], 0.0, a, ia))
            s2, h2 = ops.adain_coeffs(xt, self._gb(f"{blk['name']}.adain2.{j}").contiguous())
            a, ia = blk["a2"][j]
            last = j == len(blk["dils"]) - 1
            if last and defer_last:
                def final(xt=xt, s2=s2, h2=h2, a=a, ia=ia, x=x, j=j):
                    return ops.conv1d(xt, blk["c2"][j], pad_left=(k - 1) // 2, pre=Pre(s2, h2, ACT["snake"], 0.0, a, ia), res=x,
                                      out=out, out_scale=out_scale, accumulate=accumulate)
                return final
            if last:
                x = ops.conv1d(xt, blk["c2"][j], pad_left=(k - 1) // 2, pre=Pre(s2, h2, ACT["snake"], 0.0, a, ia), res=x,
                               out=out, out_scale=out_scale, accumulate=accumulate)
            else:
                x = ops.conv1d(xt, blk["c2"][j], pad_left=(k - 1) // 2, pre=Pre(s2, h2, ACT["snake"], 0.0, a, ia), res=x)
        return x


    # ------------------------------------------------------------------ fused acoustic side (one launch per layer GROUP)
    # Every dense conv below is ONE launch of csrc/conv_fused.cu that also applies the AdaIN + Snake / LeakyReLU in front of it (from the
    # (sum, sumsq) its producer accumulated) and accumulates the (sum, sumsq) of its own output for the next AdaIN.  Layers that are
    # independent of each other -- the F0 and N heads, a block's conv1 and its 1x1 shortcut, the three parallel AdaINResBlock1 branches of
    # a generator stage (kernel sizes 3 / 7 / 11) -- share one persistent grid.
    def _stats(self, C: int) -> torch.Tensor:
        if self._stats_pool is not None:                               # buffers reserved up front for a concurrent branch
            t = self._stats_pool.pop(0)
            assert t.shape[1] == C
            return t
        n = 2 * ops.STAT_BINS * C
        off = self._arena_off
        self._arena_off += n
        assert self._arena_off <= self._arena.numel()
        return self._arena[off:off + n].view(1, C, 2, ops.STAT_BINS)

    def _resblk1d_group(self, xs, sxs, blks, outs=None, sos=None):
        """AdainResBlk1d (istftnet.py:853-933) for n parallel blocks of identical structure: xs[i] [1,L,Cin] with statistics sxs[i]
        -> outs[i] [1, L or 2L, Cout] (statistics of the outputs added to sos[i] when given)."""
        n = len(blks)
        outs = outs or [None] * n
        sos = sos or [None] * n
        up = blks[0]["up"]
        L = xs[0].shape[1]
        lrelu = ACT["lrelu"]
        s1 = [self._stats(b["conv1"].cout) for b in blks]
        first = []
        if up:
            rs = []
            for x, sx, b in zip(xs, sxs, blks):
                sc, sh = ops.coeffs_from_stats(sx, L, self._gb(b["name"] + ".norm1"))
                cpad = -(-x.shape[2] // 4) * 4                         # row stride padded to 16 bytes: the fused conv loads float4 chunks
                r = torch.empty(1, 2 * L, cpad, device=x.device, dtype=torch.float32)[:, :, :x.shape[2]]
                rs.append(ops.conv1d(x, b["pool"], stride=2, pad_left=1, lout=2 * L, pre=Pre(sc, sh, lrelu, 0.2), transpose=True, out=r))
            first = [ops.FusedProblem(r, b["conv1"], pad_left=1, stats_out=st) for r, b, st in zip(rs, blks, s1)]
        else:
            first = [ops.FusedProblem(x, b["conv1"], pad_left=1, pre=ops.PreStats(sx, self._gb(b["name"] + ".norm1"), 1e-5, lrelu, 0.2), stats_out=st)
                     for x, sx, b, st in zip(xs, sxs, blks, s1)]
        shortcut = [ops.FusedProblem(x, b["sc"]) for x, b in zip(xs, blks) if "sc" in b]
        res = ops.conv_fused(first + shortcut) if len(first) + len(shortcut) <= 4 else ops.conv_fused(first) + ops.conv_fused(shortcut)
        r1 = res[:n]
        scs = res[n:] if shortcut else xs
        second = [ops.FusedProblem(r, b["conv2"], pad_left=1, pre=ops.PreStats(st, self._gb(b["name"] + ".norm2"), 1e-5, lrelu, 0.2), res=sc,
                                   res_div=2 if up else 1, out_scale=1.0 / math.sqrt(2.0), out=o, stats_out=so)
                  for r, b, st, sc, o, so in zip(r1, blks, s1, scs, outs, sos)]
        return ops.conv_fused(second)

    def _resblock1_group(self, xs, sxs, blks, outs=None):
        """AdaINResBlock1 (istftnet.py:341-396) for n parallel blocks (different kernel sizes) -> n outputs."""
        n = len(blks)
        outs = outs or [None] * n
        cur, scur = list(xs), list(sxs)
        for j in range(3):
            last = j == 2
            st1 = [self._stats(b["c1"][j].cout) for b in blks]
            c1 = [ops.FusedProblem(x, b["c1"][j], dilation=b["dils"][j], pad_left=(b["k"] * b["dils"][j] - b["dils"][j]) // 2,
                                   pre=ops.PreStats(sx, self._gb(f"{b['name']}.adain1.{j}"), 1e-5, ACT["snake"], 0.0, *b["a1"][j]), stats_out=st)
                  for x, sx, b, st in zip(cur, scur, blks, st1)]
            xt = ops.conv_fused(c1)
            snew = [None if last else self._stats(b["c2"][j].cout) for b in blks]
            c2 = [ops.FusedProblem(t, b["c2"][j], pad_left=(b["k"] - 1) // 2,
                                   pre=ops.PreStats(st, self._gb(f"{b['name']}.adain2.{j}"), 1e-5, ACT["snake"], 0.0, *b["a2"][j]), res=x,
                                   out=outs[i] if last else None, stats_out=sn)
                  for i, (t, st, x, b, sn) in enumerate(zip(xt, st1, cur, blks, snew))]
            cur, scur = ops.conv_fused(c2), snew
        return cur

    @torch.no_grad()
    def _acoustic_side_fused(self, st, F: int, noise=None, f0n_override=None):
        W, cfg, dev = self._w, self.config, self.device
        self._bind(st)
        hd = cfg.hidden_dim
        par = self.concurrent
        X, t_en = st["X"], st["t_en"]
        idx = st["idx"][:F]
        self._arena = torch.zeros(1 << 19, device=dev, dtype=torch.int64)            # every (sum, sumsq) accumulator of the utterance: one memset
        self._arena_off = 0
        # ---- F0 / N prediction: the two heads run as 2-problem groups
        en = ops.gather_rows(X, idx)                                   # [F,640]  == d^T @ aln
        xs = self._lstm_run(en, W["shared"])[None]                     # [1,F,512]
        sxs = self._stats(xs.shape[2])
        ops.channel_stats(xs, sxs)
        F0N = torch.empty(2, 2 * F, 1, device=dev, dtype=torch.float32)
        hcur, scur = [xs, xs], [sxs, sxs]
        for bi in range(3):
            blks = [W["F0"][bi], W["N"][bi]]
            sos = [self._stats(b["conv2"].cout) for b in blks] if bi < 2 else None
            hcur = self._resblk1d_group(hcur, scur, blks, sos=sos)
            scur = sos
        ops.conv1d(hcur[0], W["F0_proj"], out=F0N[0:1])
        ops.conv1d(hcur[1], W["N_proj"], out=F0N[1:2])
        if f0n_override is not None:
            F0N[0, :, 0].copy_(torch.as_tensor(f0n_override[0]).to(device=dev, dtype=torch.float32).reshape(-1))
            F0N[1, :, 0].copy_(torch.as_tensor(f0n_override[1]).to(device=dev, dtype=torch.float32).reshape(-1))
        f0_curve, n_curve = F0N[0:1], F0N[1:2]                         # [1,2F,1]
        self._tap("en", en)
        self._tap("F0", f0_curve)
        self._tap("N", n_curve)
        # ---- harmonic-source path: its own branch (concurrent with the decoder blocks)
        ist = cfg.istftnet
        rates, ks = ist["upsample_rates"], ist["upsample_kernel_sizes"]
        nk = len(ist["resblock_kernel_sizes"])
        n_har = 120 * F + 1
        xsrcs = []
        for i in range(len(rates)):
            sf0 = math.prod(rates[i + 1:]) if i + 1 < len(rates) else 1
            Li = (n_har + 2 * ((sf0 + 1) // 2) - (2 * sf0 - 1) - 1) // sf0 + 1 if sf0 > 1 else n_har
            xsrcs.append(torch.empty(1, Li, W["noise_convs"][i].cout, device=dev, dtype=torch.float32))
        src_stats = [self._stats(W["noise_convs"][i].cout) for i in range(len(rates))]
        src_arena = [[self._stats(W["noise_convs"][i].cout) for _ in range(5)] for i in range(len(rates))]   # reserved up front: the branch runs concurrently

        def source_branch():
            har = ops.kokoro_source(f0_curve.reshape(1, 2 * F), noise, *W["src_lin"])      # [1,120F+1,22]
            self._tap("har", har)
            ts = []
            for i in range(len(rates)):
                if i + 1 < len(rates):
                    sf0 = math.prod(rates[i + 1:])
                    t = ops.kokoro_source_conv(har, W["noise_convs"][i], stride=sf0, pad_left=(sf0 + 1) // 2)
                else:
                    t = ops.kokoro_source_conv(har, W["noise_convs"][i])
                ops.channel_stats(t, src_stats[i])
                ts.append(t)
            # both noise-resblock chains in shared launches (one problem per up-sampling stage); _resblock1_group takes a statistics
            # buffer for each problem in turn, so the reserved buffers are interleaved by stage
            pool, self._stats_pool = self._stats_pool, [s for group in zip(*src_arena) for s in group]
            try:
                self._resblock1_group(ts, src_stats, W["noise_res"], outs=xsrcs)
            finally:
                self._stats_pool = pool

        if par:
            side_src = ops.fork(dev, 1)
            with torch.cuda.stream(side_src[0]):
                source_branch()
        # ---- decoder
        b514 = torch.empty(1, F, hd + 4, device=dev, dtype=torch.float32)[:, :, :hd + 2]     # row stride padded to a multiple of 4 floats
        ops.gather_rows(t_en, idx, out=b514[0, :, :hd])                # asr = t_en @ aln
        ops.conv1d(f0_curve, W["F0_conv"], stride=2, pad_left=1, out=b514[:, :, hd:hd + 1])
        ops.conv1d(n_curve, W["N_conv"], stride=2, pad_left=1, out=b514[:, :, hd + 1:hd + 2])
        bufs = [torch.empty(1, F, 1024 + 64 + 4, device=dev, dtype=torch.float32)[:, :, :1024 + 64 + 2] for _ in range(2)]
        ops.conv1d(b514[:, :, :hd], W["asr_res"], out=bufs[0][:, :, 1024:1088])
        ops.copy2d(b514[0, :, hd:], bufs[0][0, :, 1088:])
        ops.copy2d(bufs[0][0, :, 1024:], bufs[1][0, :, 1024:])
        s514 = self._stats(hd + 2)
        ops.channel_stats(b514, s514)
        nblk = len(W["decode"])
        sbuf = [self._stats(1024 + 64 + 2) for _ in range(nblk)]       # statistics of each decode block's input [conv out | asr_res | F0 | N]
        ops.channel_stats(bufs[0][:, :, 1024:], [sb[:, 1024:] for sb in sbuf])      # the side channels are the same for every block
        self._resblk1d_group([b514], [s514], [W["encode"]], outs=[bufs[0][:, :, :1024]], sos=[sbuf[0][:, :1024]])
        self._tap("dec_encode", bufs[0][:, :, :1024])
        cur = 0
        x = None
        for i, blk in enumerate(W["decode"]):
            if blk["up"]:
                x = self._resblk1d_group([bufs[cur]], [sbuf[i]], [blk])[0]              # [1,2F,512]
            else:
                self._resblk1d_group([bufs[cur]], [sbuf[i]], [blk], outs=[bufs[1 - cur][:, :, :1024]], sos=[sbuf[i + 1][:, :1024]])
                cur = 1 - cur
        self._tap("dec_out", x)
        if par:
            ops.join(dev, side_src)
        else:
            source_branch()
        # ---- generator: per stage one polyphase transposed conv + six grouped launches (3 dilations x (c1, c2)) of nk problems each
        x_add, in_scale = (), 1.0
        for i, (u, kk) in enumerate(zip(rates, ks)):
            last = i == len(rates) - 1
            xsrc = xsrcs[i]
            L = x.shape[1]
            lout = (L - 1) * u + kk - 2 * ((kk - u) // 2)
            cout = W["ups"][i].cout
            sy = self._stats(cout)
            pre = Pre(act=ACT["lrelu"], p0=0.1)
            if last:                                                   # "ReflectionPad1d((1,0))" is a zero pad on the left
                y = torch.empty(1, lout + 1, cout, device=dev, dtype=torch.float32)
                ops.copy2d(xsrc[0, :1], y[0, :1])
                ops.channel_stats(y[:, :1], sy)                        # row 0 never passes through the conv's epilogue
                ops.conv_fused(ops.FusedProblem(x, W["ups"][i], stride=u, pad_left=(kk - u) // 2, pre=pre, transpose=True, res=xsrc[:, 1:],
                                                out=y[:, 1:], x_add=x_add, in_scale=in_scale, stats_out=sy))
            else:
                y = ops.conv_fused(ops.FusedProblem(x, W["ups"][i], stride=u, pad_left=(kk - u) // 2, pre=pre, transpose=True, res=xsrc,
                                                    x_add=x_add, in_scale=in_scale, stats_out=sy))[0]
            blks = [W["resblocks"][i * nk + j] for j in range(nk)]
            outs = self._resblock1_group([y] * nk, [sy] * nk, blks)
            x, x_add, in_scale = outs[0], tuple(outs[1:]), 1.0 / nk    # the average of the nk branches is folded into the consumer's load
            if self.tap is not None:
                self._tap(f"gen_stage{i}", sum(outs) / nk)
        xpost = ops.conv_fused(ops.FusedProblem(x, W["conv_post"], pad_left=3, pre=Pre(act=ACT["lrelu"], p0=0.01), x_add=x_add,
                                                in_scale=in_scale))[0][:, :, :W["n_post"]]
        self._tap("xpost", xpost)
        return ops.kokoro_istft_head(xpost)[0]

    # ------------------------------------------------------------------ forward
    # The utterance has exactly one data-dependent size: F = sum(pred_dur).  Everything in front of it (`_text_side`: ALBERT, text
    # encoder, duration encoder, duration head, alignment indices) depends on T only; everything behind it (`_acoustic_side`: F0 / N
    # heads, decoder, generator, iSTFT head) on (T, F).  `forward_ids` runs both eagerly; `synthesize_ids` replays one CUDA graph per
    # side with a single host read of F in between (the reference syncs once per phoneme, kokoro.py:148-152).
    @torch.no_grad()
    @_fused_layers
    def _text_side(self, ids, ref_s, speed: float = 1.0, pred_dur=None):
        """ids int64 [T] + style [1,256] (device) -> state dict: X [T,640] = [d_en | style], t_en [T,512], pred_dur, alignment
        indices (first `total` valid), total (device int64 [1]), the two style-projection rows."""
        W, cfg, dev = self._w, self.config, self.device
        T = ids.shape[0]
        s_dec, s_pred = ref_s[:, :128].contiguous(), ref_s[:, 128:].contiguous()
        st = {"T": T}
        st["gb_pred"] = ops.linear(s_pred, W["ada_all"])              # [1, sum 2C]  (all style projections at once)
        st["gb_dec"] = ops.linear(s_dec, W["ada_all"])
        self._bind(st)
        hd = cfg.hidden_dim
        par = self.concurrent
        # ---- text encoder: independent of the ALBERT / duration chain -> its own branch (parallel graph path)
        t_en = torch.empty(T, hd, device=dev, dtype=torch.float32)

        def text_branch():
            te = ops.gather_rows(W["te_emb"], ids)[None]
            k = cfg.text_encoder_kernel_size
            for cw, lw, lb in W["te_cnn"]:
                te = ops.conv1d(te, cw, pad_left=(k - 1) // 2)
                te = ops.layernorm(te, lw, lb, eps=1e-5, post_act=ACT["lrelu"], post_p0=0.2)
            self._lstm_run(te[0], W["te_lstm"], out=t_en)

        # ---- ALBERT
        e = ops.gather_rows(W["word_emb"], ids)
        nh = cfg.plbert["num_attention_heads"]
        hs = cfg.plbert["hidden_size"]
        scale = 1.0 / math.sqrt(hs // nh)
        if self._albert_planes(T):
            # every layer in one persistent launch (csrc/albert.cu); bit-identical to the branch below
            _, ep = ops.layernorm(e, *W["emb_ln"], eps=1e-12, res=W["pos_type"][:T], planes=True)
            h, hp = ops.linear(ep, W["map_in"], planes=True)
            ops.albert_encoder(h, hp, cfg.plbert["num_hidden_layers"], W["qkv"], W["attn_out"], W["ffn"], W["ffn_out"], W["attn_ln"],
                               W["full_ln"], heads=nh, scale=scale, eps=1e-12)
            h = h[0]
        else:
            # The GEMMs stay on conv_tc like the chain's: above 256 rows the fused kernel would take them and split K across CTAs,
            # which sums in a different order.
            with ops.fused_dispatch(False):
                e = ops.layernorm(e, *W["emb_ln"], eps=1e-12, res=W["pos_type"][:T])
                h = ops.linear(e, W["map_in"])
                for _ in range(cfg.plbert["num_hidden_layers"]):
                    qkv = ops.linear(h, W["qkv"])[None]                       # [1,T,3*hs]
                    ctx = ops.attention(qkv[:, :, :hs], qkv[:, :, hs:2 * hs], qkv[:, :, 2 * hs:], n_heads=nh, scale=scale)[0]
                    a = ops.linear(ctx, W["attn_out"], res=h)
                    a = ops.layernorm(a, *W["attn_ln"], eps=1e-12)
                    f1 = ops.linear(a, W["ffn"], post_act=ACT["gelu"])
                    f2 = ops.linear(f1, W["ffn_out"], res=a)
                    h = ops.layernorm(f2, *W["full_ln"], eps=1e-12)
        self._tap("bert", h)
        if par:
            side_text = ops.fork(dev, 1)
            with torch.cuda.stream(side_text[0]):
                text_branch()
        # ---- duration encoder: X640 = [d_en | style]
        stl = cfg.style_dim
        X = torch.empty(T, hd + stl, device=dev, dtype=torch.float32)
        ops.linear(h, W["bert_encoder"], out=X[:, :hd])
        ops.copy2d(s_pred.expand(T, stl), X[:, hd:])
        for i in range(cfg.n_layer):
            o = self._lstm_run(X, W["dur_lstms"][i])
            ops.layernorm(o, eps=1e-5, ada=self._gb(f"adaln.{i}").reshape(-1).contiguous(), out=X[:, :hd])
        xl = self._lstm_run(X, W["pred_lstm"])
        dsig = ops.linear(xl, W["dur_proj"], post_act=ACT["sigmoid"])
        dsum = ops.linear(dsig, W["dur_sum"]).reshape(-1).contiguous()
        self._tap("d", X)
        self._tap("dur", dsum)
        max_frames = 100 * T
        if pred_dur is not None:
            pred, idx, total = ops.durations_to_index(pred_dur, max_frames)
        else:
            pred, idx, total = ops.durations_to_index(dsum, max_frames, float(speed))
        if par:
            ops.join(dev, side_text)
        else:
            text_branch()
        self._tap("t_en", t_en)
        st.update(X=X, t_en=t_en, pred=pred, idx=idx, total=total)
        return st

    def _albert_planes(self, T: int) -> bool:
        """ALBERT runs as one persistent kernel (ops.albert_encoder) when every GEMM takes the tensor-core path at T rows and the
        attention the tensor-core kernel (64-wide heads, 64 to 512 keys); otherwise (short or long utterances, B2A_TC=off,
        B2A_ATTN=cuda) as separate ops."""
        W, pb = self._w, self.config.plbert
        return (64 <= T <= 512 and ops.ATTN_MODE[0] == "tc" and pb["hidden_size"] == 64 * pb["num_attention_heads"]
                and pb["hidden_size"] % 64 == 0 and W["map_in"].cin % 64 == 0
                and all(ops.emit_tc_eligible(W[k], T) and W[k].w_tc_lo is None for k in ("map_in", "qkv", "attn_out", "ffn", "ffn_out")))

    def _bind(self, st):
        """Point the style-projection lookups (`_gb`) at this utterance's rows."""
        self._pred_set = set(self._ada_pred)
        self._gb_pred, self._gb_dec = st["gb_pred"], st["gb_dec"]

    @torch.no_grad()
    @_fused_layers
    def _acoustic_side(self, st, F: int, noise=None, f0n_override=None):
        """State of `_text_side` + the frame count -> waveform [600 F] samples."""
        if ops.FUSED[0] and ops.TC_MODE[0] != "off":
            return self._acoustic_side_fused(st, F, noise, f0n_override)
        W, cfg, dev = self._w, self.config, self.device
        self._bind(st)
        hd = cfg.hidden_dim
        par = self.concurrent
        X, t_en = st["X"], st["t_en"]
        idx = st["idx"][:F]
        # ---- F0 / N prediction
        en = ops.gather_rows(X, idx)                                   # [F,640]  == d^T @ aln
        xs = self._lstm_run(en, W["shared"])[None]                     # [1,F,512]
        F0N = torch.empty(2, 2 * F, 1, device=dev, dtype=torch.float32)

        def head(n_i, name):
            hcur = xs
            for blk in W[name]:
                hcur = self._adain_resblk1d(hcur, blk)
            ops.conv1d(hcur, W[name + "_proj"], out=F0N[n_i:n_i + 1])

        if par:
            side = ops.fork(dev, 1)
            with torch.cuda.stream(side[0]):
                head(1, "N")
            head(0, "F0")
            ops.join(dev, side)
        else:
            head(0, "F0")
            head(1, "N")
        if f0n_override is not None:
            F0N[0, :, 0].copy_(torch.as_tensor(f0n_override[0]).to(device=dev, dtype=torch.float32).reshape(-1))
            F0N[1, :, 0].copy_(torch.as_tensor(f0n_override[1]).to(device=dev, dtype=torch.float32).reshape(-1))
        f0_curve, n_curve = F0N[0:1], F0N[1:2]                         # [1,2F,1]
        self._tap("en", en)
        self._tap("F0", f0_curve)
        self._tap("N", n_curve)
        # ---- harmonic-source path (depends on the F0 curve only): source -> STFT -> noise convs -> noise resblocks, run as a
        #      branch concurrent with the decoder blocks
        ist = cfg.istftnet
        rates, ks = ist["upsample_rates"], ist["upsample_kernel_sizes"]
        nk = len(ist["resblock_kernel_sizes"])
        n_har = 120 * F + 1
        xsrcs, Lh = [], n_har
        for i in range(len(rates)):
            sf0 = math.prod(rates[i + 1:]) if i + 1 < len(rates) else 1
            Li = (n_har + 2 * ((sf0 + 1) // 2) - (2 * sf0 - 1) - 1) // sf0 + 1 if sf0 > 1 else n_har
            xsrcs.append(torch.empty(1, Li, W["noise_convs"][i].cout, device=dev, dtype=torch.float32))
        del Lh

        def source_branch():
            har = ops.kokoro_source(f0_curve.reshape(1, 2 * F), noise, *W["src_lin"])      # [1,120F+1,22]
            self._tap("har", har)
            for i in range(len(rates)):
                if i + 1 < len(rates):
                    sf0 = math.prod(rates[i + 1:])
                    t = ops.conv1d(har, W["noise_convs"][i], stride=sf0, pad_left=(sf0 + 1) // 2)
                else:
                    t = ops.conv1d(har, W["noise_convs"][i])
                self._adain_resblock1(t, W["noise_res"][i], out=xsrcs[i])

        if par:
            side_src = ops.fork(dev, 1)
            with torch.cuda.stream(side_src[0]):
                source_branch()
        # ---- decoder
        b514 = torch.empty(1, F, hd + 4, device=dev, dtype=torch.float32)[:, :, :hd + 2]     # row stride padded to a multiple of 4 floats
        ops.gather_rows(t_en, idx, out=b514[0, :, :hd])                # asr = t_en @ aln
        ops.conv1d(f0_curve, W["F0_conv"], stride=2, pad_left=1, out=b514[:, :, hd:hd + 1])
        ops.conv1d(n_curve, W["N_conv"], stride=2, pad_left=1, out=b514[:, :, hd + 1:hd + 2])
        bufs = [torch.empty(1, F, 1024 + 64 + 4, device=dev, dtype=torch.float32)[:, :, :1024 + 64 + 2] for _ in range(2)]
        ops.conv1d(b514[:, :, :hd], W["asr_res"], out=bufs[0][:, :, 1024:1088])
        ops.copy2d(b514[0, :, hd:], bufs[0][0, :, 1088:])
        ops.copy2d(bufs[0][0, :, 1024:], bufs[1][0, :, 1024:])
        self._adain_resblk1d(b514, W["encode"], out=bufs[0][:, :, :1024])
        self._tap("dec_encode", bufs[0][:, :, :1024])
        cur = 0
        x = None
        for i, blk in enumerate(W["decode"]):
            if blk["up"]:
                x = self._adain_resblk1d(bufs[cur], blk)              # [1,2F,512]
            else:
                self._adain_resblk1d(bufs[cur], blk, out=bufs[1 - cur][:, :, :1024])
                cur = 1 - cur
        self._tap("dec_out", x)
        if par:
            ops.join(dev, side_src)
        else:
            source_branch()
        # ---- generator
        for i, (u, kk) in enumerate(zip(rates, ks)):
            last = i == len(rates) - 1
            xsrc = xsrcs[i]
            L = x.shape[1]
            lout = (L - 1) * u + kk - 2 * ((kk - u) // 2)
            cout = W["ups"][i].cout
            if last:                                                   # "ReflectionPad1d((1,0))" is a zero pad on the left
                y = torch.empty(1, lout + 1, cout, device=dev, dtype=torch.float32)
                ops.copy2d(xsrc[0, :1], y[0, :1])
                ops.conv1d(x, W["ups"][i], stride=u, pad_left=(kk - u) // 2, pre=Pre(act=ACT["lrelu"], p0=0.1), transpose=True,
                           res=xsrc[:, 1:], out=y[:, 1:])
            else:
                y = ops.conv1d(x, W["ups"][i], stride=u, pad_left=(kk - u) // 2, pre=Pre(act=ACT["lrelu"], p0=0.1), transpose=True, res=xsrc)
            acc = torch.empty_like(y)
            if par:                                                    # the nk resblocks read the same y: parallel branches; only the
                sides = ops.fork(dev, nk - 1)                          # final accumulate-into-acc convs are serialised after the join
                finals = [None] * nk
                for j in range(1, nk):
                    with torch.cuda.stream(sides[j - 1]):
                        finals[j] = self._adain_resblock1(y, W["resblocks"][i * nk + j], out=acc, out_scale=1.0 / nk, accumulate=True,
                                                          defer_last=True)
                finals[0] = self._adain_resblock1(y, W["resblocks"][i * nk], out=acc, out_scale=1.0 / nk, accumulate=False, defer_last=True)
                ops.join(dev, sides)
                for fn in finals:
                    fn()
            else:
                for j in range(nk):
                    self._adain_resblock1(y, W["resblocks"][i * nk + j], out=acc, out_scale=1.0 / nk, accumulate=j > 0)
            x = acc
            self._tap(f"gen_stage{i}", x)
        xpost = ops.conv1d(x, W["conv_post"], pad_left=3, pre=Pre(act=ACT["lrelu"], p0=0.01))[:, :, :W["n_post"]]
        self._tap("xpost", xpost)
        audio = ops.kokoro_istft_head(xpost)[0]
        return audio


    @torch.no_grad()
    def forward_ids(self, input_ids, ref_s, speed: float = 1.0, *, noise=None, pred_dur=None, n_frames: Optional[int] = None,
                    f0n_override=None):
        """Token ids (BOS/EOS 0 included) + style [1,256] -> (audio [samples], pred_dur int64 [T]), launched eagerly.

        ``noise`` [1, 600F, 9] injects the SineGen Gaussian (istftnet.py:649); None -> noiseless source (`synthesize_ids` draws
        Philox noise on the device).  ``pred_dur`` overrides the duration head.  ``n_frames``: the caller already knows
        sum(pred_dur) -> no host sync.  ``f0n_override`` = (F0 [2F], N [2F]) replaces the predicted curves (parity tests: the
        hn-NSF phase integrates F0 over the whole utterance x300, so decoder parity is checked on identical curves; see DESIGN.md).
        """
        if self._w is None:
            raise RuntimeError("Kokoro: load_weights() has not been called")
        dev = self.device
        ids = torch.as_tensor(input_ids, dtype=torch.int64, device=dev).reshape(-1).contiguous()
        assert ids.shape[0] <= self.context_length, (ids.shape[0], self.context_length)
        ref_s = ref_s.to(device=dev, dtype=torch.float32).reshape(1, -1).contiguous()
        pd = None if pred_dur is None else torch.as_tensor(pred_dur, dtype=torch.int64, device=dev).contiguous()
        st = self._text_side(ids, ref_s, speed, pd)
        F = int(st["total"].item()) if n_frames is None else int(n_frames)   # the one host sync of the utterance
        if F <= 0:
            return torch.zeros(1, device=dev), st["pred"]
        return self._acoustic_side(st, F, noise, f0n_override), st["pred"]

    # ------------------------------------------------------------------ CUDA-graph path (what __call__ / generate use)
    def seed(self, seed: int) -> None:
        """Reset the device-resident Philox state the SineGen noise is drawn from (the analogue of ``mx.random.seed``)."""
        self._rng_state = torch.tensor([int(seed), 0], dtype=torch.int64, device=self.device)

    def _capture(self, fn):
        """Warm ``fn`` up once on a side stream (lazy kernel loading, workspace growth), then record it into a CUDA graph that shares
        this model's memory pool (graphs of one model never run concurrently).  Returns (graph, outputs of the captured run, launches)."""
        dev = self.device
        if self._warm_stream is None:
            self._warm_stream = torch.cuda.Stream(device=dev)
        s = self._warm_stream
        s.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(s):
            fn()
        torch.cuda.current_stream(dev).wait_stream(s)
        torch.cuda.synchronize(dev)
        if self._graph_pool is None and self.share_graph_pool:
            self._graph_pool = torch.cuda.graph_pool_handle()
        g = torch.cuda.CUDAGraph()
        n0 = ops.LAUNCHES[0]
        with torch.cuda.graph(g, pool=self._graph_pool if self.share_graph_pool else None):
            out = fn()
        return g, out, ops.LAUNCHES[0] - n0

    def _text_graph(self, T: int, speed: float, pinned: bool):
        key = ("text", T, float(speed), pinned)
        ent = self._graphs.get(key)
        if ent is None:
            dev = self.device
            ent = {"ids": torch.zeros(T, dtype=torch.int64, device=dev), "ref_s": torch.zeros(1, 256, dtype=torch.float32, device=dev),
                   "dur": torch.ones(T, dtype=torch.int64, device=dev) if pinned else None}
            ent["graph"], ent["st"], ent["launches"] = self._capture(lambda: self._text_side(ent["ids"], ent["ref_s"], speed, ent["dur"]))
            self._remember(key, ent)
        return ent

    def _acoustic_graph(self, tg, T: int, F: int, f0n: bool):
        key = ("acoustic", id(tg), T, F, f0n)
        ent = self._graphs.get(key)
        if ent is None:
            dev = self.device
            ent = {"noise": torch.zeros(1, F * 600, 9, dtype=torch.float32, device=dev), "text": tg,
                   "f0n": torch.zeros(2, 2 * F, dtype=torch.float32, device=dev) if f0n else None}
            ent["graph"], ent["audio"], ent["launches"] = self._capture(
                lambda: self._acoustic_side(tg["st"], F, ent["noise"], None if ent["f0n"] is None else (ent["f0n"][0], ent["f0n"][1])))
            self._remember(key, ent)
        return ent

    def _remember(self, key, ent):
        self._graphs[key] = ent
        while len(self._graphs) > self.max_graphs:                     # oldest first; a text graph drags its acoustic graphs along
            old_key = next(iter(self._graphs))
            old = self._graphs.pop(old_key)
            for k in [k for k, v in self._graphs.items() if v.get("text") is old]:
                self._graphs.pop(k)

    @torch.no_grad()
    def synthesize_ids(self, input_ids, ref_s, speed: float = 1.0, *, noise=None, pred_dur=None, n_frames: Optional[int] = None,
                       f0n_override=None, out: Optional[torch.Tensor] = None):
        """`forward_ids` by CUDA-graph replay: one graph for the text / prosody side per (T, speed), ONE host read of the frame count,
        one graph for the acoustic side per (T, F); both are captured the first time a shape is seen and cached (``max_graphs``).
        ``input_ids`` / ``ref_s`` may live in (pinned) host memory -- they are copied into the graphs' static buffers asynchronously.
        SineGen noise comes from the model's device-resident Philox state and differs on every call (``seed()`` resets it); ``noise``
        injects it instead.  Returns (audio [600 F] -- a static buffer that the next call with the same shape overwrites; pass ``out``
        (pinned host or device) to receive a copy -- and pred_dur)."""
        if self._w is None:
            raise RuntimeError("Kokoro: load_weights() has not been called")
        dev = self.device
        ids = torch.as_tensor(input_ids, dtype=torch.int64).reshape(-1)
        T = ids.shape[0]
        assert T <= self.context_length, (T, self.context_length)
        pinned = pred_dur is not None
        tg = self._text_graph(T, float(speed), pinned)
        tg["ids"].copy_(ids, non_blocking=True)
        tg["ref_s"].copy_(torch.as_tensor(ref_s).reshape(1, -1), non_blocking=True)
        if pinned:
            tg["dur"].copy_(torch.as_tensor(pred_dur, dtype=torch.int64).reshape(-1), non_blocking=True)
        tg["graph"].replay()
        ops.LAUNCHES[0] += tg["launches"]
        st = tg["st"]
        F = int(st["total"].item()) if n_frames is None else int(n_frames)   # the one host sync of the utterance
        if F <= 0:
            return torch.zeros(1, device=dev), st["pred"]
        ag = self._acoustic_graph(tg, T, F, f0n_override is not None)
        if noise is not None:
            ag["noise"].copy_(noise, non_blocking=True)
        else:
            if self._rng_state is None:
                self.seed(torch.seed() & 0x7FFFFFFF)
            ops.randn_dev_(ag["noise"], self._rng_state)
        if f0n_override is not None:
            ag["f0n"][0].copy_(torch.as_tensor(f0n_override[0]).reshape(-1), non_blocking=True)
            ag["f0n"][1].copy_(torch.as_tensor(f0n_override[1]).reshape(-1), non_blocking=True)
        ag["graph"].replay()
        ops.LAUNCHES[0] += ag["launches"]
        audio = ag["audio"]
        if out is not None:
            out.copy_(audio, non_blocking=True)
            audio = out
        return audio, st["pred"]

    def __call__(self, phonemes: str, ref_s, speed: Number = 1, return_output: bool = False, decoder=None, **kw):
        """kokoro.py:111-177: phoneme string -> waveform [1, samples] (or Output)."""
        ids = [i for i in (self.vocab.get(p) for p in phonemes) if i is not None]
        assert len(ids) + 2 <= self.context_length, (len(ids) + 2, self.context_length)
        if self.use_graphs and self.tap is None:
            audio, pred = self.synthesize_ids([0, *ids, 0], ref_s, float(speed), **kw)
            if kw.get("out") is None:
                audio = audio.clone()                                  # the graph's static output buffer is reused by the next call
        else:
            audio, pred = self.forward_ids([0, *ids, 0], ref_s, float(speed), **kw)
        audio = audio[None]
        return self.Output(audio=audio, pred_dur=pred) if return_output else audio

    # ------------------------------------------------------------------ generate (kokoro.py:278-370)
    def _get_pipeline(self, lang_code: str, **kw):
        from .pipeline import KokoroPipeline
        if lang_code not in self._pipelines:
            # the cached pipeline refers back to the model weakly: a model <-> pipeline cycle would keep the model's weights and graphs
            # in GPU memory after its last user reference is gone, until some later garbage-collection pass frees them
            self._pipelines[lang_code] = KokoroPipeline(lang_code, weakref.proxy(self), self.repo_id, **kw)
        return self._pipelines[lang_code]

    def _result(self, audio, seg_idx, n_tokens, seg_t):
        samples = audio.shape[1]
        dur = samples / self.sample_rate
        return GenerationResult(
            audio=audio[0], samples=samples, sample_rate=self.sample_rate, segment_idx=seg_idx, token_count=n_tokens,
            audio_duration=f"{int(dur // 3600):02d}:{int(dur // 60) % 60:02d}:{int(dur % 60):02d}.{int((dur % 1) * 1000):03d}",
            real_time_factor=round(seg_t / dur, 2) if dur > 0 else 0,
            prompt={"tokens": n_tokens, "tokens-per-sec": round(n_tokens / seg_t, 2) if seg_t > 0 else 0},
            audio_samples={"samples": samples, "samples-per-sec": round(samples / seg_t, 2) if seg_t > 0 else 0},
            processing_time_seconds=seg_t, peak_memory_usage=torch.cuda.max_memory_allocated(self.device) / 1e9)

    def generate(self, text: str, voice=None, speed: float = 1.0, lang_code: str = "a", split_pattern: str = r"\n+", **kwargs):
        """Generator of GenerationResult (kokoro.py:293-370).  Text goes through the pipeline (pipeline.py): G2P -- the optional ``misaki``
        package, or ``g2p=callable`` -- then <= 510-phoneme chunks, one graph-replayed model call per chunk, ``voice`` = the name of a pack
        under ``voices_dir=`` / a file path / several names averaged / a tensor ``[510, 1, 256]``.  Without G2P pass ``phonemes=`` (a string
        or a list of strings, each <= 510) and either a voice pack or a fixed style row ``ref_s=`` [1, 256]."""
        phonemes = kwargs.pop("phonemes", None)
        ref_s = kwargs.pop("ref_s", None)
        pipe_kw = {k: kwargs.pop(k) for k in ("g2p", "voices_dir") if k in kwargs}
        start = time.time()
        if phonemes is not None:
            from .pipeline import MAX_PHONEMES
            pack = None
            if ref_s is None:
                if voice is None:
                    raise ValueError("pass ref_s [1,256] or a voice (pack tensor [N,1,256], file path or name) with phonemes=")
                pack = self._get_pipeline(lang_code, **pipe_kw).load_voice(voice)
            for seg_idx, ps in enumerate(phonemes if isinstance(phonemes, (list, tuple)) else [phonemes]):
                if len(ps) > MAX_PHONEMES:
                    raise ValueError(f"Phoneme string too long: {len(ps)} > {MAX_PHONEMES}")
                audio = self(ps, ref_s if ref_s is not None else pack[len(ps) - 1], speed)          # pipeline.py:303
                torch.cuda.synchronize(self.device)
                now = time.time()
                seg_t, start = now - start, now
                yield self._result(audio, seg_idx, len(ps), seg_t)
            return
        pipeline = self._get_pipeline(lang_code, **pipe_kw)
        if voice is None:
            voice = "af_heart"
        for seg_idx, (_gs, ps, audio) in enumerate(pipeline(text, voice=voice, speed=speed, split_pattern=split_pattern)):
            torch.cuda.synchronize(self.device)
            now = time.time()
            seg_t, start = now - start, now
            assert audio is not None and audio.shape[1] > 0, "No audio generated"
            yield self._result(audio, seg_idx, len(ps) if ps is not None else 0, seg_t)
