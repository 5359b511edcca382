"""Oracle for Soprano (tts/models/soprano/soprano.py, decoder.py; lm/sample_utils.py; lm/models/qwen3.py): float64 restatement.

TEST INFRASTRUCTURE (see oracle/__init__.py).  Parameters are the sanitized tree (``language_model.*`` Qwen3 names, ``decoder.decoder.*`` the
Vocos backbone in MLX layout, ``decoder.head.out.*``).  The categorical draw is the inverse CDF in index order driven by an injected uniform,
the convention of oracle/qwen3.py and the CUDA samplers.
"""
from __future__ import annotations

import numpy as np
import torch

from . import dsp as D
from . import qwen3 as Q
from . import vocos as VO


# ------------------------------------------------------------------------------------------------ sampler
def keep_mask(logits, top_p: float) -> np.ndarray:
    """apply_top_p (sample_utils.py:206-238) on RAW logits [V]: keep iff the ascending-order inclusive cumulative sum of exp(logit) exceeds
    1 - top_p.  exp in float32 (an overflow to inf keeps every token from that rank up), the sum in float64, ties by lower index first."""
    x = np.asarray(logits, dtype=np.float32)
    order = np.argsort(x, kind="stable")
    with np.errstate(over="ignore"):
        cum = np.cumsum(np.exp(x[order]).astype(np.float64))
    keep = np.zeros(x.shape[0], dtype=bool)
    keep[order] = cum > 1.0 - top_p
    return keep


def sample(logits, u: float, temperature: float, top_p: float):
    """make_sampler(temperature, top_p) as soprano.py:336-346 applies it to one row -> (token, keep mask or None, draw weights or None)."""
    x = np.asarray(logits, dtype=np.float32)
    if temperature == 0:
        return int(np.argmax(x)), None, None
    keep = keep_mask(x, top_p) if 0 < top_p < 1 else np.ones(x.shape[0], dtype=bool)
    if not keep.any():
        return 0, keep, None                                             # MLX's categorical of an all -inf row
    y = (x * np.float32(1.0 / temperature)).astype(np.float64)
    y[~keep] = -np.inf
    w = np.exp(y - y.max())
    cum = np.cumsum(w)
    live = np.nonzero(w > 0)[0]
    hit = live[cum[live] > u * cum[-1]]
    return int(hit[0] if hit.size else live[-1]), keep, w


def sample_margins(logits, u: float, temperature: float, top_p: float):
    """(keep-boundary margin, draw margin), both relative: how far the cumulative sums sit from 1 - top_p and from u * Z at the decisions.
    A kernel that sums in another order may decide differently only where a margin is below ~1e-12."""
    x = np.asarray(logits, dtype=np.float32)
    if temperature == 0:
        return np.inf, np.inf
    mk = np.inf
    if 0 < top_p < 1:
        order = np.argsort(x, kind="stable")
        with np.errstate(over="ignore"):
            cum = np.cumsum(np.exp(x[order]).astype(np.float64))
        thr = 1.0 - top_p
        mk = float(np.min(np.abs(cum - thr)) / thr)
    _, keep, w = sample(x, u, temperature, top_p)
    if w is None:
        return mk, np.inf
    cum = np.cumsum(w)
    t = u * cum[-1]
    return mk, float(np.min(np.abs(cum[w > 0] - t)) / cum[-1])


# ------------------------------------------------------------------------------------------------ LM
def lm_forward(P, ids, cfg, caches):
    """Qwen3Model + final norm + lm_head (lm/models/qwen3.py, soprano.py:269-302) on ids [1, S] at the cache's offset -> (logits, hidden)."""
    x = P["language_model.embed_tokens.weight"][torch.as_tensor(ids, dtype=torch.long)]
    S = x.shape[1]
    off = Q.cache_offset(caches)
    pos = torch.arange(off, off + S)[None]
    cos, sin = Q.rope_cos_sin(pos, cfg["head_dim"], cfg["rope_theta"])
    mask = Q.causal_mask(S, off + S, torch.float64)
    h = Q._decoder_stack(P, "language_model", x, cos, sin, caches, cfg["num_hidden_layers"], cfg["num_attention_heads"],
                         cfg["num_key_value_heads"], cfg["head_dim"], cfg["rms_norm_eps"], mask)
    return h @ P["language_model.lm_head.weight"].T, h


def stream_generate(P, ids, cfg, u, temperature=0.3, top_p=0.95, max_tokens=512, stop_ids=()):
    """soprano.py:304-361 on one prompt -> (tokens [n], hidden [n + 1, H]); u[i] drives the draw at step i."""
    P = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in P.items() if k.startswith("language_model.")}
    caches = Q.make_cache(cfg["num_hidden_layers"])
    logits, h = lm_forward(P, torch.as_tensor(ids)[None], cfg, caches)
    hidden, tokens = [h[0, -1]], []
    for i in range(max_tokens):
        tok, _, _ = sample(logits[0, -1].float().numpy(), float(u[i]), temperature, top_p)
        if tok in stop_ids:
            break
        tokens.append(tok)
        logits, h = lm_forward(P, torch.tensor([[tok]]), cfg, caches)
        hidden.append(h[0, -1])
    return torch.tensor(tokens, dtype=torch.int64), torch.stack(hidden)


def teacher_forced(P, ids, tokens, cfg):
    """The LM of stream_generate fed the given tokens instead of its own draws -> (hidden [n + 1, H], logits [n + 1, V]): row i is what
    the loop yields after the prefill (i = 0) or after feeding tokens[i - 1]."""
    P = {k: torch.as_tensor(v, dtype=torch.float64) for k, v in P.items() if k.startswith("language_model.")}
    caches = Q.make_cache(cfg["num_hidden_layers"])
    logits, h = lm_forward(P, torch.as_tensor(ids)[None], cfg, caches)
    hidden, lg = [h[0, -1]], [logits[0, -1]]
    for t in tokens:
        logits, h = lm_forward(P, torch.tensor([[int(t)]]), cfg, caches)
        hidden.append(h[0, -1])
        lg.append(logits[0, -1])
    return torch.stack(hidden), torch.stack(lg)


# ------------------------------------------------------------------------------------------------ decoder
def decoder_cfg(hidden: int, dim: int, inter: int, layers: int, input_kernel: int, dw_kernel: int, n_fft=2048, hop=512) -> dict:
    return {"backbone": {"init_args": dict(input_channels=hidden, dim=dim, intermediate_dim=inter, num_layers=layers,
                                           input_kernel_size=input_kernel, dw_kernel_size=dw_kernel)},
            "head": {"init_args": {"dim": dim, "n_fft": n_fft, "hop_length": hop}}}


def upsample(x, up: int) -> np.ndarray:
    """decoder.py:102-112: [B, L, H] -> [B, up (L - 1) + 1, H] by align-corners linear interpolation (interpolate.py:61-117)."""
    x = np.asarray(x, dtype=np.float64)
    y = D.interpolate1d(x.transpose(0, 2, 1), up * (x.shape[1] - 1) + 1, mode="linear", align_corners=True)
    return y.transpose(0, 2, 1)


def decode(P, hidden, cfg: dict, up: int = 4) -> torch.Tensor:
    """SopranoDecoder.__call__: hidden [B, L, H] -> [B, hop (L - 1)]."""
    Pv = {k.replace("decoder.decoder.", "backbone.").replace("decoder.head.", "head."): v for k, v in P.items() if k.startswith("decoder.")}
    x = torch.from_numpy(upsample(hidden, up))
    Pv = dict(Pv)
    for i in range(cfg["backbone"]["init_args"]["num_layers"]):
        Pv.setdefault(f"backbone.convnext.{i}.gamma", torch.full((cfg["backbone"]["init_args"]["dim"],), VO.default_gamma(VO.backbone_args(cfg))))
    h = cfg["head"]["init_args"]
    return VO.head(Pv, VO.backbone(Pv, x, cfg), h["n_fft"], h["hop_length"])
