"""Streaming-state kernels (csrc/mimi_stream.cu, csrc/stream.cu) against float64 on every dispatch branch.  Mimi's ``decode_step`` /
``encode_step`` run ``conv1d_stream``, ``convtr1d_stream``, ``ring_rope_kv``, ``ring_attn`` and ``stream_advance``; the Qwen3-TTS
speech tokenizer's ``streaming_step`` keeps its state with ``stream_rows``.  These kernels carry state from one call to the next, so
every case runs a stream of calls (chunk schedules with empty calls, parity flips, ring wraps) and compares the concatenated outputs
with a float64 streaming reference written here.  CPU tests tie each reference to the in-repo oracle: the streaming conv / convtr
references equal ``oracle/nn.py``'s one-shot conv1d / conv_transpose1d, and the ring reference equals full windowed causal attention.

Where each kernel and branch is run:
- conv_stream_kernel, compute CTAs (grid y < cdiv(Lout, 4)): ``test_conv_stream[*]``.  Cout 1 (``cout1-k7``, Mimi's final conv), 31,
  32, 33 (a second, 1-lane 32-channel tile) and 512 (``cout512-cin512-k3``); Cin 1 (``cin1-k7``: 7 of the 8 reduction warps idle), 7,
  8, 9, 512; (K, stride, dilation) (7,1,1), (3,1,1), (3,1,3), (1,1,1) (``cin9-k1``: keff 1, the one dummy history row must keep its
  sentinel), (8,4,1), (10,5,1), (12,6,1), (16,8,1), (4,2,1) with pad_mode 1 (``down-k4s2-edge``, the encoder's downsampler) and
  (3,2,2).  The main schedule gives Lout 0, 1, 2, 3, 4, 5, 9 and 13 per call (partial 4-row tiles); its first chunk (1 row) is shorter
  than the stride where stride > 1, so the fresh call writes no output and carries everything.
- conv_stream_kernel, carry CTAs (the last grid row): every case checks, after every call, that the slot ``*step & 1`` was not
  written, that the other slot holds exactly the raw unconsumed rows, and that its remaining rows keep their sentinel.  A fresh call
  with L = 0 (``lead0`` schedule) must write nothing; non-fresh L = 0 calls (the zeros of every schedule) are a pure carry across the
  parity flip.  ``carry-gridstride-k7-cin512``: Cout 32 with (keff - 1) Cin = 3072 > 256 carry threads.  The history starts as NaN,
  so a fresh call that read it would fail.
- prologues: none, LReLU(0.2), ELU, GELU, GELU-tanh, tanh, SiLU, clip1 (``pre-*`` and the shape cases), sigmoid with pad_mode 1
  (``pre-sigmoid-edge``); sigmoid with pad_mode 0 is rejected (``test_conv_stream_rejects``).  Epilogues: post_act, post_cscale per
  (b, co), res with res_div 1 and 2, bias None or given (``post-*``), B = 3.
- Properties per case: within the bound of the float64 stream; bit-identical across the schedules ``ones``, ``one-call``, ``lead0``
  and ``random`` (per output row the sum order is k, then warp-strided ci, then the fixed 8-way reduction, whatever the split; cases
  with res_div 2 index the residual per call and are compared only on their own schedule); every batch row bit-identical to its B = 1
  stream; the stream started at odd parity (``ctr[1] = 1``) bit-identical.  ``test_conv_stream_graph_replay``: one captured step,
  replayed, equals the eager steps bit for bit.  The four cases ``7-1-1-0-False``, ``3-1-2-0-True``, ``8-4-1-0-False`` and
  ``4-2-1-1-False`` are Mimi-sized (B 2, Cin 48, Cout 40, ELU) on the chunk schedule [5, 0, 1, 13, 2, 40, 3, 0, 17].
- convtr_stream_kernel: ``test_convtr_stream[*]`` at tail lengths nt = K - s of 0 (``nt0-k4s4``: the tail is an empty tensor with a
  null pointer), 2 (Mimi's upsample), 4, 5, 6 and 8 (``nt8-k16s8``: the tail spans two 4-row tiles), nt = L s (``nt-eq-Ls-k6s2``, the
  host limit), K not a multiple of s (``nt4-k7s3``), Cout 1, 31, 33, 512 and Cin 1, 7, 9, 512, with and without ELU and bias.
- convtr_stream_dw_kernel: ``dw-c512-k4s2`` (Mimi's upsample), ``dw-nt0-k2s2`` and ``dw-gridstride`` (3 x 180 x 512 = 276 480
  outputs in one call > 1056 x 256: the grid-stride loop).  A depthwise conv of one channel has groups == 1 and runs the dense kernel:
  ``cin1-cout1-k4s2``.
- Properties per convtr case: the stream within the bound of the float64 transposed conv of the whole sequence cut to L_total s rows;
  after the last call the tail holds the next K - s rows without the bias, within the same bound; the guard words around the tail keep
  their sentinel; each batch row bit-identical to its B = 1 stream.  Bit-identity across chunkings is NOT expected here: the tail is
  summed separately from the rest of its output row, so a different split rounds differently.  ``test_convtr_stream_graph_replay``:
  replay equals eager bit for bit.  ``40-24-8-4-1``, ``64-64-4-2-64``, ``96-48-10-5-1`` run B 2 on [1, 3, 7, 1, 25, 2].
- ring_rope_kv_kernel: ``test_ring_rope_kv[*]`` at D 2, 64, 128 and H 1, 8; ``T-eq-cap`` (one call fills the ring); ``gridstride``
  (4 x 140 x 8 x 64 = 286 720 > 1056 x 256 pairs); positions up to 10^7 (``D128-H8-pos1e7``).  qkv is a column slice of a wider NaN
  buffer whose extra columns must keep their NaN; ring rows not written keep their sentinel; v is copied bit-exact.  q and k must
  equal ``ops.rope_(traditional=True, offset=p0)`` bit for bit: both kernels compile the rotation to the same DMUL + DFMA pair per
  output (a c = fma(a, cs, -(c sn)), fma(a, sn, c cs)) after the same float64 exp / sincos, as their SASS shows.
- ring_attn_kernel: ``test_ring_attn_stream[*]`` at windows 1, 2, 127, 128, 129, 250 and 1024 (WIN_MAX): n below, at and above the
  128 keys of one pass, up to 8 passes; T 1, 3, 128, 256, and the mixed schedule of 1 to 256 positions per call of
  ``test_ring_attention_across_wraps_and_chunks_against_float64`` (B 2, H 8).  Every stream wraps its ring (all but the mixed one at
  least twice), and its first queries sit at p < window - 1, where the window is clamped at 0.  Each stream runs at
  cap = window + T - 1 or just above.  Before every step the test sets every ring row that no query of the step may read to
  NaN on the device, so a read outside the window fails.  Each case is run again on a second schedule at a second capacity and must be
  bit-identical: a query's result depends only on its position, the window and the row values.  ``test_ring_attn_rejects``: window
  1025, cap = window + T - 2 and D != 64 rejected; cap = window + T - 1 accepted.
- stream_advance_kernel: ``test_stream_advance``: dpos 0 and > 0, one advance per CUDA-graph replay, dpos < 0 rejected.
- stream_rows_kernel: ``test_stream_rows_paths[*]``: the float4 path (``vec``) and the scalar path with each of its five conditions
  broken alone (``C6``, ``src_bs``, ``src_ld``, ``dst_bs``, ``dst_off``), copy and add.  ``test_stream_rows_mixed_sizes``: entries
  from 1 element to 2 x 300 x 1024 floats (153 600 float4s > 528 x 256: the grid-stride loop) in one launch.  ``test_stream_rows_limits``:
  32 entries accepted, 33 rejected, empty entries (B, rows or C zero) skipped even where their pointers overlap a live entry.
  ``test_stream_rows_overlap``: an entry's own src / dst overlap, a write to rows another entry reads and two writes to the same rows
  are rejected with ``ops.LAUNCHES`` unchanged and the destinations untouched; the ping-pong carry of a history longer than the new rows
  is accepted.  ``test_stream_rows_speech_tokenizer_tables``: the carry, overflow-add and KV-growth entry tables ``streaming_step``
  builds, on two ping-pong buffer sets.
- Host checks: ``test_conv_stream_rejects``, ``test_convtr_stream_rejects``, ``test_ring_wrappers_reject`` (mismatched, non-contiguous,
  wrong-dtype and undersized rings, a non-int32 pos): every one raises ValueError before any launch.

Tolerances (u = 2^-24).  Each assertion divides the error by its bound and requires a ratio <= 1; the largest ratio measured on an
H100 80GB HBM3 (700 W power limit) is given with each bound.  Each family has a negative control that must fail by more than NEG = 5 times.
- conv_stream / convtr_stream: max |y - ref| <= 2e-5 max |ref|.  An output is an fp32 sum of n = K Cin (convtr: about K Cin / s)
  products in chains of n / 8 plus an 8-way tree, so its error is below (n / 8 + 3) u sum |w x|, and the prologue activation adds a
  few ulp of each input.  The weights are scaled by 1 / sqrt(K Cin), so sum |w x| is about 0.6 sqrt(n) times the output scale: at the
  largest n here (K 7, Cin 512, n = 3584) the worst case is ~1e-3 |y|, but rounding errors of random sign grow as sqrt(n / 8) u times
  the partial sums (~|y|), ~1.3e-6 |y|; 2e-5 of the largest output leaves room for the tail of that distribution at every shape.
  Measured: conv 0.022 (``carry-gridstride-k7-cin512``), convtr 0.012 (``cin512-cout512-k4s2``), the tail 0.0063.  Negative controls:
  the stream run without ``stream_advance`` (it reads the stale slot; 3.4e4), a reference that drops the history (3.4e4), a reference
  with pad_mode swapped (2.4e4); the convtr tail dropped (4.0e4, 4.6e4 depthwise) and the bias counted twice (2.7e3, 2.1e3 depthwise).
- ring_rope_kv: max |y - ref| <= 1e-6 max |ref| for q and k: the angle and rotation are float64 (relative error ~1e-16, times the
  position 10^7 ~1e-9 rad) and the result is rounded once, u |y|.  Measured: 0.048 (``gridstride``), 0.031 at positions near 10^7.
  Negative control: float32 angles at p0 = 10^6, where one ulp is 0.0625 rad (2.1e4).
- ring_attn: max |out - ref| <= 2e-5 max |ref| against float64 attention with float64 RoPE on the fp32 inputs.  The rotated q, k carry
  u each, the 64-term score dots 64 u |q| |k| (scores ~ N(0, 1) here), expf 2 ulp, the sums over up to 1024 keys n / 128 + 7 roundings
  of positive terms; about 1e-6 in all.  Measured: 0.018 (``w129-T3``), 0.014 at window 1024, exactly 0 at window 1.  Negative
  controls: the window one key short (3.2e3) and one key long (3.5e3).
- stream_rows: exact (copies bit for bit, add equal to the float32 ``o + s``).
"""
import math
import random

import pytest
import torch

from oracle import nn as ON

gpu = pytest.mark.gpu
DEV = "cuda:0"
NEG = 5
CONV_TOL = 2e-5
ROPE_TOL = 1e-6
ATTN_TOL = 2e-5
NAN = float("nan")
SENT = -7.25                      # sentinel of history rows, tails and ring rows a call must not touch

ACTS = {"none": 0, "lrelu": 1, "elu": 3, "gelu": 4, "gelu_tanh": 5, "tanh": 6, "sigmoid": 7, "silu": 8, "clip1": 9}
LRELU_SLOPE = 0.2


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _report(name, ratio):
    print(f"{name}: max error / bound = {ratio:.3g}")


def _rel(got, ref, tol):
    """max |got - ref| / (tol max |ref|); NaN counts as an infinite error."""
    err = (got.double().cpu() - ref).abs()
    if err.numel() == 0:
        return 0.0
    if torch.isnan(err).any():
        return math.inf
    return float(err.max() / (tol * ref.abs().max().clamp_min(1e-300)))


def _check(name, got, ref, tol):
    r = _rel(got, ref, tol)
    _report(name, r)
    assert r <= 1.0, (name, r)
    return r


def _neg(name, got, bad_ref, tol):
    r = _rel(got, bad_ref, tol)
    _report(name + " (negative control)", r)
    assert r > NEG, (name, r)


def _bits(t):
    return t.contiguous().view(torch.int32).cpu()


def _same_bits(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


def _wide(t, extra=7, off=3):
    """[B, L, C] float32 on the device as a view: channels offset inside wider NaN rows, every other batch item of a NaN buffer."""
    B, L, C = t.shape
    buf = torch.full((2 * B, L, C + extra), NAN)
    buf[::2, :, off:off + C] = t
    return buf.to(DEV)[::2, :, off:off + C]


def _guarded(B, L, C):
    """(buffer, view): a NaN-filled [B, L + 2, C + 8] device buffer and its [B, L, C] view with guard rows and columns."""
    buf = torch.full((B, L + 2, C + 8), NAN, device=DEV)
    return buf, buf[:, 1:1 + L, 4:4 + C]


def _guards_nan(buf, L, C):
    m = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    m[:, 1:1 + L, 4:4 + C] = False
    return bool(torch.isnan(buf[m]).all())


def act64(x, act, p0=LRELU_SLOPE):
    """float64 reference of b2a_act for the prologue / epilogue activations."""
    if act == 0:
        return x
    if act == 1:
        return torch.where(x > 0, x, x * p0)
    if act == 3:
        return ON.elu(x)
    if act == 4:
        return ON.gelu(x)
    if act == 5:
        return 0.5 * x * (1.0 + torch.tanh(0.7978845608028654 * (x + 0.044715 * x ** 3)))
    if act == 6:
        return torch.tanh(x)
    if act == 7:
        return torch.sigmoid(x)
    if act == 8:
        return x * torch.sigmoid(x)
    if act == 9:
        return x.clamp(-1.0, 1.0)
    raise ValueError(act)


# ======================================================================================================================== references
class ConvStreamRef:
    """StreamableConv1d.step in float64: causal conv of [history | act(new rows)], the unconsumed activated rows carried.  The fresh
    call pads keff - stride rows of zeros (pad_mode 0) or of the first activated row (pad_mode 1).  ``drop_history`` / ``swap_pad``
    are the negative controls."""

    def __init__(self, w, bias, stride, dil, pad_mode, pre_act, drop_history=False, swap_pad=False):
        self.w = w.double()                      # [Cout, K, Cin]
        self.bias = None if bias is None else bias.double()
        self.s, self.d, self.pre = stride, dil, pre_act
        self.pad_mode = 1 - pad_mode if swap_pad else pad_mode
        self.keff = (w.shape[1] - 1) * dil + 1
        self.drop = drop_history
        self.hist = None

    def step(self, x):
        B, c = x.shape[0], x.shape[1]
        xa = act64(x.double(), self.pre)
        if self.hist is None:
            if c == 0:
                return torch.zeros(B, 0, self.w.shape[0], dtype=torch.float64)
            n = self.keff - self.s
            pad = xa[:, :1].expand(B, n, xa.shape[2]) if self.pad_mode == 1 else torch.zeros(B, n, xa.shape[2], dtype=torch.float64)
            v = torch.cat([pad, xa], 1)
        else:
            v = torch.cat([torch.zeros_like(self.hist) if self.drop else self.hist, xa], 1)
        V = v.shape[1]
        lout = (V - self.keff) // self.s + 1 if V >= self.keff else 0
        if lout:
            y = ON.conv1d(v[:, :(lout - 1) * self.s + self.keff], self.w, stride=self.s, dilation=self.d, bias=self.bias)
        else:
            y = torch.zeros(B, 0, self.w.shape[0], dtype=torch.float64)
        self.hist = v[:, lout * self.s:]
        return y


class ConvTrStreamRef:
    """StreamableConvTranspose1d.step in float64: y = bias + the transposed conv of act(x), its first K - s rows plus the held-back
    tail; the tail becomes the next K - s rows without the bias.  ``drop_tail`` / ``bias_twice`` are the negative controls."""

    def __init__(self, w, bias, stride, groups, pre_act, B, drop_tail=False, bias_twice=False):
        self.w, self.s, self.g, self.pre = w.double(), stride, groups, pre_act
        self.bias = None if bias is None else bias.double()
        self.nt = w.shape[1] - stride
        self.tail = torch.zeros(B, self.nt, w.shape[0], dtype=torch.float64)
        self.drop, self.twice = drop_tail, bias_twice

    def step(self, x):
        L = x.shape[1]
        full = ON.conv_transpose1d(act64(x.double(), self.pre), self.w, stride=self.s, groups=self.g)
        y = full[:, :L * self.s].clone()
        if not self.drop:
            y[:, :self.nt] += self.tail
        self.tail = full[:, L * self.s:].clone()
        if self.bias is not None:
            y = y + self.bias
            if self.twice:
                self.tail = self.tail + self.bias
        return y


def rope64(x, offset, base=10000.0):
    """Interleaved-pair RoPE in float64 on [B, T, H, D] at positions offset + t (oracle.nn.rope_traditional)."""
    return ON.rope_traditional(x.permute(0, 2, 1, 3), offset, base).permute(0, 2, 1, 3)


class RingAttnRef:
    """The ring KV cache in float64: k (RoPE'd) and v stored at row p % cap, each query at p attends [max(0, p - window + 1), p]."""

    def __init__(self, B, H, D, cap, window, base=10000.0):
        self.k = torch.full((B, cap, H, D), NAN, dtype=torch.float64)
        self.v = torch.full((B, cap, H, D), NAN, dtype=torch.float64)
        self.H, self.D, self.cap, self.win, self.base, self.pos = H, D, cap, window, base, 0

    def step(self, qkv):
        """qkv float32 [B, T, 3 H D] -> float64 [B, T, H D]; advances the position by T."""
        B, T, _ = qkv.shape
        H, D, p0 = self.H, self.D, self.pos
        x = qkv.double().reshape(B, T, 3, H, D)
        q, k = rope64(x[:, :, 0], p0, self.base), rope64(x[:, :, 1], p0, self.base)
        rows = torch.arange(p0, p0 + T) % self.cap
        self.k[:, rows], self.v[:, rows] = k, x[:, :, 2]
        out = torch.empty(B, T, H, D, dtype=torch.float64)
        for t0 in range(0, T, 32):                                      # query blocks bound the gathered [B, 32, window, H, D]
            t1 = min(T, t0 + 32)
            p = torch.arange(p0 + t0, p0 + t1)[:, None]
            kp = p - self.win + 1 + torch.arange(self.win)[None]       # [t, window] key positions
            valid = kp >= 0
            kr = self.k[:, kp.clamp_min(0) % self.cap]
            vr = self.v[:, kp.clamp_min(0) % self.cap].masked_fill(~valid[None, :, :, None, None], 0.0)
            s = torch.einsum("bthd,btjhd->bthj", q[:, t0:t1], kr) / math.sqrt(D)
            s = s.masked_fill(~valid[None, :, None, :], -math.inf)
            out[:, t0:t1] = torch.einsum("bthj,btjhd->bthd", s.softmax(-1), vr)
        self.pos += T
        return out.reshape(B, T, H * D)


def windowed_attn_full(qkv, H, window, base=10000.0):
    """Full windowed causal attention of a whole sequence (oracle.nn.sdpa with the window mask), float64 RoPE."""
    B, N, _ = qkv.shape
    D = qkv.shape[2] // (3 * H)
    x = qkv.double().reshape(B, N, 3, H, D)
    q = ON.rope_traditional(x[:, :, 0].permute(0, 2, 1, 3), 0, base)
    k = ON.rope_traditional(x[:, :, 1].permute(0, 2, 1, 3), 0, base)
    v = x[:, :, 2].permute(0, 2, 1, 3)
    i, j = torch.arange(N)[:, None], torch.arange(N)[None]
    mask = torch.where((j <= i) & (i - j < window), 0.0, -math.inf).double()
    return ON.sdpa(q, k, v, D ** -0.5, mask).permute(0, 2, 1, 3).reshape(B, N, H * D)


# ======================================================================================================================== CPU ties
def _conv_w(Cout, K, Cin, g):
    return torch.randn(Cout, K, Cin, generator=g) / math.sqrt(K * Cin)


@pytest.mark.parametrize("K,s,d,pad_mode", [(7, 1, 1, 0), (3, 1, 3, 0), (8, 4, 1, 0), (4, 2, 1, 1), (3, 2, 2, 0), (1, 1, 1, 0)])
def test_conv_stream_reference_equals_one_shot_oracle(K, s, d, pad_mode):
    """Concatenated per-call outputs of ConvStreamRef == oracle.nn.conv1d of the padded whole sequence (every complete window)."""
    g = _gen(100 + K * 10 + s)
    B, Cin, Cout = 2, 5, 6
    w, bias = _conv_w(Cout, K, Cin, g), torch.randn(Cout, generator=g)
    chunks = [1, 0, 3, 7, 0, 2, 11, 5]
    x = torch.randn(B, sum(chunks), Cin, generator=g)
    ref = ConvStreamRef(w, bias, s, d, pad_mode, ACTS["elu"])
    outs, a = [], 0
    for c in chunks:
        outs.append(ref.step(x[:, a:a + c]))
        a += c
    got = torch.cat(outs, 1)
    keff = (K - 1) * d + 1
    xa = ON.elu(x.double())
    pad = xa[:, :1].expand(B, keff - s, Cin) if pad_mode else torch.zeros(B, keff - s, Cin, dtype=torch.float64)
    one = ON.conv1d(torch.cat([pad, xa], 1), w.double(), stride=s, dilation=d, bias=bias.double())
    assert got.shape == one.shape
    assert float((got - one).abs().max()) <= 1e-12 * float(one.abs().max())


@pytest.mark.parametrize("K,s,groups", [(4, 2, 1), (7, 3, 1), (4, 4, 1), (16, 8, 1), (4, 2, 6)])
def test_convtr_stream_reference_equals_one_shot_oracle(K, s, groups):
    """Concatenated ConvTrStreamRef outputs == oracle.nn.conv_transpose1d of the whole sequence cut to L_total s rows, and the final
    tail == its next K - s rows without the bias."""
    g = _gen(200 + K * 10 + s)
    B, Cin, Cout = 2, 6, 6
    w, bias = torch.randn(Cout, K, Cin // groups, generator=g), torch.randn(Cout, generator=g)
    chunks = [2, 3, 7, 2, 5]
    x = torch.randn(B, sum(chunks), Cin, generator=g)
    ref = ConvTrStreamRef(w, bias, s, groups, ACTS["elu"], B)
    outs, a = [], 0
    for c in chunks:
        outs.append(ref.step(x[:, a:a + c]))
        a += c
    n = sum(chunks) * s
    one = ON.conv_transpose1d(ON.elu(x.double()), w.double(), stride=s, groups=groups, bias=bias.double())
    scale = float(one.abs().max())
    assert float((torch.cat(outs, 1) - one[:, :n]).abs().max()) <= 1e-12 * scale
    assert ref.tail.shape == one[:, n:].shape
    assert torch.allclose(ref.tail, one[:, n:] - bias.double(), rtol=0.0, atol=1e-12 * scale)


@pytest.mark.parametrize("window,cap,chunks", [(4, 6, [1, 3, 2, 1, 3, 3, 1]), (7, 9, [3, 3, 3, 1, 2, 3, 3, 2]), (1, 3, [3, 1, 2])])
def test_ring_reference_equals_full_windowed_attention(window, cap, chunks):
    g = _gen(300 + window)
    B, H, D = 2, 2, 8
    qkv = torch.randn(B, sum(chunks), 3 * H * D, generator=g)
    ref = RingAttnRef(B, H, D, cap, window)
    outs, a = [], 0
    for c in chunks:
        outs.append(ref.step(qkv[:, a:a + c]))
        a += c
    full = windowed_attn_full(qkv, H, window)
    assert float((torch.cat(outs, 1) - full).abs().max()) <= 1e-12 * float(full.abs().max())


# ======================================================================================================================== conv_stream
def _schedules(s, main):
    n = sum(main)
    rnd = random.Random(n * 7 + s)
    r, left = [], n
    while left:
        c = min(left, rnd.choice([0, 0, 1, 2, 3, s, 2 * s + 1, 5 * s]))
        r.append(c)
        left -= c
    return {"ones": [1] * n, "one-call": [n], "lead0": [0, 0] + main, "random": r}


def _main_schedule(s):
    return [1] + [s * n for n in (2, 0, 1, 3, 4, 5, 9, 0, 13)]


# id: (B, Cin, Cout, K, stride, dilation, pad_mode, pre, post, cscale, res_div (0: no res), bias, chunks or None)
MOVED = [5, 0, 1, 13, 2, 40, 3, 0, 17]
CONV_CASES = {
    "cout1-k7": (3, 64, 1, 7, 1, 1, 0, "elu", "none", False, 0, True, None),
    "cout31-k3d3": (3, 16, 31, 3, 1, 3, 0, "lrelu", "none", False, 0, True, None),
    "cout32-k8s4": (3, 24, 32, 8, 4, 1, 0, "elu", "none", False, 0, True, None),
    "cout33-k10s5": (3, 12, 33, 10, 5, 1, 0, "elu", "none", False, 0, False, None),
    "cout512-cin512-k3": (3, 512, 512, 3, 1, 1, 0, "elu", "none", False, 1, True, None),
    "cin1-k7": (3, 1, 64, 7, 1, 1, 0, "none", "none", False, 0, True, None),
    "cin7-k12s6": (3, 7, 40, 12, 6, 1, 0, "elu", "none", False, 0, True, None),
    "cin8-k16s8": (3, 8, 40, 16, 8, 1, 0, "gelu", "none", False, 0, True, None),
    "cin9-k1": (3, 9, 40, 1, 1, 1, 0, "elu", "none", False, 1, True, None),
    "k3-pad-edge": (3, 16, 24, 3, 1, 1, 1, "elu", "none", False, 0, True, None),
    "down-k4s2-edge": (3, 32, 48, 4, 2, 1, 1, "none", "none", False, 0, True, None),
    "k3s2d2": (3, 20, 24, 3, 2, 2, 0, "tanh", "none", False, 0, True, None),
    "carry-gridstride-k7-cin512": (3, 512, 32, 7, 1, 1, 0, "elu", "none", False, 0, True, None),
    "pre-gelu_tanh": (3, 16, 24, 7, 1, 1, 0, "gelu_tanh", "none", False, 0, True, None),
    "pre-silu": (3, 16, 24, 7, 1, 1, 0, "silu", "none", False, 0, True, None),
    "pre-clip1": (3, 16, 24, 7, 1, 1, 0, "clip1", "none", False, 0, True, None),
    "pre-sigmoid-edge": (3, 16, 24, 4, 2, 1, 1, "sigmoid", "none", False, 0, True, None),
    "post-elu-cscale-res1-nobias": (3, 24, 40, 3, 1, 1, 0, "elu", "elu", True, 1, False, None),
    "post-gelu-cscale-res2": (3, 24, 40, 7, 1, 1, 0, "elu", "gelu", True, 2, True, None),
    "post-tanh-res2-s2": (3, 24, 40, 4, 2, 1, 0, "none", "tanh", False, 2, True, None),
    "7-1-1-0-False": (2, 48, 40, 7, 1, 1, 0, "elu", "none", False, 0, True, MOVED),
    "3-1-2-0-True": (2, 48, 40, 3, 1, 2, 0, "elu", "none", False, 1, True, MOVED),
    "8-4-1-0-False": (2, 48, 40, 8, 4, 1, 0, "elu", "none", False, 0, True, MOVED),
    "4-2-1-1-False": (2, 48, 40, 4, 2, 1, 1, "elu", "none", False, 0, True, MOVED),
}


class ConvCase:
    def __init__(self, cid):
        (self.B, self.Cin, self.Cout, self.K, self.s, self.d, self.pad_mode, pre, post, cscale, self.res_div, bias,
         chunks) = CONV_CASES[cid]
        from mlx_audio_b200 import ops
        g = _gen(sum(map(ord, cid)))
        self.pre, self.post = ACTS[pre], ACTS[post]
        self.keff = (self.K - 1) * self.d + 1
        self.w = _conv_w(self.Cout, self.K, self.Cin, g)
        self.bias = torch.randn(self.Cout, generator=g) * 0.1 if bias else None
        self.cw = ops.pack_conv(self.w, self.bias, 1, DEV)
        self.main = chunks or _main_schedule(self.s)
        self.N = sum(self.main)
        self.x = torch.randn(self.B, self.N, self.Cin, generator=g)
        self.lt = (self.keff - self.s + self.N - self.keff) // self.s + 1
        self.cscale = (torch.rand(self.B, self.Cout, generator=g) + 0.5) if cscale else None
        self.res = torch.randn(self.B, self.lt, self.Cout, generator=g) if self.res_div else None

    def reference(self, chunks, **kw):
        ref = ConvStreamRef(self.w, self.bias, self.s, self.d, self.pad_mode, self.pre, **kw)
        outs, a, lo = [], 0, 0
        for c in chunks:
            y = act64(ref.step(self.x[:, a:a + c]), self.post)
            if self.cscale is not None:
                y = y * self.cscale.double()[:, None]
            if self.res is not None:
                y = y + self.res.double()[:, lo + torch.arange(y.shape[1]) // self.res_div]
            outs.append(y)
            a += c
            lo += y.shape[1]
        return torch.cat(outs, 1)

    def run(self, chunks, *, b=None, parity=0, advance=True, check_state=False, hist_fill=NAN):
        """The device stream over ``chunks`` (batch row ``b`` alone when given) -> concatenated output [B, L, Cout] (CPU)."""
        from mlx_audio_b200 import ops
        sel = slice(None) if b is None else slice(b, b + 1)
        x, B = self.x[sel], (self.B if b is None else 1)
        cs = None if self.cscale is None else self.cscale[sel].to(DEV)
        res = None if self.res is None else self.res[sel]
        hist = torch.full((2, B, max(self.keff - 1, 1), self.Cin), hist_fill, device=DEV)
        ctr = torch.tensor([0, parity], dtype=torch.int32, device=DEV)
        H, fresh, a, lo, outs, par = self.keff - self.s, True, 0, 0, [], parity & 1
        raw = None                                                      # raw carried rows (CPU), None before the first rows
        for c in chunks:
            lout = (H + c - self.keff) // self.s + 1 if H + c >= self.keff else 0
            obuf, out = _guarded(B, lout, self.Cout)
            r = None
            if res is not None:
                r = _wide(res[:, lo:lo + -(-lout // self.res_div)])
            before = hist.clone() if check_state else None
            ops.conv1d_stream(_wide(x[:, a:a + c]) if c else None, self.cw, hist, H, ctr[1:], B=B, stride=self.s, dilation=self.d,
                              pad_mode=self.pad_mode, fresh=fresh, pre=ops.Pre(act=self.pre, p0=LRELU_SLOPE) if self.pre else None,
                              post_act=self.post, cscale=cs, res=r, res_div=max(self.res_div, 1), out=out)
            assert _guards_nan(obuf, lout, self.Cout)
            if check_state:
                if fresh and c == 0:
                    assert _same_bits(hist, before)                     # a fresh call without rows writes nothing
                else:
                    xc = x[:, a:a + c]
                    if fresh:
                        n0 = self.keff - self.s
                        raw = xc[:, :1].expand(B, n0, self.Cin) if self.pad_mode else torch.zeros(B, n0, self.Cin)
                    v = torch.cat([raw, xc], 1)
                    raw = v[:, lout * self.s:]
                    n = raw.shape[1]
                    assert _same_bits(hist[par], before[par]), "the slot being read was written"
                    assert _same_bits(hist[1 - par, :, :n], raw), "the new history is not the raw unconsumed rows"
                    assert _same_bits(hist[1 - par, :, n:], before[1 - par, :, n:]), "rows past the new history were written"
            if not (fresh and c == 0):
                H += c - lout * self.s
                fresh = False
            if advance:
                ops.stream_advance(ctr, 0)
                par ^= 1
            outs.append(out.cpu())
            a += c
            lo += lout
        got = torch.cat(outs, 1)
        assert got.shape == (B, self.lt, self.Cout)
        return got


@gpu
@pytest.mark.parametrize("cid", list(CONV_CASES))
def test_conv_stream(cid):
    k = ConvCase(cid)
    got = k.run(k.main, check_state=True)
    _check(f"conv_stream {cid}", got, k.reference(k.main), CONV_TOL)
    if k.res_div <= 1:
        for name, sch in _schedules(k.s, k.main).items():
            assert _same_bits(k.run(sch, check_state=name == "lead0"), got), name
    for b in range(k.B):
        assert _same_bits(k.run(k.main, b=b), got[b:b + 1]), b
    assert _same_bits(k.run(k.main, parity=1), got)


@gpu
def test_conv_stream_negative_controls():
    k = ConvCase("cout32-k8s4")
    got = k.run(k.main)
    _neg("conv_stream history dropped", got, k.reference(k.main, drop_history=True), CONV_TOL)
    _neg("conv_stream pad_mode swapped", got, k.reference(k.main, swap_pad=True), CONV_TOL)
    stale = k.run([c for c in k.main if c], advance=False, hist_fill=0.0)     # every call after the first reads the stale slot
    _neg("conv_stream without stream_advance", stale, k.reference([c for c in k.main if c]), CONV_TOL)


@gpu
@pytest.mark.parametrize("cid", ["cout32-k8s4", "down-k4s2-edge", "post-gelu-cscale-res2"])
def test_conv_stream_graph_replay(cid):
    """One captured step (conv + stream_advance), replayed on fresh inputs, equals the eager steps bit for bit."""
    from mlx_audio_b200 import ops
    k = ConvCase(cid)
    c, steps = 3 * k.s, 6
    n = c * steps
    k.x = k.x[:, :n] if k.N >= n else torch.randn(k.B, n, k.Cin, generator=_gen(1))
    k.N, k.lt = n, (n - k.s) // k.s + 1
    if k.res is not None:
        k.res = torch.randn(k.B, k.lt, k.Cout, generator=_gen(2))
    if k.res_div:
        k.res_div = 1
    eager = k.run([c] * steps)
    hist = torch.full((2, k.B, max(k.keff - 1, 1), k.Cin), NAN, device=DEV)
    ctr = torch.zeros(2, dtype=torch.int32, device=DEV)
    pre = ops.Pre(act=k.pre, p0=LRELU_SLOPE) if k.pre else None
    cs = None if k.cscale is None else k.cscale.to(DEV)
    kw = dict(B=k.B, stride=k.s, dilation=k.d, pad_mode=k.pad_mode, pre=pre, post_act=k.post, cscale=cs)
    H = k.keff - k.s
    xin = k.x[:, :c].to(DEV).contiguous()
    rin = None if k.res is None else k.res[:, :c // k.s].to(DEV).contiguous()
    outs = [ops.conv1d_stream(xin, k.cw, hist, H, ctr[1:], fresh=True, res=rin, **kw).cpu()]
    ops.stream_advance(ctr, 0)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        yg = ops.conv1d_stream(xin, k.cw, hist, H, ctr[1:], res=rin, **kw)
        ops.stream_advance(ctr, 0)
    for i in range(1, steps):
        xin.copy_(k.x[:, i * c:(i + 1) * c])
        if rin is not None:
            rin.copy_(k.res[:, i * (c // k.s):(i + 1) * (c // k.s)])
        g.replay()
        outs.append(yg.cpu())
    assert int(ctr[1]) == steps
    assert _same_bits(torch.cat(outs, 1), eager)


@gpu
def test_conv_stream_rejects():
    """Host checks of conv1d_stream: each raises ValueError and launches nothing."""
    from mlx_audio_b200 import ops
    g = _gen(5)
    B, Cin, Cout = 2, 8, 16
    cw7 = ops.pack_conv(_conv_w(Cout, 7, Cin, g), None, 1, DEV)
    cw2 = ops.pack_conv(_conv_w(Cout, 2, Cin, g), None, 1, DEV)
    x = torch.randn(B, 10, Cin, device=DEV)
    ctr = torch.zeros(2, dtype=torch.int32, device=DEV)
    hist7 = torch.zeros(2, B, 6, Cin, device=DEV)
    base = dict(B=B, fresh=True)
    bad = {
        "sigmoid prologue with zero padding": lambda: ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], pre=ops.Pre(act=ACTS["sigmoid"]), **base),
        "stride > keff": lambda: ops.conv1d_stream(x, cw2, torch.zeros(2, B, 1, Cin, device=DEV), 0, ctr[1:], stride=3, **base),
        "undersized res": lambda: ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], res=torch.zeros(B, 9, Cout, device=DEV), **base),
        "undersized res (res_div 2)": lambda: ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], res=torch.zeros(B, 4, Cout, device=DEV),
                                                                res_div=2, **base),
        "res of the wrong batch": lambda: ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], res=torch.zeros(1, 10, Cout, device=DEV), **base),
        "undersized out": lambda: ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], out=torch.zeros(B, 9, Cout, device=DEV), **base),
        "out with wrong channels": lambda: ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], out=torch.zeros(B, 10, Cout - 1, device=DEV), **base),
        "int64 step": lambda: ops.conv1d_stream(x, cw7, hist7, 6, torch.zeros(1, dtype=torch.int64, device=DEV), **base),
        "CPU step": lambda: ops.conv1d_stream(x, cw7, hist7, 6, torch.zeros(1, dtype=torch.int32), **base),
        "input channels": lambda: ops.conv1d_stream(x[..., :Cin - 1], cw7, hist7, 6, ctr[1:], **base),
        "history shape": lambda: ops.conv1d_stream(x, cw7, hist7[:, :, :5], 6, ctr[1:], **base),
    }
    for name, f in bad.items():
        n = ops.LAUNCHES[0]
        with pytest.raises(ValueError):
            f()
        assert ops.LAUNCHES[0] == n, name
    # the sigmoid prologue is accepted with edge padding, res of exactly ceil(Lout / res_div) rows is accepted
    ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], pre=ops.Pre(act=ACTS["sigmoid"]), pad_mode=1, **base)
    ops.conv1d_stream(x, cw7, hist7, 6, ctr[1:], res=torch.zeros(B, 5, Cout, device=DEV), res_div=2, **base)
    torch.cuda.synchronize()


@gpu
def test_conv_stream_sigmoid_zero_padding_would_disagree_with_conv1d():
    """Why sigmoid needs pad_mode 1: the one-shot conv pads after the prologue, so its first keff - stride rows see sigmoid(x) next to
    zeros, while a stream that padded before the prologue would see sigmoid(0) = 0.5.  With edge padding the stream matches the
    float64 reference of the activated, edge-padded input."""
    k = ConvCase("pre-sigmoid-edge")
    got = k.run(k.main)
    _check("conv_stream sigmoid edge", got, k.reference(k.main), CONV_TOL)


# ======================================================================================================================== convtr_stream
# id: (B, Cin, Cout, K, stride, groups, pre, bias, chunks or None)
MOVED_TR = [1, 3, 7, 1, 25, 2]
CONVTR_CASES = {
    "nt0-k4s4": (3, 16, 32, 4, 4, 1, "elu", True, None),
    "nt2-k4s2": (3, 64, 33, 4, 2, 1, "elu", True, None),
    "nt4-k8s4-cout31-cin9": (3, 9, 31, 8, 4, 1, "none", True, None),
    "nt5-k10s5-cin1": (3, 1, 48, 10, 5, 1, "elu", False, None),
    "nt6-k12s6-cout1-cin7": (3, 7, 1, 12, 6, 1, "elu", True, None),
    "nt8-k16s8": (3, 24, 40, 16, 8, 1, "elu", True, None),
    "nt4-k7s3": (3, 20, 24, 7, 3, 1, "elu", True, None),
    "cin512-cout512-k4s2": (2, 512, 512, 4, 2, 1, "elu", True, [1, 3, 4, 2]),
    "nt-eq-Ls-k6s2": (3, 16, 24, 6, 2, 1, "elu", True, [2, 2, 2, 2, 2]),
    "cin1-cout1-k4s2": (3, 1, 1, 4, 2, 1, "none", True, None),
    "dw-c512-k4s2": (3, 512, 512, 4, 2, 512, "elu", True, None),
    "dw-nt0-k2s2": (3, 64, 64, 2, 2, 64, "none", False, None),
    "dw-gridstride": (3, 512, 512, 4, 2, 512, "none", False, [90, 1, 95]),
    "40-24-8-4-1": (2, 40, 24, 8, 4, 1, "elu", True, MOVED_TR),
    "64-64-4-2-64": (2, 64, 64, 4, 2, 64, "none", True, MOVED_TR),
    "96-48-10-5-1": (2, 96, 48, 10, 5, 1, "elu", True, MOVED_TR),
}


class ConvTrCase:
    def __init__(self, cid):
        self.B, self.Cin, self.Cout, self.K, self.s, groups, pre, bias, chunks = CONVTR_CASES[cid]
        from mlx_audio_b200 import ops
        g = _gen(sum(map(ord, cid)))
        self.g = groups
        self.pre = ACTS[pre]
        self.nt = self.K - self.s
        self.w = torch.randn(self.Cout, self.K, self.Cin // self.g, generator=g) / math.sqrt(self.K * self.Cin / self.g / self.s)
        self.bias = torch.randn(self.Cout, generator=g) * 0.1 if bias else None
        self.cw = ops.pack_conv(self.w, self.bias, self.g, DEV)
        self.chunks = [max(c, -(-self.nt // self.s)) for c in (chunks or [1, 3, 7, 1, 12, 2, 5])]
        self.x = torch.randn(self.B, sum(self.chunks), self.Cin, generator=g)

    def reference(self, **kw):
        ref = ConvTrStreamRef(self.w, self.bias, self.s, self.g, self.pre, self.B, **kw)
        outs, a = [], 0
        for c in self.chunks:
            outs.append(ref.step(self.x[:, a:a + c]))
            a += c
        return torch.cat(outs, 1), ref.tail

    def run(self, b=None):
        from mlx_audio_b200 import ops
        sel = slice(None) if b is None else slice(b, b + 1)
        x, B = self.x[sel], (self.B if b is None else 1)
        n, G = B * self.nt * self.Cout, 5
        if self.nt:
            tbuf = torch.full((n + 2 * G,), SENT, device=DEV)
            tbuf[G:G + n] = 0
            tail = tbuf[G:G + n].view(B, self.nt, self.Cout)
        else:
            tbuf, tail = None, torch.zeros(B, 0, self.Cout, device=DEV)
            assert tail.data_ptr() == 0                                 # an empty CUDA tensor: the kernel gets a null tail
        outs, a = [], 0
        pre = ops.Pre(act=self.pre) if self.pre else None
        for c in self.chunks:
            obuf, out = _guarded(B, c * self.s, self.Cout)
            ops.convtr1d_stream(_wide(x[:, a:a + c]), self.cw, tail, stride=self.s, pre=pre, out=out)
            assert _guards_nan(obuf, c * self.s, self.Cout)
            outs.append(out.cpu())
            a += c
        if tbuf is not None:
            assert bool((tbuf[:G] == SENT).all()) and bool((tbuf[G + n:] == SENT).all()), "a tail guard word was written"
        return torch.cat(outs, 1), tail.cpu()


@gpu
@pytest.mark.parametrize("cid", list(CONVTR_CASES))
def test_convtr_stream(cid):
    k = ConvTrCase(cid)
    got, tail = k.run()
    ref, ref_tail = k.reference()
    r = _check(f"convtr_stream {cid}", got, ref, CONV_TOL)
    if k.nt:
        rt = _rel(tail, ref_tail, CONV_TOL * float(ref.abs().max()) / float(ref_tail.abs().max().clamp_min(1e-300)))
        _report(f"convtr_stream tail {cid}", rt)
        assert rt <= 1.0, rt
    for b in range(k.B):
        gb, tb = k.run(b)
        assert _same_bits(gb, got[b:b + 1]) and _same_bits(tb, tail[b:b + 1]), b
    assert r <= 1.0


@gpu
@pytest.mark.parametrize("cid", ["nt2-k4s2", "dw-c512-k4s2"])
def test_convtr_stream_negative_controls(cid):
    k = ConvTrCase(cid)
    got, _ = k.run()
    _neg(f"convtr_stream tail dropped {cid}", got, k.reference(drop_tail=True)[0], CONV_TOL)
    _neg(f"convtr_stream bias twice {cid}", got, k.reference(bias_twice=True)[0], CONV_TOL)


@gpu
@pytest.mark.parametrize("cid", ["nt2-k4s2", "dw-c512-k4s2", "nt0-k4s4"])
def test_convtr_stream_graph_replay(cid):
    from mlx_audio_b200 import ops
    k = ConvTrCase(cid)
    c, steps = 3, 5
    k.chunks = [c] * steps
    k.x = torch.randn(k.B, c * steps, k.Cin, generator=_gen(3))
    eager, eager_tail = k.run()
    tail = torch.zeros(k.B, k.nt, k.Cout, device=DEV)
    pre = ops.Pre(act=k.pre) if k.pre else None
    xin = k.x[:, :c].to(DEV).contiguous()
    outs = [ops.convtr1d_stream(xin, k.cw, tail, stride=k.s, pre=pre).cpu()]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        yg = ops.convtr1d_stream(xin, k.cw, tail, stride=k.s, pre=pre)
    for i in range(1, steps):
        xin.copy_(k.x[:, i * c:(i + 1) * c])
        g.replay()
        outs.append(yg.cpu())
    assert _same_bits(torch.cat(outs, 1), eager) and _same_bits(tail, eager_tail)


@gpu
def test_convtr_stream_rejects():
    from mlx_audio_b200 import ops
    g = _gen(6)
    B, Cin, Cout = 2, 8, 16
    cw = ops.pack_conv(torch.randn(Cout, 6, Cin, generator=g), None, 1, DEV)
    x = torch.randn(B, 3, Cin, device=DEV)
    tail = torch.zeros(B, 4, Cout, device=DEV)
    bad = {
        "tail longer than the output": lambda: ops.convtr1d_stream(x[:, :1], cw, tail, stride=2),
        "tail shape": lambda: ops.convtr1d_stream(x, cw, tail[:, :3], stride=2),
        "tail dtype": lambda: ops.convtr1d_stream(x, cw, tail.double(), stride=2),
        "out shape": lambda: ops.convtr1d_stream(x, cw, tail, stride=2, out=torch.zeros(B, 5, Cout, device=DEV)),
    }
    for name, f in bad.items():
        n = ops.LAUNCHES[0]
        with pytest.raises(ValueError):
            f()
        assert ops.LAUNCHES[0] == n, name
    assert bool((tail == 0).all())


# ======================================================================================================================== ring_rope_kv
# id: (B, T, H, D, cap, p0)
ROPE_CASES = {
    "D2-H1": (2, 5, 1, 2, 9, 3),
    "D64-H8": (2, 7, 8, 64, 16, 12),
    "D128-H1": (3, 4, 1, 128, 6, 1000),
    "D128-H8-pos1e7": (2, 5, 8, 128, 11, 10 ** 7 - 2),
    "T-eq-cap": (2, 16, 8, 64, 16, 5),
    "gridstride": (4, 140, 8, 128, 140, 77),
}


def _run_rope(B, T, H, D, cap, p0, g):
    from mlx_audio_b200 import ops
    HD = H * D
    qkv = torch.randn(B, T, 3 * HD, generator=g)
    buf = torch.full((B, T, 3 * HD + 12), NAN)
    buf[:, :, 5:5 + 3 * HD] = qkv
    dbuf = buf.to(DEV)
    view = dbuf[:, :, 5:5 + 3 * HD]
    kr = torch.full((B, cap, HD), SENT, device=DEV)
    vr = torch.full((B, cap, HD), SENT, device=DEV)
    pos = torch.tensor([p0, 0], dtype=torch.int32, device=DEV)
    ops.ring_rope_kv(view, H, kr, vr, pos, base=10000.0)
    assert torch.isnan(dbuf[:, :, :5]).all() and torch.isnan(dbuf[:, :, 5 + 3 * HD:]).all()
    assert int(pos[0]) == p0                                           # the call does not advance the counter
    rows = torch.tensor([(p0 + t) % cap for t in range(T)])
    return qkv, view.cpu(), kr.cpu(), vr.cpu(), rows


@gpu
@pytest.mark.parametrize("cid", list(ROPE_CASES))
def test_ring_rope_kv(cid):
    from mlx_audio_b200 import ops
    B, T, H, D, cap, p0 = ROPE_CASES[cid]
    HD = H * D
    qkv, out, kr, vr, rows = _run_rope(B, T, H, D, cap, p0, _gen(sum(map(ord, cid))))
    x = qkv.double().reshape(B, T, 3, H, D)
    q_ref, k_ref = rope64(x[:, :, 0], p0).reshape(B, T, HD), rope64(x[:, :, 1], p0).reshape(B, T, HD)
    _check(f"ring_rope_kv q {cid}", out[:, :, :HD], q_ref, ROPE_TOL)
    _check(f"ring_rope_kv k {cid}", kr[:, rows], k_ref, ROPE_TOL)
    assert _same_bits(vr[:, rows], qkv[:, :, 2 * HD:])
    assert _same_bits(out[:, :, HD:], qkv[:, :, HD:])                   # k and v columns of qkv are not rewritten
    rest = torch.ones(cap, dtype=torch.bool)
    rest[rows] = False
    assert bool((kr[:, rest] == SENT).all()) and bool((vr[:, rest] == SENT).all())
    q1 = ops.rope_(qkv[:, :, :HD].contiguous().to(DEV), H, offset=p0, base=10000.0, traditional=True).cpu()
    k1 = ops.rope_(qkv[:, :, HD:2 * HD].contiguous().to(DEV), H, offset=p0, base=10000.0, traditional=True).cpu()
    assert _same_bits(out[:, :, :HD], q1) and _same_bits(kr[:, rows], k1)


@gpu
def test_ring_rope_kv_negative_control():
    B, T, H, D, cap, p0 = 2, 4, 2, 64, 4, 10 ** 6
    qkv, out, _, _, _ = _run_rope(B, T, H, D, cap, p0, _gen(11))
    x = qkv.double().reshape(B, T, 3, H, D)
    inv = torch.exp(-torch.arange(D // 2, dtype=torch.float32) * (math.log(10000.0) / (D // 2)))
    ang = (torch.arange(p0, p0 + T, dtype=torch.float32)[:, None] * inv).double()      # float32 angles
    a, c = x[:, :, 0, :, 0::2], x[:, :, 0, :, 1::2]
    cs, sn = ang.cos()[None, :, None], ang.sin()[None, :, None]
    bad = torch.stack([a * cs - c * sn, a * sn + c * cs], -1).reshape(B, T, H * D)
    _neg("ring_rope_kv float32 angles", out[:, :, :H * D], bad, ROPE_TOL)


# ======================================================================================================================== ring_attn
# id: (B, H, window, cap, chunks)
MOVED_RING = [1, 3, 50, 2, 256, 100, 1, 1, 200, 7]
RING_CASES = {
    "w1-T1": (3, 2, 1, 1, [1] * 7),
    "w2-T3": (3, 2, 2, 4, [3] * 6),
    "w127-T128": (3, 2, 127, 254, [128] * 5),
    "w128-T1": (3, 1, 128, 128, [1] * 300),
    "w129-T3": (3, 2, 129, 131, [3] * 100),
    "w250-T128": (3, 2, 250, 377, [128] * 8),
    "w250-T256": (3, 2, 250, 505, [256] * 5),
    "w1024-T256": (3, 1, 1024, 1279, [256] * 11),
}


def _run_ring(qkv, H, window, cap, chunks, nan_fill=True):
    from mlx_audio_b200 import ops
    B, N, w3 = qkv.shape
    HD = w3 // 3
    D = HD // H
    kr = torch.full((B, cap, HD), NAN, device=DEV)
    vr = torch.full((B, cap, HD), NAN, device=DEV)
    ctr = torch.zeros(2, dtype=torch.int32, device=DEV)
    a, outs = 0, []
    for c in chunks:
        if nan_fill:                                                    # rows no query of this step may read
            keep = {p % cap for p in range(max(0, a - window + 1), a)}
            idx = torch.tensor([r for r in range(cap) if r not in keep], dtype=torch.int64, device=DEV)
            if idx.numel():
                kr[:, idx] = NAN
                vr[:, idx] = NAN
        view = _wide(qkv[:, a:a + c], extra=8, off=4)
        ops.ring_rope_kv(view, H, kr, vr, ctr, base=10000.0)
        obuf, out = _guarded(B, c, HD)
        ops.ring_attn(view[:, :, :HD], kr, vr, ctr, n_heads=H, scale=D ** -0.5, window=window, out=out)
        ops.stream_advance(ctr, c)
        assert _guards_nan(obuf, c, HD)
        outs.append(out.cpu())
        a += c
    assert int(ctr[0]) == N and int(ctr[1]) == len(chunks)
    return torch.cat(outs, 1)


def _ring_reference(qkv, H, window, chunks):
    B, N, w3 = qkv.shape
    D = w3 // (3 * H)
    ref = RingAttnRef(B, H, D, window + max(chunks) - 1, window)
    outs, a = [], 0
    for c in chunks:
        outs.append(ref.step(qkv[:, a:a + c]))
        a += c
    return torch.cat(outs, 1)


def _other_schedule(chunks, seed):
    rnd, n, out = random.Random(seed), sum(chunks), []
    tmax = max(chunks)
    while n:
        c = min(n, rnd.choice([1, 2, tmax, max(1, tmax // 2), 3]))
        out.append(c)
        n -= c
    return out


def _ring_stream_case(cid, B, H, window, cap, chunks):
    assert cap >= window + max(chunks) - 1 and sum(chunks) > cap
    qkv = torch.randn(B, sum(chunks), 3 * H * 64, generator=_gen(sum(map(ord, cid))))
    got = _run_ring(qkv, H, window, cap, chunks)
    _check(f"ring_attn {cid}", got, _ring_reference(qkv, H, window, chunks), ATTN_TOL)
    other = _other_schedule(chunks, len(cid))
    cap2 = window + max(other) - 1 + 37
    assert _same_bits(_run_ring(qkv, H, window, cap2, other, nan_fill=False), got)


@gpu
@pytest.mark.parametrize("cid", list(RING_CASES))
def test_ring_attn_stream(cid):
    _ring_stream_case(cid, *RING_CASES[cid])


@gpu
def test_ring_attention_across_wraps_and_chunks_against_float64():
    """Mimi's attention shape (B 2, H 8, window 250) on a mixed schedule of 1 to 256 positions per call, 621 in all, at a capacity of
    window + 2 x 128 + 2: the ring wraps, with a different T on almost every call."""
    _ring_stream_case("chunks-1-3-50-2-256-100-1-1-200-7", 2, 8, 250, 508, MOVED_RING)


@gpu
def test_ring_attn_negative_controls():
    B, H, window, cap, chunks = RING_CASES["w250-T128"]
    qkv = torch.randn(B, sum(chunks), 3 * H * 64, generator=_gen(12))
    got = _run_ring(qkv, H, window, cap, chunks)
    _neg("ring_attn window one key short", got, _ring_reference(qkv, H, window - 1, chunks), ATTN_TOL)
    _neg("ring_attn window one key long", got, _ring_reference(qkv, H, window + 1, chunks), ATTN_TOL)


@gpu
def test_ring_attn_rejects():
    from mlx_audio_b200 import ops
    B, T, H = 2, 5, 2
    q = torch.randn(B, T, H * 64, device=DEV)
    ctr = torch.zeros(2, dtype=torch.int32, device=DEV)

    def call(window, cap, qq=q, heads=H):
        hd = qq.shape[2]
        kr, vr = torch.zeros(B, cap, hd, device=DEV), torch.zeros(B, cap, hd, device=DEV)
        return ops.ring_attn(qq, kr, vr, ctr, n_heads=heads, scale=0.125, window=window)

    n = ops.LAUNCHES[0]
    with pytest.raises(ValueError, match="1024"):
        call(1025, 1025 + T)
    with pytest.raises(ValueError, match="capacity"):
        call(100, 100 + T - 2)
    with pytest.raises(NotImplementedError, match="head dim"):
        call(8, 8 + T, torch.randn(B, T, H * 32, device=DEV))
    assert ops.LAUNCHES[0] == n
    call(100, 100 + T - 1)                                              # cap == window + T - 1
    call(1024, 1024 + T - 1)
    torch.cuda.synchronize()


@gpu
def test_ring_wrappers_reject():
    """ring_rope_kv / ring_attn validate both rings and pos: each raises ValueError before any launch."""
    from mlx_audio_b200 import ops
    B, T, H, D, cap = 2, 3, 2, 64, 8
    qkv = torch.randn(B, T, 3 * H * D, device=DEV)
    kr = torch.zeros(B, cap, H * D, device=DEV)
    ctr = torch.zeros(2, dtype=torch.int32, device=DEV)
    wide = torch.zeros(B, cap, H * D + 4, device=DEV)
    rings = {
        "v ring of another capacity": (kr, torch.zeros(B, cap - 1, H * D, device=DEV), ctr),
        "v ring with other strides": (kr, wide[:, :, :H * D], ctr),
        "k ring not contiguous": (wide[:, :, :H * D], kr.clone(), ctr),
        "rings of a smaller batch": (kr[:1].clone(), kr[:1].clone(), ctr),
        "rings of a larger batch": (torch.zeros(B + 1, cap, H * D, device=DEV), torch.zeros(B + 1, cap, H * D, device=DEV), ctr),
        "rows of another width": (torch.zeros(B, cap, H * D + 4, device=DEV), torch.zeros(B, cap, H * D + 4, device=DEV), ctr),
        "float64 rings": (kr.double(), kr.double(), ctr),
        "CPU rings": (kr.cpu(), kr.cpu(), ctr),
        "int64 pos": (kr, kr.clone(), ctr.long()),
        "CPU pos": (kr, kr.clone(), ctr.cpu()),
    }
    before = qkv.clone()
    for name, (k, v, p) in rings.items():
        n = ops.LAUNCHES[0]
        with pytest.raises(ValueError):
            ops.ring_rope_kv(qkv, H, k, v, p, base=10000.0)
        with pytest.raises(ValueError):
            ops.ring_attn(qkv[:, :, :H * D], k, v, p, n_heads=H, scale=0.125, window=4)
        assert ops.LAUNCHES[0] == n, name
    assert torch.equal(qkv, before)


# ======================================================================================================================== stream_advance
@gpu
def test_stream_advance():
    from mlx_audio_b200 import ops
    ctr = torch.tensor([5, 0], dtype=torch.int32, device=DEV)
    ops.stream_advance(ctr, 0)
    assert ctr.tolist() == [5, 1]
    ops.stream_advance(ctr, 7)
    assert ctr.tolist() == [12, 2]
    n = ops.LAUNCHES[0]
    with pytest.raises(ValueError):
        ops.stream_advance(ctr, -1)
    assert ops.LAUNCHES[0] == n and ctr.tolist() == [12, 2]
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        ops.stream_advance(ctr, 3)
    assert ctr.tolist() == [12, 2]                                      # capture does not run it
    for _ in range(4):
        g.replay()
    assert ctr.tolist() == [24, 6]


# ======================================================================================================================== stream_rows
def _rows_bufs(shape, seed):
    g = _gen(seed)
    return torch.randn(*shape, generator=g).to(DEV), torch.randn(*shape, generator=g).to(DEV)


# id: (B, rows, C, src layout (bs extra, ld extra, offset), dst layout) -- the views are [B, rows, C] of flat buffers
ROWS_PATHS = {
    "vec": (3, 5, 8, (4, 4, 4), (8, 0, 0)),
    "C6": (3, 5, 6, (4, 2, 4), (8, 2, 0)),
    "src_bs": (3, 5, 8, (5, 4, 4), (8, 0, 0)),
    "src_ld": (3, 5, 8, (3, 1, 4), (8, 0, 0)),
    "dst_bs": (3, 5, 8, (4, 4, 4), (7, 0, 0)),
    "dst_off": (3, 5, 8, (4, 4, 4), (8, 0, 1)),
}


def _strided(buf, B, rows, C, lay):
    """A [B, rows, C] view of the flat device buffer with row stride C + ld_extra, batch stride rows (C + ld_extra) + bs_extra and a
    float offset (the buffer itself is 256-byte aligned)."""
    bsx, ldx, off = lay
    ld = C + ldx
    bs = rows * ld + bsx
    return buf.as_strided((B, rows, C), (bs, ld, 1), buf.storage_offset() + off)


def _rows_case(B, rows, C, ls, ld, seed):
    n = B * (rows * (C + 8) + 8) + 16
    src_buf = torch.randn(n, generator=_gen(seed)).to(DEV)
    dst_buf = torch.randn(n, generator=_gen(seed + 1)).to(DEV)
    return src_buf, dst_buf, _strided(src_buf, B, rows, C, ls), _strided(dst_buf, B, rows, C, ld)


def _mask_of(view, buf):
    """Boolean mask over buf's elements covered by the view."""
    m = torch.zeros(buf.numel(), dtype=torch.bool, device=buf.device)
    m.as_strided(view.shape, view.stride(), view.storage_offset() - buf.storage_offset())[...] = True
    return m


@gpu
@pytest.mark.parametrize("add", [False, True], ids=["copy", "add"])
@pytest.mark.parametrize("cid", list(ROWS_PATHS))
def test_stream_rows_paths(cid, add):
    from mlx_audio_b200 import ops
    B, rows, C, ls, ld = ROWS_PATHS[cid]
    sbuf, dbuf, src, dst = _rows_case(B, rows, C, ls, ld, 40)
    vec = all(v % 4 == 0 for v in (C, src.stride(0), src.stride(1), dst.stride(0), dst.stride(1))) and \
        (src.data_ptr() | dst.data_ptr()) % 16 == 0
    assert vec == (cid == "vec")
    before, want = dbuf.clone(), (dst + src if add else src.clone())
    sb = sbuf.clone()
    ops.stream_rows([(src, dst, add)])
    assert _same_bits(dst, want)
    m = _mask_of(dst, dbuf)
    assert _same_bits(dbuf[~m], before[~m]) and _same_bits(sbuf, sb)


@gpu
def test_stream_rows_mixed_sizes():
    """One launch with entries from one element to 614 400 floats (the grid-stride loop), copies and adds, vec and scalar."""
    from mlx_audio_b200 import ops
    shapes = [(1, 1, 1), (2, 300, 1024), (3, 7, 6), (1, 1, 4), (2, 33, 130)]
    ents, checks = [], []
    for i, (B, rows, C) in enumerate(shapes):
        s = torch.randn(B, rows, C, generator=_gen(50 + i)).to(DEV)
        dbuf = torch.full((B, rows + 1, C + 4), SENT, device=DEV)
        d = dbuf[:, :rows, 1:1 + C] if i % 2 else dbuf[:, :rows, :C]
        add = i in (1, 2)
        if add:
            d.copy_(torch.randn(B, rows, C, generator=_gen(60 + i)).to(DEV))
        want = d + s if add else s.clone()
        ents.append((s, d, add))
        checks.append((dbuf, d, want))
    ops.stream_rows(ents)
    for dbuf, d, want in checks:
        assert _same_bits(d, want)
        m = torch.ones(dbuf.shape, dtype=torch.bool, device=DEV)
        m.as_strided(d.shape, d.stride(), d.storage_offset() - dbuf.storage_offset())[...] = False
        assert bool((dbuf[m] == SENT).all())


@gpu
def test_stream_rows_limits():
    from mlx_audio_b200 import ops
    src = torch.randn(33, 2, 3, 8, device=DEV)
    dst = torch.full((33, 2, 3, 8), SENT, device=DEV)
    ops.stream_rows([(src[i], dst[i], False) for i in range(32)])
    assert _same_bits(dst[:32], src[:32]) and bool((dst[32] == SENT).all())
    dst2 = torch.full((33, 2, 3, 8), SENT, device=DEV)
    n = ops.LAUNCHES[0]
    with pytest.raises(ValueError):
        ops.stream_rows([(src[i], dst2[i], False) for i in range(33)])
    assert ops.LAUNCHES[0] == n and bool((dst2 == SENT).all())
    # empty entries are skipped, even one whose pointers overlap a live entry, and do not count against the 32
    dst3 = torch.full((33, 2, 3, 8), SENT, device=DEV)
    empties = [(src[1][:0], dst3[1][:0], False), (src[2][:, :0], dst3[2][:, :0], True), (src[3][:, :, :0], dst3[3][:, :, :0], False),
               (dst3[0][:, :0], src[0][:, :0], False), (dst3[0][:0], dst3[0][:0], True)]
    ents = [(src[i], dst3[i], False) for i in range(32)]
    ents[1:1] = empties                                                  # 37 entries, 32 of them live
    ops.stream_rows(ents)
    assert _same_bits(dst3[:32], src[:32]) and bool((dst3[32] == SENT).all())
    n = ops.LAUNCHES[0]
    ops.stream_rows(empties)
    assert ops.LAUNCHES[0] == n


@gpu
def test_stream_rows_overlap():
    from mlx_audio_b200 import ops
    buf = torch.randn(2, 40, 8, generator=_gen(70)).to(DEV)
    other = torch.randn(2, 40, 8, generator=_gen(71)).to(DEV)
    bad = {
        "own overlap": [(buf[:, 0:10], buf[:, 5:15], False)],
        "write to rows another entry reads": [(buf[:, 0:5], other[:, 0:5], False), (other[:, 20:25], buf[:, 2:7], False)],
        "two writes to the same rows": [(buf[:, 0:5], other[:, 0:5], False), (buf[:, 10:15], other[:, 3:8], True)],
    }
    for name, ents in bad.items():
        b0, o0, n = buf.clone(), other.clone(), ops.LAUNCHES[0]
        with pytest.raises(ValueError):
            ops.stream_rows(ents)
        assert ops.LAUNCHES[0] == n and _same_bits(buf, b0) and _same_bits(other, o0), name
    # ping-pong carry of a history (H = 12 rows) longer than the new rows (L = 5): the last H rows of buffer p become the head of q
    H, L = 12, 5
    p = torch.randn(2, H + L, 8, generator=_gen(72)).to(DEV)
    q = torch.full((2, H + L, 8), SENT, device=DEV)
    ops.stream_rows([(p[:, L:L + H], q[:, :H], False)])
    assert _same_bits(q[:, :H], p[:, L:]) and bool((q[:, H:] == SENT).all())


@gpu
def test_stream_rows_speech_tokenizer_tables():
    """The three entry tables streaming_step builds, on two ping-pong buffer sets of layers (H, C, rows per frame, overflow):
    the carry (last H rows of every buffer into the other copy's head), the transposed conv's overflow add into the next call's
    output head, and the KV-cache growth into a larger buffer, each in one launch."""
    from mlx_audio_b200 import ops
    layers = [(6, 64, 1, 0), (4, 48, 2, 2), (54, 24, 8, 4), (6, 16, 8, 0)]
    B, L, cap = 2, 3, 4
    g = _gen(80)
    bufs = [[torch.randn(B, H + cap * rpf + extra, C, generator=g).to(DEV) for _ in range(2)] for (H, C, rpf, extra) in layers]
    p = 0
    carry, want = [], []
    for (H, C, rpf, extra), (b0, b1) in zip(layers, bufs):
        X, nb = (b0, b1) if p == 0 else (b1, b0)
        end = H + L * rpf
        carry.append((X[:, end - H:end], nb[:, :H], False))
        want.append((nb, X[:, end - H:end].clone(), H))
    ops.stream_rows(carry)
    for nb, w, H in want:
        assert _same_bits(nb[:, :H], w)
    for (H, C, rpf, extra), (X, prev) in zip(layers, bufs):
        if not extra:
            continue
        t0 = H + L * rpf
        head = X[:, H:H + extra].clone()
        ops.stream_rows([(prev[:, t0:t0 + extra], X[:, H:H + extra], True)])
        assert _same_bits(X[:, H:H + extra], head + prev[:, t0:t0 + extra])
    kv = [torch.randn(B, 256, 3 * 2 * 64, generator=g).to(DEV) for _ in range(3)]
    new = [torch.full((B, 512, 3 * 2 * 64), SENT, device=DEV) for _ in kv]
    off = 250
    ops.stream_rows([(old[:, :off], nb[:, :off], False) for old, nb in zip(kv, new)])
    for old, nb in zip(kv, new):
        assert _same_bits(nb[:, :off], old[:, :off]) and bool((nb[:, off:] == SENT).all())
