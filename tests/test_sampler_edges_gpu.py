"""The token samplers (csrc/sampler.cu: b2a_sample_token, b2a_whisper_greedy_step) and the frame-input embedding sum
(csrc/lm.cu: b2a_embed_sum) against the oracle where a sampler goes wrong quietly: ties at every cutoff (signed zeros
included), adjacent logits that tie only after the division by the temperature, both ends of the vocabulary range of the
4096-slot kernel, draws next to a cumulative boundary, and the arguments the Qwen3-TTS frame loop passes.

Reference: oracle/qwen3.py:sample_token (divide by the temperature, rank by value desc then index asc, inverse CDF in index
order) and oracle/whisper.py:apply_filters / sample_update.  After suppress, penalty and temperature the filtered logits of
both kernel paths ("fast": top-k only; "sorted": top-p or min-p) are the scaled logits or -inf, so they are compared with
torch.equal and tokens with ==.  Two things the kernel computes in another order than the oracle -- the float32 top-p
prefix scan and the float64 draw sums -- are only exercised where a float64 check on the CPU keeps every boundary out of
their reach: cumulative top-p sums at least 1e-5 from 1 - top_p, min-p log ratios at least 1e-4 from log(min_p), and the
draw target at least 1e-9 of the total from every cumulative sum (u = 0 is exact: every live weight is positive).
test_constructions_hold_on_cpu checks those constructions without a GPU."""
import math

import numpy as np
import pytest
import torch

from oracle import qwen3 as Q
from oracle import whisper as OW

U_LAST = 1.0 - 2.0 ** -24                 # the largest float32 below 1
TOPP_MARGIN, MINP_MARGIN, DRAW_MARGIN = 1e-5, 1e-4, 1e-9
TINY_MIN_P = 1e-30                        # routes a row to the sorted path without removing anything (checked per case)


def _dev():
    return torch.device("cuda:0")


# ------------------------------------------------------------------------------------------------ constructions (CPU)
def div_tie_pair(t, seed=0):
    """Adjacent float32 logits a < b (seeded search) with a / t == b / t but a * (1 / t) != b * (1 / t) in float32: they tie
    after the reference's division by the temperature and do not after a multiplication by its reciprocal."""
    tf = np.float32(t)
    inv = np.float32(1.0) / tf
    rng = np.random.default_rng(seed)
    for _ in range(100000):
        a = np.float32(rng.uniform(0.25, 1.0))
        b = np.nextafter(a, np.float32(np.inf))
        if a / tf == b / tf and a * inv != b * inv:
            return float(a), float(b)
    raise AssertionError(f"no tie pair for t={t}")


def grid_row(V, seed):
    """Logits on a coarse grid (multiples of 0.25 in [-3, 3]) with both signed zeros: long runs of equal values."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(-12, 13, (V,), generator=g).float() * 0.25
    zeros = (x == 0).nonzero().flatten()
    x[zeros[torch.rand(zeros.numel(), generator=g) < 0.5]] = -0.0
    return x


def scaled_row(x, temperature, rep=1.0, seen=None, suppress=None):
    """The oracle's logits after suppress, repetition penalty and temperature (no rank filter)."""
    return Q.sample_token(x, 0.0, temperature, 0, 1.0, rep, seen, suppress, 0.0, return_filtered=True)[1]


def filter_margins(scaled, top_k, top_p, min_p):
    """Float64 distances of a row's scaled logits from the top-p and min-p cutoffs (inf where the filter is off).  Logits
    equal to the row maximum are exact on both sides (the comparison is x - max < log(min_p) <= 0) and are left out."""
    s = scaled.double()
    if 0 < top_k < s.shape[0]:
        s = Q.apply_top_k(s, top_k)
    mp = mm = math.inf
    if 0 < top_p < 1:
        cum = torch.cumsum(torch.sort(torch.softmax(s, 0)).values, 0)     # ascending; the order among equal values does not change the sums
        mp = float((cum - (1 - top_p)).abs().min())
    if min_p > 0:
        live = s[torch.isfinite(s)]
        d = live - live.max()
        d = d[d < 0]
        if d.numel():
            mm = float((d - math.log(min_p)).abs().min())
    return mp, mm


def draw_margin(filtered, u):
    """Distance of the draw target u * total from the nearest cumulative sum of the index-order CDF, as a share of the total.
    The last sum is the total itself, which u < 1 keeps above the target in any summation order, and u = 0 is below every
    sum; neither counts."""
    if float(u) == 0.0:
        return math.inf
    w = torch.exp((filtered - filtered.max()).double())
    cum = torch.cumsum(w, 0)
    tot = float(cum[-1])
    inner = cum[w > 0][:-1]
    return float((inner - float(u) * tot).abs().min()) / tot if inner.numel() else math.inf


def u_at(filtered, i):
    """A float32 uniform whose draw target sits in the middle of token i's interval of the index-order CDF."""
    w = torch.exp((filtered - filtered.max()).double())
    cum = torch.cumsum(w, 0)
    return float(np.float32((float(cum[i]) - float(w[i]) / 2) / float(cum[-1])))


def expect(logits, u, temperature, top_k=0, top_p=1.0, min_p=0.0, rep=1.0, seen=None, suppress=None, check=True):
    """The oracle's token and filtered logits for every row of ``logits`` [B, V]; with ``check`` each row's margins are
    asserted, otherwise (None, None) comes back when one of them fails."""
    toks, filt = [], []
    for b in range(logits.shape[0]):
        ub = 0.0 if u is None else float(u[b])
        gen = seen[b] if seen else None
        tok, f = Q.sample_token(logits[b], ub, temperature, top_k, top_p, rep, gen, suppress, min_p, return_filtered=True)
        if temperature > 0:
            mp, mm = filter_margins(scaled_row(logits[b], temperature, rep, gen, suppress), top_k, top_p, min_p)
            dm = draw_margin(f, ub)
            ok = mp >= TOPP_MARGIN and mm >= MINP_MARGIN and dm >= DRAW_MARGIN
            if check:
                assert ok, (b, mp, mm, dm)
            elif not ok:
                return None, None
        toks.append(tok)
        filt.append(f)
    return toks, torch.stack(filt)


def removes_nothing(logits, u, temperature, top_k=0, rep=1.0, seen=None, suppress=None):
    """min_p = TINY_MIN_P leaves the oracle's filtered logits as top-k alone leaves them."""
    a = expect(logits, u, temperature, top_k, 1.0, TINY_MIN_P, rep, seen, suppress)[1]
    b = expect(logits, u, temperature, top_k, 1.0, 0.0, rep, seen, suppress)[1]
    return torch.equal(a, b)


# ---- shape and filter matrix
VS = (1, 7, 33, 1000, 1024, 2048, 3072, 4095, 4096)
TS = (0.9, 0.7, 1.0, 0.05, 3.0)
SORTED = ((0.9, 0.0), (1.0, 0.05), (0.8, 0.02), (0.95, 0.1))            # (top_p, min_p): top_p < 1 or min_p > 0


def top_ks(V):
    return (0, 1, 2, 50, V - 1, V, V + 7)


def matrix():
    """Two cases per (V, path).  Along each path every V, B, top_k and temperature value appears (offsets differ per path)."""
    cases = []
    for path, ok, ot in (("fast", 0, 0), ("sorted", 3, 2)):
        for n in range(2 * len(VS)):
            V = VS[n // 2]
            top_p, min_p = (1.0, 0.0) if path == "fast" else SORTED[n % len(SORTED)]
            ki = (n + ok) % 7
            cases.append(dict(path=path, n=n, V=V, B=(1, 5)[n % 2], ki=ki, top_k=top_ks(V)[ki], temperature=TS[(n + ot) % 5],
                              top_p=top_p, min_p=min_p))
    return cases


def matrix_inputs(c):
    """Gaussian logits, uniforms, a repetition-penalty set on every third case and a suppress list on every fourth: the first
    seed whose rows keep every margin."""
    V, B = c["V"], c["B"]
    kw = dict(top_k=c["top_k"], top_p=c["top_p"], min_p=c["min_p"])
    for seed in range(200):
        g = torch.Generator().manual_seed(100000 * (c["path"] == "sorted") + 1000 * c["n"] + seed)
        logits = torch.randn(B, V, generator=g) * 2.0
        u = torch.rand(B, generator=g)
        seen = [torch.randint(0, V, (V // 8 + 1,), generator=g).tolist() for _ in range(B)] if c["n"] % 3 == 0 else None
        suppress = sorted(set(torch.randint(0, V, (V // 10,), generator=g).tolist())) if c["n"] % 4 == 1 else None
        kw.update(rep=1.3 if seen else 1.0, seen=seen, suppress=suppress or None)
        toks, filt = expect(logits, u, c["temperature"], **kw, check=False)
        if toks is not None:
            return logits, u, kw, toks, filt
    raise AssertionError(f"no seed keeps the margins for {c}")


# ---- ties
TIE_KINDS = ("top_k_in_zeros", "top_k_in_run", "top_p_in_zeros", "min_p_1_top_k_in_max_run", "min_p_1")


def tie_case(kind, V, t, seed=0):
    """A grid row and filters whose cutoff falls inside a run of equal values.  Returns (x, sorted-path filters, the top_k
    that gives the same kept set on the fast path, the kept indices, the run's last kept index, u in the middle of its
    interval).
    The zero cases take the first seed whose cut leaves a -0.0 kept ahead of a dropped +0.0, so ranking +0.0 above -0.0
    would change the kept set."""
    for s in range(seed, seed + 50):
        x = grid_row(V, s)
        if kind in ("top_k_in_zeros", "top_p_in_zeros"):
            level = 0.0
        elif kind == "top_k_in_run":
            level = 1.0
        else:
            level = float(x.max())
        run = (x == level).nonzero().flatten().tolist()
        above = [i for i in range(V) if x[i] > level]
        keep = len(run) // 2 if kind in ("top_k_in_zeros", "top_k_in_run") else len(run) - len(run) // 2
        if kind == "min_p_1_top_k_in_max_run":
            keep = 2
        if kind == "min_p_1":
            keep = len(run)
        if level == 0.0:
            neg = torch.signbit(x[run])
            if not (bool(neg[:keep].any()) and not bool(neg[keep:].all())):
                continue
        break
    else:
        raise AssertionError(f"no seed separates the signed zeros for {kind}")
    assert 0 < keep <= len(run) and len(run) >= 3
    fast_k = len(above) + keep
    if kind.startswith("top_k"):
        filters = dict(top_k=fast_k, min_p=TINY_MIN_P)
    elif kind == "top_p_in_zeros":
        sc = scaled_row(x, t).double()
        p = torch.softmax(sc, 0)
        c0 = float(p[x < 0].sum())
        drop = len(run) - keep                                           # the highest-index zeros come first in ascending order
        filters = dict(top_p=1.0 - (c0 + (drop + 0.5) * float(p[run[0]])))
    elif kind == "min_p_1_top_k_in_max_run":
        filters = dict(top_k=2, min_p=1.0)
    else:
        filters = dict(min_p=1.0)
    kept = sorted(above + run[:keep])
    f = expect(x[None], torch.zeros(1), t, **filters)[1][0]
    return x, filters, fast_k, kept, run[keep - 1], u_at(f, run[keep - 1])


# ---- temperature rounding
def pair_row(V, t, k=50, lo=100, hi=200, seed=0):
    """k - 1 logits above a tie pair (a at index lo, b = nextafter(a) at index hi), the rest below: the pair sits at ranks k
    and k + 1, so top-k keeps exactly one of them."""
    a, b = div_tie_pair(t, seed)
    g = torch.Generator().manual_seed(seed)
    x = -3.0 * torch.rand(V, generator=g)
    idx = [i for i in torch.randperm(V, generator=g).tolist() if i not in (lo, hi)][: k - 1]
    x[idx] = 2.0 + torch.rand(k - 1, generator=g)
    x[lo], x[hi] = a, b
    return x


# ---- draw boundaries
def draw_case(V, where, sorted_path, seed=0):
    """Live tokens only in the first lane's chunk of the 32-lane draw, only in the last lane's chunk, or a single one; the last
    live token is given the row's maximum so u = 1 - 2^-24 lands on it.  Five copies of the row with u = 0, 1 - 2^-24 and
    three seeded interior uniforms."""
    per = (V + 31) // 32
    live = {"first_lane": list(range(0, per)), "last_lane": list(range(31 * per, V)), "single": [V // 2 + 3]}[where]
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(V, generator=g) * 1.5
    x[live[-1]] = x[live].max()
    suppress = sorted(set(range(V)) - set(live))
    u = torch.cat([torch.tensor([0.0, U_LAST]), torch.rand(3, generator=g)])
    kw = dict(top_k=0, top_p=0.9 if sorted_path else 1.0, min_p=0.02 if sorted_path else 0.0, suppress=suppress)
    return x[None].repeat(5, 1), u, kw, live


# ---- Whisper step at temperature > 0
def whisper_hist(spec):
    """The crafted token histories of test_whisper_gpu.py: first sampled position, after one timestamp, text, text then a
    timestamp, a closed timestamp pair, a finished (eot) row."""
    sot, tb = list(spec.sot_sequence), spec.timestamp_begin
    return [sot, sot + [tb + 5], sot + [tb + 5, 100], sot + [tb + 5, 100, tb + 20], sot + [tb + 5, 100, tb + 20, tb + 20],
            sot + [tb + 5, 100, spec.eot]]


WHISPER_SB, WHISPER_SUPPRESS, WHISPER_MAX_TS = 3, (7, 8, 9), 50


def whisper_case(h, scale, ts_boost, t, seed):
    """Three rows with history h: u = 0, u in the middle of the heaviest token's interval, and u = 1 - 2^-24 with the last live
    token raised to the row's maximum + 2.  The kernel forms x - max in float32 before its float64 exponent, so every draw
    target is asserted at least 4 * 2^-24 * span / t of the total (span: range of the live logits) from every cumulative sum.
    Returns the logits, the uniforms, the oracle's filtered logits and which rows keep a live token (the timestamp rules can
    mask a whole row)."""
    spec = OW.TokenizerSpec()
    V, tb = 51865, spec.timestamp_begin
    g = torch.Generator().manual_seed(seed)
    logits = torch.randn(3, V, generator=g) * scale
    logits[:, tb:] += ts_boost
    rows = [h] * 3
    f = OW.apply_filters(logits.double(), rows, spec, WHISPER_SB, WHISPER_SUPPRESS, WHISPER_MAX_TS)
    alive = [bool(torch.isfinite(f[b]).any()) for b in range(3)]
    if alive[2]:
        last = int(torch.isfinite(f[2]).nonzero().flatten()[-1])
        logits[2, last] = float(f[2][torch.isfinite(f[2])].max()) + 2.0
        f = OW.apply_filters(logits.double(), rows, spec, WHISPER_SB, WHISPER_SUPPRESS, WHISPER_MAX_TS)
        assert int(torch.isfinite(f[2]).nonzero().flatten()[-1]) == last
    u = torch.tensor([0.0, u_at(f[1] / t, int(torch.argmax(f[1]))) if alive[1] else 0.5, U_LAST])
    for b in (1, 2):
        if alive[b]:
            live = f[b][torch.isfinite(f[b])]
            need = max(DRAW_MARGIN, 4 * 2.0 ** -24 * float(live.max() - live.min()) / t)
            assert draw_margin(f[b] / t, u[b]) >= need, (h, scale, ts_boost, t, b)
    return logits, u, f, alive


# ------------------------------------------------------------------------------------------------ kernel runner
def mask_of(V, idx):
    m = torch.zeros(V)
    if idx:
        m[list(idx)] = float("-inf")
    return m


def seen_rows(V, lists, pad=0):
    """uint8 [B, V + pad]: 1 at every listed token; the caller slices [:, :V] so the row stride is V + pad."""
    s = torch.zeros(len(lists), V + pad, dtype=torch.uint8)
    for b, l in enumerate(lists):
        if l:
            s[b, l] = 1
    return s


def run(logits, u, temperature, top_k=0, top_p=1.0, min_p=0.0, rep=1.0, seen=None, suppress=None, seen_pad=0):
    from mlx_audio_b200 import ops
    dev = _dev()
    V = logits.shape[1]
    sm = mask_of(V, suppress).to(dev) if suppress else None
    sd = seen_rows(V, seen, seen_pad).to(dev)[:, :V] if seen else None
    tok, filt = ops.sample_token(logits.to(dev), temperature=temperature, top_k=top_k, top_p=top_p, min_p=min_p,
                                 u=None if u is None else u.float().to(dev), suppress_mask=sm, seen=sd, repetition_penalty=rep,
                                 return_filtered=True)
    return tok.cpu().tolist(), filt.cpu()


def check(logits, u, temperature, seen_pad=0, **kw):
    """Kernel vs oracle: equal tokens; at temperature > 0 also torch.equal filtered logits."""
    want_t, want_f = expect(logits, u, temperature, **kw)
    got_t, got_f = run(logits, u, temperature, seen_pad=seen_pad, **kw)
    assert got_t == want_t
    if temperature > 0:
        assert torch.equal(got_f, want_f)
    return got_t, got_f


# ------------------------------------------------------------------------------------------------ CPU
def test_constructions_hold_on_cpu():
    """The cases below are what they claim to be: the temperature pair ties under division only, the matrix covers every
    axis value on both paths and every case keeps its margins, the tie cuts fall inside runs, the draw and Whisper cases
    keep their margins."""
    for t in (0.9, 0.7):
        a, b = div_tie_pair(t)
        tf, inv = np.float32(t), np.float32(1.0) / np.float32(t)
        assert a < b and np.nextafter(np.float32(a), np.float32(np.inf)) == np.float32(b)
        assert np.float32(a) / tf == np.float32(b) / tf and np.float32(a) * inv < np.float32(b) * inv
        ab = torch.tensor([a, b])
        assert float((ab / t)[0]) == float((ab / t)[1])                  # the oracle's own arithmetic ties them
        for V in (3072, 2048):
            x = pair_row(V, t)
            order = sorted(range(V), key=lambda i: (-float(x[i] / t), i))
            assert order[49:51] == [100, 200]
            f = expect(x[None], torch.zeros(1), t, top_k=50)[1][0]
            assert torch.isfinite(f[100]) and torch.isinf(f[200])
            assert removes_nothing(x[None], torch.zeros(1), t, top_k=50)
    cases = matrix()
    assert 30 <= len(cases) <= 45
    for path in ("fast", "sorted"):
        cs = [c for c in cases if c["path"] == path]
        assert {c["V"] for c in cs} == set(VS) and {c["B"] for c in cs} == {1, 5} and {c["temperature"] for c in cs} == set(TS)
        assert {c["ki"] for c in cs} == set(range(7))
        assert all((c["top_p"] == 1.0 and c["min_p"] == 0.0) == (path == "fast") for c in cs)
    for c in cases:
        matrix_inputs(c)
    for kind in TIE_KINDS:
        for V, t in ((200, 1.0), (3072, 0.9)):
            x, filters, fast_k, kept, _, _ = tie_case(kind, V, t)
            for kw in (filters, dict(top_k=fast_k)):
                f = expect(x[None], torch.zeros(1), t, **kw)[1][0]
                assert torch.isfinite(f).nonzero().flatten().tolist() == kept, (kind, kw)
    for V in (2048, 3072, 4095):
        for where in ("first_lane", "last_lane", "single"):
            for sorted_path in (False, True):
                rows, u, kw, live = draw_case(V, where, sorted_path)
                toks, f = expect(rows, u, 1.0, **kw)
                w = torch.exp((f[0] - f[0].max()).double())
                alive = (w > 0).nonzero().flatten().tolist()
                assert set(alive) <= set(live) and toks[0] == alive[0] and toks[1] == alive[-1] and float(w[alive[-1]] / w.sum()) >= 1e-6
    spec = OW.TokenizerSpec()
    for t in (0.5, 1.0):
        n_alive = 0
        for i, (scale, boost) in enumerate(((3.0, 0.0), (3.0, 6.0), (0.01, 0.0))):
            for j, h in enumerate(whisper_hist(spec)):
                n_alive += sum(whisper_case(h, scale, boost, t, seed=10 * i + j)[3])
        assert 36 <= n_alive < 54                                        # mostly live rows, and some fully masked ones


# ------------------------------------------------------------------------------------------------ GPU: b2a_sample_token
@pytest.mark.gpu
@pytest.mark.parametrize("c", matrix(), ids=lambda c: f"{c['path']}-V{c['V']}-B{c['B']}-k{c['top_k']}-t{c['temperature']}")
def test_shape_and_filter_matrix(c):
    logits, u, kw, toks, filt = matrix_inputs(c)
    got_t, got_f = run(logits, u, c["temperature"], **kw)
    assert got_t == toks and torch.equal(got_f, filt)


@pytest.mark.gpu
@pytest.mark.parametrize("V,t", [(200, 1.0), (3072, 0.9)])
@pytest.mark.parametrize("kind", TIE_KINDS)
def test_ties_keep_the_lowest_indices_on_both_paths(kind, V, t):
    """Cutoffs inside runs of equal grid values, signed zeros included: the kept set is every value above the run plus the
    run's lowest indices, on the sorted path with the case's own filter and on the fast path with the top_k that keeps the
    same set."""
    x, filters, fast_k, kept, last, u = tie_case(kind, V, t)
    uu = torch.tensor([u])
    tok_s, f_sorted = check(x[None], uu, t, **filters)
    tok_f, f_fast = check(x[None], uu, t, top_k=fast_k)
    assert torch.isfinite(f_sorted[0]).nonzero().flatten().tolist() == kept and torch.equal(f_fast, f_sorted)
    assert tok_s == tok_f == [last]


@pytest.mark.gpu
def test_greedy_ties_pick_the_lowest_index():
    """temperature 0: the first maximal index, across signed zeros and across a run of equal maxima."""
    rows = torch.stack([-grid_row(3072, 1).abs(), grid_row(3072, 2), grid_row(3072, 3).clamp(max=2.0)])
    rows[0, :5] = -1.0                                                   # row 0: the maximum is a run of -0.0 / +0.0 after index 4
    for b in range(3):
        assert int((rows[b] == rows[b].max()).sum()) >= 3
    toks, _ = check(rows, None, 0.0)
    for b in range(3):
        assert toks[b] == int((rows[b] == rows[b].max()).nonzero()[0])


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["fast", "sorted"])
@pytest.mark.parametrize("V", [3072, 2048])
@pytest.mark.parametrize("t", [0.9, 0.7])
def test_temperature_tie_pair_at_the_top_k_cut(t, V, path):
    """Logits a < b one ulp apart at ranks 50 and 51 with a / t == b / t: the reference keeps the lower index (a at 100), and
    the draw is aimed at it.  Multiplying by 1 / t instead separates them and keeps b at 200."""
    x = pair_row(V, t)
    f = expect(x[None], torch.zeros(1), t, top_k=50)[1][0]
    u = torch.tensor([u_at(f, 100)])
    tok, got = check(x[None], u, t, top_k=50, min_p=TINY_MIN_P if path == "sorted" else 0.0)
    assert tok == [100] and torch.isfinite(got[0, 100]) and torch.isinf(got[0, 200])


@pytest.mark.gpu
@pytest.mark.parametrize("V,t,top_k", [(3072, 0.9, 50), (2048, 0.9, 50), (4095, 0.7, 0), (4096, 3.0, 1000), (1000, 1.0, 0)])
def test_fast_and_sorted_paths_agree(V, t, top_k):
    """The same rows through the fast path and through the sorted path with a min_p that removes nothing (checked on the CPU):
    identical tokens and filtered logits."""
    g = torch.Generator().manual_seed(V + top_k)
    logits = torch.randn(5, V, generator=g) * 2.0
    u = torch.rand(5, generator=g)
    assert removes_nothing(logits, u, t, top_k)
    ta, fa = check(logits, u, t, top_k=top_k)
    tb, fb = check(logits, u, t, top_k=top_k, min_p=TINY_MIN_P)
    assert ta == tb and torch.equal(fa, fb)


@pytest.mark.gpu
@pytest.mark.parametrize("sorted_path", [False, True])
@pytest.mark.parametrize("where", ["first_lane", "last_lane", "single"])
@pytest.mark.parametrize("V", [2048, 3072, 4095])
def test_draw_boundaries(V, where, sorted_path):
    """u = 0 draws the first live token, u = 1 - 2^-24 the last, interior uniforms the oracle's token; the live tokens sit in
    one lane's chunk of the warp draw, or there is one live token."""
    rows, u, kw, live = draw_case(V, where, sorted_path)
    toks, f = check(rows, u, 1.0, **kw)
    alive = torch.isfinite(f[0]).nonzero().flatten().tolist()
    assert set(alive) <= set(live) and toks[0] == alive[0] and toks[1] == alive[-1]
    if where == "single":
        assert toks == [live[0]] * 5


@pytest.mark.gpu
def test_masks_and_repetition_penalty():
    """Everything suppressed but one token; the penalty on negative, positive and both zero logits with a ``seen`` row stride
    larger than V; an all -inf row."""
    g = torch.Generator().manual_seed(6)
    for V, t, kw in ((3072, 0.9, dict(top_k=50)), (2048, 0.7, dict(top_k=50, top_p=0.9)), (4096, 0.0, {})):
        logits = torch.randn(2, V, generator=g)
        one = 1234
        u = torch.tensor([0.0, U_LAST])
        toks, f = check(logits, u, t, suppress=[i for i in range(V) if i != one], **kw)
        assert toks == [one, one]
        if t > 0:
            assert torch.isfinite(f).sum(1).tolist() == [1, 1]
    x = grid_row(3072, 7)
    logits = torch.stack([x, x.flip(0)])
    seen = [[i for i in range(3072) if i % 3 == 0], [i for i in range(3072) if i % 2 == 1]]
    for b, row in enumerate(logits):
        s = row[seen[b]]
        assert bool((s < 0).any()) and bool((s > 0).any()) and bool((torch.signbit(s) & (s == 0)).any()) and bool((~torch.signbit(s) & (s == 0)).any())
    u = torch.rand(2, generator=g)
    for t, kw in ((0.9, dict(top_k=50)), (0.9, dict(top_k=200, min_p=0.05)), (0.0, {})):
        check(logits, u if t > 0 else None, t, rep=1.3, seen=seen, seen_pad=37, **kw)
    # An all -inf row has no reference answer (the oracle finds no live token).  The kernel draws token 0 on every path and
    # returns without hanging; the filtered row stays -inf.
    for t, kw in ((0.9, dict(top_k=50)), (0.9, dict(top_p=0.9)), (0.9, {}), (0.0, {})):
        toks, f = run(torch.randn(2, 2048, generator=g), torch.tensor([0.3, U_LAST]), t, suppress=list(range(2048)), **kw)
        assert toks == [0, 0]
        if t > 0:
            assert bool(torch.isinf(f).all()) and bool((f < 0).all())


@pytest.mark.gpu
@pytest.mark.parametrize("temperature", [0.0, 0.9])
def test_frame_loop_arguments(temperature):
    """The talker draw as the Qwen3-TTS frame loop makes it (suppress, penalty, mark_seen, finished / eos, out = column 0 of
    the [B, 16] code matrix), then a code-predictor draw into column 1: a finished row emits eos and marks nothing, a row that
    draws eos becomes finished and marks nothing, every other row marks exactly its token, other columns stay untouched."""
    from mlx_audio_b200 import ops
    dev = _dev()
    B, V, eos = 5, 3072, 2150
    g = torch.Generator().manual_seed(12)
    suppress = [i for i in range(V - 1024, V) if i != eos]
    logits = torch.randn(B, V, generator=g) * 2.5
    logits[3, eos] = 30.0                                                # row 3 draws eos
    seen = [torch.randint(0, 2048, (40,), generator=g).tolist() for _ in range(B)]
    u = torch.rand(B, generator=g)
    want, _ = expect(logits, u, temperature, top_k=50, rep=1.05, seen=seen, suppress=suppress)
    assert want[3] == eos and eos not in (want[0], want[2], want[4])
    codes = torch.full((B, 16), -7, dtype=torch.int64, device=dev)
    fin = torch.tensor([0, 1, 0, 0, 0], dtype=torch.uint8, device=dev)
    seen_d = seen_rows(V, seen).to(dev)
    before = seen_d.cpu().clone()
    ops.sample_token(logits.to(dev), temperature=temperature, top_k=50, top_p=1.0, u=u.to(dev), suppress_mask=mask_of(V, suppress).to(dev),
                     seen=seen_d, repetition_penalty=1.05, mark_seen=True, out=codes[:, 0], finished=fin, eos=eos)
    got = codes.cpu()
    assert got[:, 0].tolist() == [want[0], eos, want[2], eos, want[4]]
    assert fin.cpu().tolist() == [0, 1, 0, 1, 0]
    after = before.clone()
    for b in (0, 2, 4):
        after[b, want[b]] = 1
    assert torch.equal(seen_d.cpu(), after)
    assert bool((got[:, 1:] == -7).all())
    lg = torch.randn(B, 2048, generator=g) * 2.5
    u2 = torch.rand(B, generator=g)
    want2, _ = expect(lg, u2, temperature, top_k=50)
    ops.sample_token(lg.to(dev), temperature=temperature, top_k=50, top_p=1.0, u=u2.to(dev), out=codes[:, 1])
    got2 = codes.cpu()
    assert got2[:, 1].tolist() == want2 and torch.equal(got2[:, 0], got[:, 0]) and bool((got2[:, 2:] == -7).all())


@pytest.mark.gpu
def test_argument_checks():
    from mlx_audio_b200 import ops
    dev = _dev()
    u = torch.full((2,), 0.5, device=dev)
    with pytest.raises(NotImplementedError, match="vocab 4097"):
        ops.sample_token(torch.zeros(2, 4097, device=dev), temperature=0.9, top_k=50, u=u)
    for min_p in (-0.1, 1.5):
        with pytest.raises(ValueError, match="min_p"):
            ops.sample_token(torch.zeros(2, 64, device=dev), temperature=0.9, min_p=min_p, u=u)
    with pytest.raises(ValueError, match="uniform"):
        ops.sample_token(torch.zeros(2, 64, device=dev), temperature=0.9, top_k=5)


# ------------------------------------------------------------------------------------------------ GPU: Whisper step, embed_sum
@pytest.mark.gpu
@pytest.mark.parametrize("t", [0.5, 1.0])
def test_whisper_step_sampled_matches_oracle(t):
    """b2a_whisper_greedy_step at temperature > 0 vs OW.apply_filters + OW.sample_update on every crafted history: equal
    tokens, sum_logprobs (un-tempered) within 2e-4, equal not_done counts; the eot row keeps eot and its sum."""
    from mlx_audio_b200 import ops
    dev = _dev()
    spec = OW.TokenizerSpec()
    V, tb = 51865, spec.timestamp_begin
    sup = torch.zeros(V)
    sup[list(WHISPER_SUPPRESS)] = float("-inf")
    blank = torch.zeros(V)
    blank[list(spec.blank_ids) + [spec.eot]] = float("-inf")
    for i, (scale, boost) in enumerate(((3.0, 0.0), (3.0, 6.0), (0.01, 0.0))):
        for j, h in enumerate(whisper_hist(spec)):
            logits, u, f, alive = whisper_case(h, scale, boost, t, seed=10 * i + j)
            slp0 = torch.tensor([-0.5, -1.25, -2.0], dtype=torch.float64)
            # A row the filters mask completely has no reference draw.  The kernel gives it what the greedy step gives: token 0
            # (the argmax of an all -inf row) and a NaN log-probability; an eot row keeps eot and its sum either way.
            ref_tok = [spec.eot if h[-1] == spec.eot else 0] * 3
            ref_lp = torch.where(torch.tensor(h[-1] == spec.eot), slp0, torch.full_like(slp0, math.nan))
            lr = [b for b in range(3) if alive[b]]
            if lr:
                rt, _, rl = OW.sample_update([h] * len(lr), f[lr], slp0[lr], spec.eot, t, u[lr].double())
                for k, b in enumerate(lr):
                    ref_tok[b], ref_lp[b] = rt[k][-1], rl[k]
            tokens = torch.zeros(3, 64, dtype=torch.int64)
            tokens[:, :len(h)] = torch.tensor(h)
            slp = slp0.float().to(dev)
            nd = torch.zeros(1, dtype=torch.int32, device=dev)
            nxt = ops.whisper_greedy_step(logits.to(dev), tokens.to(dev), len(h), WHISPER_SB, suppress_mask=sup.to(dev),
                                          blank_mask=blank.to(dev), eot=spec.eot, no_timestamps=spec.no_timestamps, timestamp_begin=tb,
                                          max_initial_ts=WHISPER_MAX_TS, without_timestamps=False, sum_logprobs=slp, not_done=nd,
                                          temperature=t, u=u.to(dev))
            assert nxt.cpu().tolist() == ref_tok, (h, scale, boost)
            assert torch.allclose(slp.cpu().double(), ref_lp, atol=2e-4, equal_nan=True), (h, slp, ref_lp)
            assert int(nd.item()) == sum(r != spec.eot for r in ref_tok)
            if h[-1] == spec.eot:
                assert ref_tok == [spec.eot] * 3 and torch.equal(slp.cpu(), slp0.float())
            else:                                                        # u = 0: first live token; u = 1 - 2^-24: last live token
                for b, end in ((0, 0), (2, -1)):
                    if alive[b]:
                        assert ref_tok[b] == int(torch.isfinite(f[b]).nonzero().flatten()[end])


@pytest.mark.gpu
def test_embed_sum_matches_float64_sum():
    """b2a_embed_sum vs a float64 sum of the table rows (bound: n * 2^-24 * sum |terms| for n float32 additions): pad only; no
    base; per-row trailing indices with the clamp-pad rule and only unfinished rows advancing; codes -1 and ``bins`` flag ``err``
    and are skipped; G = 0; trailing text without per-row indices is refused."""
    from mlx_audio_b200 import ops
    dev = _dev()
    g = torch.Generator().manual_seed(4)
    B, dim, n_text, bins = 4, 300, 5, (3072, 2048, 2048, 2048)
    tabs = [torch.randn(n, dim, generator=g) for n in bins]
    T = ops.EmbedTables([t.to(dev) for t in tabs])
    T0 = ops.EmbedTables([tabs[0].to(dev)])
    codes = torch.stack([torch.randint(0, n, (B,), generator=g) for n in bins], 1)
    codes[0, 0], codes[1, 3], codes[2, 1] = bins[0] - 1, bins[3] - 1, 0
    text_full = torch.randn(B, n_text + 2, dim, generator=g)
    text = text_full[:, 1:n_text + 1]                                    # strided: row stride (n_text + 2) * dim
    pad = torch.randn(dim, generator=g)
    text_d = text_full.to(dev)[:, 1:n_text + 1]
    pad_d = pad.to(dev)
    err = torch.zeros(1, dtype=torch.int32, device=dev)

    def want(cd, base):
        terms = [base.double()] + [torch.stack([tabs[gi][int(cd[b, gi])] if 0 <= int(cd[b, gi]) < bins[gi] else torch.zeros(dim)
                                                for b in range(B)]).double() for gi in range(cd.shape[1])]
        return sum(terms), len(terms) * 2.0 ** -24 * sum(t.abs() for t in terms)

    def call_and_check(cols, base, tabs_d, cd=codes, **kw):
        out_full = torch.full((B, 2, dim), 7.0, device=dev)          # out: row stride 2 * dim, as the frame loop's input rows
        ops.embed_sum(cd.to(dev)[:, cols], tabs_d, out=out_full[:, 0], err=err, **kw)
        ref, tol = want(cd[:, cols], base)
        got = out_full[:, 0].cpu().double()
        assert bool(((got - ref).abs() <= tol + 1e-30).all()) and bool((out_full[:, 1] == 7.0).all())

    every = slice(None)
    call_and_check(every, pad.expand(B, dim), T, pad=pad_d)
    call_and_check(slice(0, 1), torch.zeros(B, dim), T0)                # one column of the [B, 4] codes (row stride 4)
    call_and_check(slice(0, 0), text[:, 2], T, text=text_d, pad=pad_d, tidx=torch.full((B,), 2, dtype=torch.int32, device=dev))
    assert int(err.item()) == 0
    with pytest.raises(ValueError, match="tidx"):
        ops.embed_sum(codes.to(dev), T, text=text_d, pad=pad_d)
    tidx0 = [0, n_text - 2, n_text - 1, n_text + 3]
    tidx = torch.tensor(tidx0, dtype=torch.int32, device=dev)
    fin = torch.tensor([0, 1, 0, 1], dtype=torch.uint8, device=dev)
    base = torch.stack([text[b, i] if i < n_text - 1 else pad for b, i in enumerate(tidx0)])
    call_and_check(every, base, T, text=text_d, pad=pad_d, tidx=tidx, finished=fin)
    assert tidx.cpu().tolist() == [1, n_text - 2, n_text, n_text + 3] and int(err.item()) == 0
    bad = codes.clone()
    bad[1, 2], bad[3, 0] = -1, bins[0]
    call_and_check(every, pad.expand(B, dim), T, cd=bad, pad=pad_d)
    assert int(err.item()) == 1
