"""Soprano on the GPU against the float64 oracle (oracle/soprano.py): the mlx-lm sampler kernel, the up-sampling kernel, the decoder at
the released geometry, the LM loop with graph replay and batching, and ``generate`` end to end from a local directory.  LM weights are
synthetic bf16 at the reference's test configuration (hidden 512, 8 / 4 heads of 64, intermediate 1024, 12 layers, vocabulary 32 000)."""
import json

import numpy as np
import pytest
import torch

from oracle import soprano as OS

pytestmark = pytest.mark.gpu
DEV = "cuda"
MARGIN = 1e-6
LM_MARGIN = 1e-3     # along the LM loop the kernel sees logits from fp32 activations and bf16 weights, not the oracle's float64 ones


def _model(decoder=None, layers=12, device=DEV):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.soprano import DecoderConfig, Model, ModelConfig
    cfg = dict(synth.SOPRANO_LM, num_hidden_layers=layers)
    dc = DecoderConfig(**(decoder or {}))
    m = Model(ModelConfig.from_dict({**cfg, "decoder_config": dc}), device=device)
    P = synth.soprano_weights(m)
    m.load_weights(list(P.items()))
    m._stop_token_id = 1
    return m, P, cfg


@pytest.fixture(scope="module")
def lm():
    return _model({"decoder_num_layers": 2, "decoder_dim": 128, "decoder_intermediate_dim": 256})


def _rows(V, n, seed):
    g = torch.Generator().manual_seed(seed)
    scale = torch.tensor([1.0, 3.0, 6.0, 12.0, 30.0, 0.3, 8.0, 90.0])[torch.arange(n) % 8]
    x = torch.randn(n, V, generator=g) * scale[:, None] - torch.tensor([4.0, 8.0, 20.0, 2.0, 0.0, 0.0, 40.0, 0.0])[torch.arange(n) % 8, None]
    return x.float()


@pytest.mark.parametrize("V", [4097, 32000, 151936])
@pytest.mark.parametrize("temperature,top_p", [(0.3, 0.95), (1.0, 0.5), (0.7, 0.999), (0.3, 1.0), (0.5, 0.0), (0.0, 0.95)])
def test_sampler_matches_float64(V, temperature, top_p):
    from mlx_audio_b200 import ops
    x = _rows(V, 8, V + int(100 * top_p))
    u = torch.rand(8, 3, generator=torch.Generator().manual_seed(5))
    step = torch.tensor([1], dtype=torch.int32, device=DEV)
    tok = ops.lm_sample_mlx(x.to(DEV), temperature=temperature, top_p=top_p, u=u.to(DEV), step_dev=step).cpu()
    checked = 0
    for b in range(8):
        ref, _, _ = OS.sample(x[b].numpy(), float(u[b, 1]), temperature, top_p)
        mk, md = OS.sample_margins(x[b].numpy(), float(u[b, 1]), temperature, top_p)
        if mk > MARGIN and md > MARGIN:
            assert int(tok[b]) == ref, (b, int(tok[b]), ref)
            checked += 1
    assert checked >= 6
    for b in range(8):                                                   # each row alone: the same token
        one = ops.lm_sample_mlx(x[b:b + 1].to(DEV), temperature=temperature, top_p=top_p, u=u[b:b + 1].to(DEV), step_dev=step).cpu()
        assert int(one[0]) == int(tok[b])


def test_sampler_edges():
    from mlx_audio_b200 import ops
    V = 32000
    x = torch.randn(4, V) * 2
    x[:, 17] = x[:, 900] = x.max() + 1                                   # argmax tie: first index
    assert ops.lm_sample_mlx(x.to(DEV), temperature=0.0, top_p=0.95).cpu().tolist() == [17] * 4
    # an exp that overflows keeps every token from its rank up; large logits filter nothing
    big = torch.randn(2, V) * 3 + 100.0
    u = torch.rand(2, 1)
    for top_p in (0.5, 0.95):
        got = ops.lm_sample_mlx(big.to(DEV), temperature=1.0, top_p=top_p, u=u.to(DEV)).cpu()
        for b in range(2):
            assert OS.keep_mask(big[b].numpy(), top_p).all()
            assert int(got[b]) == OS.sample(big[b].numpy(), float(u[b, 0]), 1.0, top_p)[0]
    # top_p 0 or 1: no filter -> same as the unfiltered draw
    a = ops.lm_sample_mlx(x.to(DEV), temperature=0.8, top_p=0.0, u=u[:1].expand(4, 1).contiguous().to(DEV)).cpu()
    b_ = ops.lm_sample_mlx(x.to(DEV), temperature=0.8, top_p=1.0, u=u[:1].expand(4, 1).contiguous().to(DEV)).cpu()
    assert a.tolist() == b_.tolist()
    # every exp-sum under 1 - top_p: nothing kept -> token 0
    tiny = torch.full((1, 4097), -30.0)
    assert int(ops.lm_sample_mlx(tiny.to(DEV), temperature=1.0, top_p=0.9, u=u[:1].to(DEV))[0]) == 0
    # finished rows write nothing; a stop id marks the row finished; history at the step
    g = torch.zeros(3, 64)
    g[0, 5] = g[1, 7] = g[2, 9] = 10.0
    out = torch.full((3,), -5, dtype=torch.int64, device=DEV)
    hist = torch.full((3, 4), -5, dtype=torch.int64, device=DEV)
    fin = torch.tensor([0, 0, 1], dtype=torch.uint8, device=DEV)
    step = torch.tensor([2], dtype=torch.int32, device=DEV)
    ops.lm_sample_mlx(g.to(DEV), temperature=0.0, top_p=1.0, step_dev=step, out=out, hist=hist, finished=fin, stop_ids=(7, 99))
    assert out.cpu().tolist() == [5, 7, -5] and fin.cpu().tolist() == [0, 1, 1]
    assert hist[:, 2].cpu().tolist() == [5, 7, -5] and (hist[:, [0, 1, 3]] == -5).all()


@pytest.mark.parametrize("L", [1, 2, 5, 33])
def test_upsample_bit_exact(L):
    from mlx_audio_b200 import ops
    x = torch.randn(2, L, 512)
    Lo = 4 * (L - 1) + 1
    if L == 1:
        ref = x.expand(2, Lo, 512)
    else:
        pos = torch.arange(Lo, dtype=torch.float32) * torch.tensor((L - 1) / (Lo - 1), dtype=torch.float32)
        lo = torch.floor(pos).long()
        hi = torch.clamp(lo + 1, max=L - 1)
        f = pos - lo.float()
        ref = x[:, lo] * (1 - f)[None, :, None] + x[:, hi] * f[None, :, None]
    y = ops.soprano_upsample(x.to(DEV), 4).cpu()
    assert torch.equal(y, ref)
    cw = ops.pack_conv(torch.randn(64, 3, 512).bfloat16().float(), None, 1, DEV)
    pl = ops.soprano_upsample(x.to(DEV), 4, planes_for=cw)
    assert pl.hi.shape == (2, Lo, cw.cin_pad)
    assert torch.equal(pl.hi.float().cpu(), ref.bfloat16().float())
    if pl.lo is not None:
        assert torch.equal(pl.lo.float().cpu(), (ref - ref.bfloat16().float()).bfloat16().float())


@pytest.mark.parametrize("input_kernel", [1, 3])
def test_decoder_released_geometry(input_kernel):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.soprano import DecoderConfig, Model, ModelConfig
    dc = DecoderConfig(input_kernel=input_kernel)
    m = Model(ModelConfig.from_dict({**synth.SOPRANO_LM, "num_hidden_layers": 1, "decoder_config": dc}), device=DEV)
    P = synth.soprano_weights(m)
    m.load_weights(list(P.items()))
    cfg = OS.decoder_cfg(512, 768, 2304, 8, input_kernel, 3)
    for L in (1, 2, 5, 40):
        h = torch.randn(1, L, 512, generator=torch.Generator().manual_seed(L))
        y = m.decoder(h.to(DEV)).double().cpu()
        assert y.shape == (1, 2048 * (L - 1))
        if L > 1:
            ref = OS.decode(P, h.double().numpy(), cfg)
            err = float(torch.sqrt(((y - ref) ** 2).mean()) / torch.sqrt((ref ** 2).mean()))
            assert err < 1e-4, (L, err)


def test_lm_against_oracle_and_graph(lm):
    m, P, cfg = lm
    ids = [3, 17, 200, 4001, 9, 31999, 12]
    n = 64
    u = torch.rand(1, n, generator=torch.Generator().manual_seed(3))
    m._stop_token_id = None
    toks, hid = m.generate_from_ids([ids], temperature=0.3, top_p=0.95, max_tokens=n, u=u)
    toks_e, hid_e = m.generate_from_ids([ids], temperature=0.3, top_p=0.95, max_tokens=n, u=u, use_graph=False)
    assert torch.equal(toks[0], toks_e[0]) and torch.equal(hid[0], hid_e[0])        # graph replay == eager, bit for bit
    # teacher forcing: the oracle is fed the product's tokens, so all 64 hidden states are compared whatever the draw margins
    ref_h, ref_lg = OS.teacher_forced(P, ids, toks[0].tolist(), cfg)
    g = hid[0].double().cpu()
    assert g.shape == ref_h.shape == (n + 1, cfg["hidden_size"])
    err = float(torch.sqrt(((g - ref_h) ** 2).mean()) / torch.sqrt((ref_h ** 2).mean()))
    assert err < 1e-3, err
    # each token is the oracle's draw from the oracle's logits at that step wherever the draw margin exceeds LM_MARGIN (the keep-boundary
    # margin is not used: with 32 000 small exp terms the cumulative sum passes 1 - top_p in steps far below 1e-3, but the tokens at the
    # boundary carry exp(logit / 0.3) weights ~1e-20 of the kept mass, so moving the boundary cannot move the draw)
    checked = 0
    for i in range(n):
        x = ref_lg[i].float().numpy()
        _, md = OS.sample_margins(x, float(u[0, i]), 0.3, 0.95)
        if md > LM_MARGIN:
            assert int(toks[0][i]) == OS.sample(x, float(u[0, i]), 0.3, 0.95)[0], i
            checked += 1
    assert checked >= 48, checked
    m._stop_token_id = 1


def test_graphs_survive_batch_size_changes(lm):
    """Batch sizes 2, 3, 2, 1, 3 in turn (each reallocates the shared K/V cache): every graph-replayed call returns the bits of eager
    steps, so no replay touches a freed cache."""
    m, P, cfg = lm
    n = 20
    batches = {2: [[4, 5, 6, 7], [8, 9]], 3: [[10, 11, 12], [13, 14, 15, 16, 17], [18]], 1: [[19, 20, 21]]}
    hold = []                                                            # earlier results stay alive, as a caller's audio would
    for B in (2, 3, 2, 1, 3):
        u = torch.rand(B, n, generator=torch.Generator().manual_seed(B))
        tg, hg = m.generate_from_ids(batches[B], temperature=0.5, top_p=0.9, max_tokens=n, u=u)
        te, he = m.generate_from_ids(batches[B], temperature=0.5, top_p=0.9, max_tokens=n, u=u, use_graph=False)
        for b in range(B):
            assert torch.equal(tg[b], te[b]) and torch.equal(hg[b], he[b]), (B, b)
        hold.append(hg)


def test_istft_head_shape_pin():
    from mlx_audio.tts.models.soprano.decoder import ISTFTHead
    y = ISTFTHead(dim=16, n_fft=64, hop_length=16, device=DEV)(torch.randn(1, 5, 16))
    assert tuple(y.shape) == (1, 64)                                     # [1, hop (L - 1)], the reference keeps the batch axis


def test_batch_rows_match_alone(lm):
    m, P, cfg = lm
    rows = [[5, 6, 7, 8, 9, 10, 11, 12, 13], [40, 41, 42], [7, 7, 7, 7, 7, 100]]
    n = 24
    u = torch.rand(3, n, generator=torch.Generator().manual_seed(9))
    toks, hid = m.generate_from_ids(rows, temperature=0.3, top_p=0.95, max_tokens=n, u=u)
    for b in range(3):
        t1, h1 = m.generate_from_ids([rows[b]], temperature=0.3, top_p=0.95, max_tokens=n, u=u[b:b + 1])
        assert torch.equal(toks[b], t1[0]), b
        # the batched prefill runs on the tensor-core GEMM (B * P > 16 rows) and the attention sees left-pad keys masked to zero
        # weight, so hidden states agree to rounding, not bit for bit
        err = float((hid[b] - h1[0]).norm() / h1[0].norm())
        assert err < 1e-5, (b, err)


def test_stop_and_stream(lm):
    m, P, cfg = lm
    ids = [11, 12, 13, 14]
    u = torch.rand(1, 20, generator=torch.Generator().manual_seed(1))
    m._stop_token_id = None
    toks, _ = m.generate_from_ids([ids], temperature=0.3, top_p=0.95, max_tokens=20, u=u)
    assert toks[0].numel() == 20                                        # max_tokens hit
    stop = int(toks[0][5])
    first = int(torch.nonzero(toks[0] == stop)[0])
    m._stop_token_id = stop
    t2, h2 = m.generate_from_ids([ids], temperature=0.3, top_p=0.95, max_tokens=20, u=u)
    assert torch.equal(t2[0], toks[0][:first]) and h2[0].shape[0] == first + 1
    streamed = list(m.stream_generate(ids, max_tokens=20, temperature=0.3, top_p=0.95, u=u))
    assert streamed[0][0] is None and len(streamed) == first + 1
    assert [int(t[0, 0]) for t, _ in streamed[1:]] == t2[0].tolist()
    assert torch.equal(torch.cat([h for _, h in streamed], 1)[0], h2[0])
    m._stop_token_id = 1


def _write_dir(tmp_path, m, P, cfg, name):
    from safetensors.torch import save_file
    from tokenizers import Tokenizer, models, pre_tokenizers
    d = tmp_path / name
    d.mkdir()
    words = ["[UNK]", "[STOP]", "[TEXT]", "[START]"] + "hello world this is a test of the soprano model . , ! ? one two three".split()
    tk = Tokenizer(models.WordLevel({w: i for i, w in enumerate(words)}, unk_token="[UNK]"))
    tk.pre_tokenizer = pre_tokenizers.Whitespace()
    tk.add_special_tokens(["[STOP]", "[TEXT]", "[START]"])
    tk.save(str(d / "tokenizer.json"))
    (d / "tokenizer_config.json").write_text(json.dumps({"tokenizer_class": "PreTrainedTokenizerFast"}))
    dc = m.config.decoder_config
    (d / "config.json").write_text(json.dumps({**cfg, "decoder_config": {"decoder_num_layers": dc.decoder_num_layers, "decoder_dim": dc.decoder_dim,
                                                                         "decoder_intermediate_dim": dc.decoder_intermediate_dim}}))
    save_file({("model." + k[len("language_model."):] if k.startswith("language_model.") else k): v.contiguous() for k, v in P.items()},
              str(d / "model.safetensors"))
    return d


def test_generate_end_to_end(lm, tmp_path):
    from mlx_audio_b200.tts.models.soprano import Model
    m0, P, cfg = lm
    d = _write_dir(tmp_path, m0, P, cfg, "tiny-soprano")
    m = Model.from_pretrained(str(d), device=DEV)
    assert m._stop_token_id == 1 and m.config.decoder_config.decoder_dim == 128
    text = "hello world, this is a test of the soprano model. one two three!\nthis is a test."
    res = list(m.generate(text, max_tokens=12, seed=0))
    assert [r.segment_idx for r in res] == [0, 1]
    for r in res:
        assert r.sample_rate == 32000 and r.audio.dim() == 1 and r.samples == r.audio.shape[0]
        assert torch.isfinite(r.audio).all()
    # each sentence: 2048 (n - 1) samples for n hidden states
    sentences = m._preprocess_text(["this is a test."])
    _, hid = m.generate_from_ids([m._tokenize(p) for p, _, _ in sentences], max_tokens=12, seed=0)
    assert res[1].samples == 2048 * (hid[0].shape[0] - 1) and res[1].token_count == hid[0].shape[0]
    # the first sample is a stop id: one hidden state, an empty waveform
    first = int(m.generate_from_ids([m._tokenize(sentences[0][0])], max_tokens=12, seed=0)[0][0][0])
    m._stop_token_id = first
    r = list(m.generate("this is a test.", max_tokens=12, seed=0))[0]
    assert r.samples == 0 and r.token_count == 1


def test_generic_loader_resolves_soprano(lm, tmp_path):
    from mlx_audio_b200.tts.models.soprano import Model
    from mlx_audio_b200.utils import load_model
    m0, P, cfg = lm
    d = _write_dir(tmp_path, m0, P, cfg, "Soprano-1.1-80M-bf16")
    m = load_model(str(d))
    assert isinstance(m, Model) and m.config.decoder_config.decoder_dim == 128
    toks, hid = m.generate_from_ids([[2, 5, 6, 3]], max_tokens=4, seed=1)
    assert hid[0].shape[1] == 512
