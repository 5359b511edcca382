"""EnCodec on the GPU at the released widths with synthetic float32 weights: the LSTM recurrence kernel against float64, the 24 kHz and
48 kHz models against oracle/encodec.py, batching, and Vocos with an EnCodec model attached."""
import numpy as np
import pytest
import torch

from mlx_audio_b200 import configs, ops, synth
from oracle import encodec as OE
from oracle import vocos as OV

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _rel_rms(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    assert a.shape == b.shape, (a.shape, b.shape)
    return float(((a - b) ** 2).mean().sqrt() / (b ** 2).mean().sqrt())


@pytest.fixture(scope="module")
def m24():
    from mlx_audio_b200.codec import Encodec
    P = synth.encodec_weights(configs.ENCODEC_24K)
    return Encodec(configs.ENCODEC_24K).load_weights(P), P


@pytest.fixture(scope="module")
def m48():
    from mlx_audio_b200.codec import Encodec
    P = synth.encodec_weights(configs.ENCODEC_48K, seed=16)
    return Encodec(configs.ENCODEC_48K).load_weights(P), P


def _audio(n, c=1, b=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64) / 24000
    x = 0.1 * torch.randn(b, n, c, generator=g, dtype=torch.float64) + 0.3 * torch.sin(2 * np.pi * 220 * t)[None, :, None]
    return x.float()


def _lstm_ref(xp, wh):
    R, T, G = xp.shape
    H = G // 4
    h = torch.zeros(R, H, dtype=torch.float64)
    c = torch.zeros_like(h)
    out = []
    for t in range(T):
        g = xp[:, t] + h @ wh.T
        i, f, gg, o = torch.sigmoid(g[:, :H]), torch.sigmoid(g[:, H:2 * H]), torch.tanh(g[:, 2 * H:3 * H]), torch.sigmoid(g[:, 3 * H:])
        c = f * c + i * gg
        h = o * torch.tanh(c)
        out.append(h)
    return torch.stack(out, 1)


@pytest.mark.parametrize("R,T,layers", [(1, 1500, 1), (1, 600, 2), (3, 400, 2), (16, 200, 1)])
def test_lstm_kernel_against_float64(R, T, layers):
    H = 512
    g = torch.Generator().manual_seed(R * 1000 + T)
    x = torch.randn(R, T, H, generator=g, dtype=torch.float64)
    err = torch.zeros(1, device=DEV, dtype=torch.int32)
    h_gpu, h_ref = x.float().to(DEV), x
    for j in range(layers):
        wx = 0.5 / np.sqrt(H) * torch.randn(4 * H, H, generator=g, dtype=torch.float64)
        wh = 0.5 / np.sqrt(H) * torch.randn(4 * H, H, generator=g, dtype=torch.float64)
        b = 0.1 * torch.randn(4 * H, generator=g, dtype=torch.float64)
        last = j == layers - 1
        xp = h_gpu.double().cpu() @ wx.T + b                                 # the kernel's input, formed in float64 from its own output
        h_gpu = ops.encodec_lstm(xp.float().to(DEV).contiguous(), wh.float().to(DEV).contiguous(), err,
                                 skip=x.float().to(DEV).contiguous() if last else None)
        h_ref = _lstm_ref(h_ref @ wx.T + b, wh) + (x if last else 0)
        if R == 1 or last:
            scale = float(h_ref.abs().max())
            e = float((h_gpu.double().cpu() - h_ref).abs().max())
            assert e <= 2e-5 * scale, (j, e, scale)
        if R > 1:                                                            # every row is its own R = 1 run, bit for bit
            for r in range(R):
                one = ops.encodec_lstm(xp[r:r + 1].float().to(DEV).contiguous(), wh.float().to(DEV).contiguous(), err,
                                       skip=x[r:r + 1].float().to(DEV).contiguous() if last else None)
                assert torch.equal(one, h_gpu[r:r + 1]), (j, r)
    torch.cuda.synchronize()
    assert int(err.item()) == 0


def _margin_ok(P, emb, nq):
    _, m = OE.quantize(P, emb, nq, with_margin=True)
    return m > 1e-5


def test_24khz_encoder_codes_decoder(m24):
    model, P = m24
    cfg = configs.ENCODEC_24K
    x = _audio(240_000)
    emb_ref = OE.encoder(P, x.double(), cfg)
    emb = model.encode_latent(x.to(DEV))
    assert float((emb.double().cpu() - emb_ref).abs().max()) <= 2e-4 * float(emb_ref.abs().max())
    for bw in (1.5, 6.0, 24.0):
        codes, scales = model.encode(x.to(DEV), bandwidth=bw)
        nq = OE.num_quantizers_for_bandwidth(cfg, bw)
        assert codes.shape == (1, 1, nq, 750) and scales == [None]
        ref = OE.quantize(P, emb_ref, nq)
        ok = _margin_ok(P, emb_ref, nq)[0]
        assert ok.float().mean() > 0.5, float(ok.float().mean())
        assert torch.equal(codes[0, 0][:, ok].cpu(), ref[0][:, ok]), bw
    y = model.decode(codes, scales)
    y_ref = OE.decode(P, codes.cpu(), scales, cfg)
    assert y.shape == (1, 240_000, 1)
    assert _rel_rms(y, y_ref) <= 1e-3


def test_24khz_reference_shape_pins(m24):
    """codec/tests/test_encodec.py: zeros [1, 120000, 1]."""
    model, _ = m24
    x = torch.zeros(1, 120_000, 1, device=DEV)
    for bw, nq in ((None, 2), (6.0, 8)):
        codes, scales = model.encode(x, bandwidth=bw)
        assert tuple(codes.shape) == (1, 1, nq, 375)
        assert tuple(model.decode(codes, scales).shape) == (1, 120_000, 1)


def test_batch_rows_equal_single_rows(m24, m48):
    model, _ = m24
    x = _audio(48_000, b=3, seed=3).to(DEV)
    codes, _ = model.encode(x, bandwidth=6.0)
    for b in range(3):
        one, _ = model.encode(x[b:b + 1], bandwidth=6.0)
        assert torch.equal(one[:, 0], codes[:, b])
        assert torch.equal(model.decode_frames(codes[0, b:b + 1]), model.decode_frames(codes[0])[b:b + 1])
    model48, _ = m48
    x = _audio(100_000, c=2, b=2, seed=4)
    inp, mask = OE.preprocess_audio([x[0], x[1, :90_000]], 48000, model48.chunk_length, model48.chunk_stride)
    inp, mask = inp.float().to(DEV), mask.to(DEV)
    codes, scales = model48.encode(inp, mask, bandwidth=6.0)
    y = model48.decode(codes, scales, mask)
    for b in range(2):
        c1, s1 = model48.encode(inp[b:b + 1], mask[b:b + 1], bandwidth=6.0)
        assert torch.equal(c1[:, 0], codes[:, b])
        assert torch.equal(model48.decode(c1, s1, mask[b:b + 1]), y[b:b + 1])


def test_48khz_chunked_stereo(m48):
    model, P = m48
    cfg = configs.ENCODEC_48K
    x = _audio(100_000, c=2, seed=5)
    inp, mask = OE.preprocess_audio([x[0]], 48000, model.chunk_length, model.chunk_stride)
    assert inp.shape[1] == 143_040
    codes, scales = model.encode(inp.float().to(DEV), mask.to(DEV), bandwidth=12.0)
    assert codes.shape == (3, 1, 8, 150)
    # the batched chunks give the codes of chunk-by-chunk encoding
    offsets, cl = OE.chunk_offsets(cfg, inp.shape[1])
    for k, o in enumerate(offsets):
        ck, sk = model.encode_frames(inp[:, o:o + cl].float().to(DEV).contiguous(), mask[:, o:o + cl].to(DEV).contiguous(), 8)
        assert torch.equal(ck, codes[k])
        assert torch.equal(sk.reshape(1, 1, 1), scales[k])
    ref_codes, ref_scales, ref_embs = OE.encode(P, inp, cfg, mask, bandwidth=12.0, return_embeddings=True)
    for k in range(3):
        s, r = float(scales[k]), float(ref_scales[k])
        assert abs(s - r) <= 1e-6 * r, (k, s, r)
        ok = _margin_ok(P, ref_embs[k], 8)[0]
        assert torch.equal(codes[k, 0][:, ok].cpu(), ref_codes[k, 0][:, ok])
    y = model.decode(codes, scales, mask)
    y_ref = OE.decode(P, codes.cpu(), [s.double().cpu() for s in scales], cfg, mask)
    assert y.shape == y_ref.shape == (1, 143_040, 2)
    mask100 = mask[:, :100_000]
    y2 = model.decode(codes, scales, mask100)
    assert y2.shape == (1, 100_000, 2) and torch.equal(y2, y[:, :100_000])
    assert _rel_rms(y, y_ref) <= 1e-3


def test_vocos_with_encodec_attached(m24):
    from mlx_audio_b200.codec import Vocos
    model, P = m24
    cfg = OV.CONFIG_ENCODEC
    voc = Vocos.from_hparams(cfg, encodec=model)
    PV = synth.vocos_weights(cfg)
    voc.load_weights(PV)
    x = _audio(48_000)[0, :, 0]
    for k in (0, 2):
        cond = [float(k)] * 4
        codes = voc.get_encodec_codes(x, [k])
        nq = OE.num_quantizers_for_bandwidth(configs.ENCODEC_24K, cfg["feature_extractor"]["init_args"]["bandwidths"][k])
        assert codes.shape == (nq, 1, 150)
        feats_ref = OE.dequantize(P, codes.permute(1, 0, 2).cpu())
        wave_ref = OV.decode(PV, feats_ref, cfg, torch.tensor([cond], dtype=torch.float64))[0]
        wave = voc(x, bandwidth_id=cond)
        assert _rel_rms(wave, wave_ref) <= 1e-3
        assert _rel_rms(voc.decode_from_codes(codes, bandwidth_id=cond), wave_ref) <= 1e-3
