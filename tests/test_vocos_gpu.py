"""Vocos on the GPU: the three kernels against float64, the whole vocoder against the oracle at released sizes, batch-row bits,
the from_pretrained round trip, the reference's shape pins and the edge cases."""
import numpy as np
import pytest
import torch

from oracle import vocos as OV

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _rel_rms(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return float(torch.sqrt(((a - b) ** 2).mean()) / torch.sqrt((b ** 2).mean()))


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("n", [513, 1000, 24_017, 240_000])
def test_logmel_kernel_against_float64(B, n):
    from mlx_audio_b200.codec.models.vocos import log_mel_spectrogram
    a = 0.2 * torch.randn(B, n, generator=torch.Generator().manual_seed(n + B), dtype=torch.float64)
    y = log_mel_spectrogram(a.float(), device=DEV).double().cpu()
    ref = OV.log_mel_spectrogram(a.float().double())
    assert y.shape == ref.shape == (B, n // 256, 100)
    m = torch.exp(ref) >= 1e-3
    assert m.float().mean() > 0.5
    err = float((y - ref).abs()[m].max())
    assert err <= 1e-4, err


def _dwnorm_ref(x, dw_w, dw_b, w, b, ada, eps=1e-6):
    x = x.double()
    if dw_w is not None:
        K, C = dw_w.shape
        y = torch.nn.functional.conv1d(x.transpose(1, 2), dw_w.double().t()[:, None, :], dw_b.double(), padding=K // 2, groups=C)
        x = y.transpose(1, 2)
    mu = x.mean(-1, keepdim=True)
    v = (x - mu) / torch.sqrt(((x - mu) ** 2).mean(-1, keepdim=True) + eps)
    if ada is not None:
        C = x.shape[-1]
        return v * ada[:, None, :C].double() + ada[:, None, C:].double()
    if w is not None:
        v = v * w.double()
    if b is not None:
        v = v + b.double()
    return v


@pytest.mark.parametrize("C", [384, 512, 768, 1024])
@pytest.mark.parametrize("K", [0, 7])
@pytest.mark.parametrize("mode", ["affine", "nobias", "ada"])
def test_dwnorm_against_float64(C, K, mode):
    from mlx_audio_b200 import ops
    g = torch.Generator().manual_seed(C + K)
    for L in (1, 2, 7, 129, 4096):
        B = 2
        x = (torch.randn(B, L, C, generator=g) + 0.5).to(DEV)
        dw = None
        if K:
            wd = torch.randn(C, K, 1, generator=g) / K ** 0.5
            dw = ops.pack_conv(wd, 0.1 * torch.randn(C, generator=g), C, DEV)
        w = (1 + 0.1 * torch.randn(C, generator=g)).to(DEV)
        b = None if mode == "nobias" else (0.1 * torch.randn(C, generator=g)).to(DEV)
        ada = None
        if mode == "ada":
            ada = torch.cat([1 + 0.3 * torch.randn(B, C, generator=g), 0.2 * torch.randn(B, C, generator=g)], 1).to(DEV)
            assert not torch.allclose(ada[0], ada[1])
        y, pl = ops.vocos_dwnorm(x, dw, None if ada is not None else w, None if ada is not None else b, ada=ada, fp32=True, planes=True)
        ref = _dwnorm_ref(x.cpu(), None if dw is None else dw.w.cpu(), None if dw is None else dw.bias.cpu(),
                          None if ada is not None else w.cpu(), None if ada is not None or b is None else b.cpu(),
                          None if ada is None else ada.cpu())
        scale = ref.abs().amax(-1, keepdim=True)
        err = float(((y.double().cpu() - ref).abs() / scale).max())
        assert err <= 1e-5, (L, err)
        hl = pl.hi.float() + pl.lo.float()
        assert float(((hl - y).abs() / y.abs().amax(-1, keepdim=True)).max()) <= 2.0 ** -16, L
        y2 = ops.vocos_dwnorm(x, dw, None if ada is not None else w, None if ada is not None else b, ada=ada)
        assert torch.equal(y, y2)
        if B > 1:
            y1 = ops.vocos_dwnorm(x[1:].contiguous(), dw, None if ada is not None else w, None if ada is not None else b,
                                  ada=None if ada is None else ada[1:].contiguous())
            assert torch.equal(y1[0], y[1])


@pytest.mark.parametrize("n_fft,hop", [(1024, 256), (1280, 320)])
@pytest.mark.parametrize("T,gain,offset", [(2, 1.0, -0.5), (5, 1.0, -0.5), (937, 1.0, -0.5), (40, 12.0, 1.0)])
def test_head_kernel_against_float64(n_fft, hop, T, gain, offset):
    from mlx_audio_b200 import ops
    from mlx_audio_b200.codec.models.vocos import hanning
    g = torch.Generator().manual_seed(T + n_fft)
    ld = -(-(n_fft + 2) // 64) * 64
    h = torch.zeros(2, T, ld)
    nb = n_fft // 2 + 1
    h[..., :nb] = gain * torch.randn(2, T, nb, generator=g) + offset
    h[..., nb:2 * nb] = 3.0 * torch.randn(2, T, nb, generator=g)
    h[..., 2 * nb:] = 1e3                                                  # pad columns: must be ignored
    y = ops.vocos_istft_head(h.to(DEV), n_fft, hop, torch.from_numpy(hanning(n_fft)).float().to(DEV))
    S, clipped = OV.spectrum(h, n_fft)
    if gain > 1:
        assert clipped >= 0.3, clipped
    ref = OV.istft(S, n_fft, hop)
    assert y.shape == ref.shape == (2, (T - 1) * hop)
    err = _rel_rms(y, ref)
    assert err <= 1e-5, err


def _model(cfg, seed=11):
    from mlx_audio_b200 import synth
    from mlx_audio_b200.codec import Vocos
    P = synth.vocos_weights(cfg, seed)
    return Vocos.from_hparams(cfg, device=DEV).load_weights(P), P


def test_released_mel_model_against_the_oracle():
    m, P = _model(OV.CONFIG_MEL)
    a = 0.3 * torch.randn(240_000, generator=torch.Generator().manual_seed(3))
    y = m(a)
    ref = OV.forward(P, a.double(), OV.CONFIG_MEL)[0]
    assert y.shape == ref.shape == (239_616,)
    err = _rel_rms(y, ref)
    print("mel model relative RMS", err)
    assert err <= 1e-3, err
    mel = m.feature_extractor(a)
    assert torch.equal(m.decode(mel), y)                                  # Vocos(audio) == decode(log_mel_spectrogram(audio))


def test_encodec_shaped_adaln_decode_against_the_oracle():
    m, P = _model(OV.CONFIG_ENCODEC)
    g = torch.Generator().manual_seed(4)
    feats = torch.randn(1, 375, 128, generator=g)
    cond = torch.tensor([[3.0, 3.0, 3.0, 3.0]])
    y = m.decode(feats, bandwidth_id=cond)
    hb = OV.backbone(P, feats.double(), OV.CONFIG_ENCODEC, cond)
    _, clipped = OV.head_spectrum(P, hb, 1280)
    assert clipped < 0.01, clipped
    ref = OV.head(P, hb, 1280, 320)[0]
    assert y.shape == ref.shape == (119_680,)
    err = _rel_rms(y, ref)
    print("EnCodec-config decode relative RMS", err, "clipped", clipped)
    assert err <= 1e-3, err
    with pytest.raises(ValueError):
        m.decode(feats)                                                   # AdaLN needs bandwidth_id


@pytest.mark.parametrize("cfg", [OV.CONFIG_MEL, OV.CONFIG_ENCODEC], ids=["mel", "encodec"])
def test_batch_rows_equal_single_rows(cfg):
    m, _ = _model(cfg)
    C = cfg["backbone"]["init_args"]["input_channels"]
    feats = torch.randn(2, 200, C, generator=torch.Generator().manual_seed(5))
    kw0, kw1, kwb = {}, {}, {}
    if "adanorm_num_embeddings" in cfg["backbone"]["init_args"]:
        cond = torch.tensor([[3.0, 3.0, 3.0, 3.0], [0.0, 1.0, 2.0, 0.5]])
        kw0, kw1, kwb = {"bandwidth_id": cond[:1]}, {"bandwidth_id": cond[1:]}, {"bandwidth_id": cond}
    yb = m.decode(feats, **kwb)
    assert yb.shape[0] == 2 and not torch.equal(yb[0], yb[1])
    assert torch.equal(m.decode(feats[:1], **kw0), yb[0]) and torch.equal(m.decode(feats[1:], **kw1), yb[1])
    if not kwb:
        a = 0.3 * torch.randn(2, 30_000, generator=torch.Generator().manual_seed(6))
        ya = m(a)
        assert torch.equal(m(a[1]), ya[1])


def test_from_pretrained_round_trip(tmp_path):
    import yaml
    from safetensors.torch import save_file
    from mlx_audio_b200.codec import Vocos
    m, P = _model(OV.CONFIG_MEL)
    torch_layout = {k: (v.transpose(1, 2).contiguous() if ("backbone.embed" in k or "dwconv" in k) and k.endswith(".weight") else v.contiguous())
                    for k, v in P.items()}
    torch_layout["feature_extractor.mel_spec.spectrogram.window"] = torch.ones(1024)
    torch_layout["head.istft.window"] = torch.ones(1024)
    save_file(torch_layout, str(tmp_path / "model.safetensors"))
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(OV.CONFIG_MEL))
    m2 = Vocos.from_pretrained(str(tmp_path), device=DEV)
    a = 0.3 * torch.randn(20_000, generator=torch.Generator().manual_seed(7))
    assert torch.equal(m(a), m2(a))


def test_reference_shape_pins_and_edges():
    from mlx_audio_b200 import ops
    from mlx_audio_b200.codec import Vocos
    m = Vocos.from_hparams(OV.CONFIG_MEL, device=DEV)                     # random weights on first use
    assert m(torch.zeros(120_000)).shape == (119_552,)
    e = Vocos.from_hparams(OV.CONFIG_ENCODEC, device=DEV)
    assert e.decode(torch.zeros(1, 375, 128), bandwidth_id=torch.tensor([[3, 3, 3, 3]])).shape == (119_680,)
    with pytest.raises(ValueError):
        m(torch.zeros(512))
    assert m(torch.randn(513)).shape == (256,)
    n0 = ops.LAUNCHES[0]
    y = m.decode(torch.randn(1, 1, 100))
    assert y.shape == (0,)
    y = m.decode(torch.randn(3, 1, 100))
    assert y.shape == (3, 0)
    assert ops.LAUNCHES[0] > n0
