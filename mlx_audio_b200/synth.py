"""Synthetic (random-init) checkpoints at the reference's real config shapes.

There is no network and no weights on disk (SURVEY.md section 0), so parity and the bench
run on random weights whose NAMES and SHAPES are the reference's MLX parameter tree
(post-``sanitize``): the same dict feeds the CPU oracle and the CUDA product.
Recipe (SURVEY.md section 8d, cfg2): N(0, 0.02) everywhere, norm gains 1 / biases 0,
weight-norm ``g = ||v||``, Snake alpha 1, values rounded to bf16 (a "bf16 checkpoint"),
returned as float32 tensors holding bf16-exact values.
"""
from __future__ import annotations

import math

import torch


def _bf16(x):
    return x.to(torch.bfloat16).to(torch.float32)


class _Gen:
    def __init__(self, seed, std=0.02):
        self.g = torch.Generator().manual_seed(seed)
        self.std = std
        self.P = {}

    def normal(self, name, *shape, std=None):
        self.P[name] = _bf16(torch.randn(*shape, generator=self.g) * (self.std if std is None else std))
        return self.P[name]

    def const(self, name, value, *shape):
        self.P[name] = torch.full(shape, float(value))

    def linear(self, pre, out_f, in_f, bias=True, std=None):
        self.normal(pre + ".weight", out_f, in_f, std=std)
        if bias:
            self.normal(pre + ".bias", out_f, std=std)

    def layer_norm(self, pre, c):
        self.const(pre + ".weight", 1.0, c)
        self.const(pre + ".bias", 0.0, c)

    def conv_weighted(self, pre, out_c, k, in_c, bias_c=None, bias=True):
        """ConvWeighted params (kokoro/istftnet.py:96-126): weight_v [out,K,in], weight_g [out,1,1] = ||v||."""
        v = self.normal(pre + ".weight_v", out_c, k, in_c)
        self.P[pre + ".weight_g"] = _bf16(torch.sqrt((v * v).sum(dim=(1, 2), keepdim=True)))
        if bias:
            self.normal(pre + ".bias", out_c if bias_c is None else bias_c)

    def lstm(self, pre, in_f, hid):
        for d in ("forward", "backward"):
            self.normal(f"{pre}.Wx_{d}", 4 * hid, in_f)
            self.normal(f"{pre}.Wh_{d}", 4 * hid, hid)
            self.normal(f"{pre}.bias_ih_{d}", 4 * hid)
            self.normal(f"{pre}.bias_hh_{d}", 4 * hid)

    def adain(self, pre, style, c):
        self.linear(pre + ".fc", 2 * c, style)

    def adain_resblk1d(self, pre, din, dout, style, upsample=False):
        self.conv_weighted(pre + ".conv1", dout, 3, din)
        self.conv_weighted(pre + ".conv2", dout, 3, dout)
        self.adain(pre + ".norm1", style, din)
        self.adain(pre + ".norm2", style, dout)
        if din != dout:
            self.conv_weighted(pre + ".conv1x1", dout, 1, din, bias=False)
        if upsample:
            self.conv_weighted(pre + ".pool", din, 3, 1)

    def adain_resblock1(self, pre, c, k, style):
        for j in range(3):
            self.conv_weighted(f"{pre}.convs1.{j}", c, k, c)
            self.conv_weighted(f"{pre}.convs2.{j}", c, k, c)
            self.adain(f"{pre}.adain1.{j}", style, c)
            self.adain(f"{pre}.adain2.{j}", style, c)
            self.const(f"{pre}.alpha1.{j}", 1.0, 1, c, 1)
            self.const(f"{pre}.alpha2.{j}", 1.0, 1, c, 1)


def kokoro_weights(cfg, seed=0):
    """Parameter tree of ``tts/models/kokoro/kokoro.py:Model`` (reference) with random values."""
    g = _Gen(seed)
    pb, hd, st = cfg["plbert"], cfg["hidden_dim"], cfg["style_dim"]
    e = pb.get("embedding_size", 128)
    hs, it = pb["hidden_size"], pb["intermediate_size"]
    # ALBERT (modules.py:434-645)
    g.normal("bert.embeddings.word_embeddings.weight", cfg["n_token"], e)
    g.normal("bert.embeddings.position_embeddings.weight", pb["max_position_embeddings"], e)
    g.normal("bert.embeddings.token_type_embeddings.weight", 2, e)
    g.layer_norm("bert.embeddings.LayerNorm", e)
    g.linear("bert.encoder.embedding_hidden_mapping_in", hs, e)
    L = "bert.encoder.albert_layer_groups.0.albert_layers.0."
    for n in ("query", "key", "value", "dense"):
        g.linear(L + "attention." + n, hs, hs)
    g.layer_norm(L + "attention.LayerNorm", hs)
    g.layer_norm(L + "full_layer_layer_norm", hs)
    g.linear(L + "ffn", it, hs)
    g.linear(L + "ffn_output", hs, it)
    g.linear("bert.pooler", hs, hs)
    g.linear("bert_encoder", hd, hs)
    # prosody predictor (modules.py:288-411)
    for i in range(cfg["n_layer"]):
        g.lstm(f"predictor.text_encoder.lstms.{2 * i}", hd + st, hd // 2)
        g.linear(f"predictor.text_encoder.lstms.{2 * i + 1}.fc", 2 * hd, st)
    g.lstm("predictor.lstm", hd + st, hd // 2)
    # duration head: bias centred on logit(0.06) and wider weights, so that sum_k sigmoid(.) -- the predicted duration -- is ~3 frames per
    # token (a realistic ~13 phonemes/s) instead of the 25 frames/token that zero-mean logits give; the 128-phoneme utterance of
    # BASELINE config 2 then comes out at ~10 s of audio through the model's OWN duration head (bench.py e2e, un-pinned durations)
    g.normal("predictor.duration_proj.linear_layer.weight", cfg["max_dur"], hd, std=0.1)
    g.P["predictor.duration_proj.linear_layer.bias"] = _bf16(-2.8 + 0.02 * torch.randn(cfg["max_dur"], generator=g.g))
    g.lstm("predictor.shared", hd + st, hd // 2)
    for name in ("F0", "N"):
        g.adain_resblk1d(f"predictor.{name}.0", hd, hd, st)
        g.adain_resblk1d(f"predictor.{name}.1", hd, hd // 2, st, upsample=True)
        g.adain_resblk1d(f"predictor.{name}.2", hd // 2, hd // 2, st)
        g.normal(f"predictor.{name}_proj.weight", 1, 1, hd // 2)
        g.normal(f"predictor.{name}_proj.bias", 1)
    # text encoder (modules.py:21-68)
    g.normal("text_encoder.embedding.weight", cfg["n_token"], hd)
    for i in range(cfg["n_layer"]):
        g.conv_weighted(f"text_encoder.cnn.{i}.0", hd, cfg["text_encoder_kernel_size"], hd)
        g.layer_norm(f"text_encoder.cnn.{i}.1", hd)
    g.lstm("text_encoder.lstm", hd, hd // 2)
    # decoder (istftnet.py:936-997)
    g.adain_resblk1d("decoder.encode", hd + 2, 1024, st)
    for i in range(3):
        g.adain_resblk1d(f"decoder.decode.{i}", 1024 + 2 + 64, 1024, st)
    g.adain_resblk1d("decoder.decode.3", 1024 + 2 + 64, 512, st, upsample=True)
    g.conv_weighted("decoder.F0_conv", 1, 3, 1)
    g.conv_weighted("decoder.N_conv", 1, 3, 1)
    g.conv_weighted("decoder.asr_res.0", 64, 1, 512)
    # generator (istftnet.py:725-835)
    ist = cfg["istftnet"]
    G = "decoder.generator"
    g.linear(G + ".m_source.l_linear", 1, 9, std=0.3)
    c0 = ist["upsample_initial_channel"]
    rates, ks = ist["upsample_rates"], ist["upsample_kernel_sizes"]
    nfft = ist["gen_istft_n_fft"]
    nk = len(ist["resblock_kernel_sizes"])
    for i, (u, k) in enumerate(zip(rates, ks)):
        cin, cout = c0 // (2 ** i), c0 // (2 ** (i + 1))
        g.conv_weighted(f"{G}.ups.{i}", cin, k, cout, bias_c=cout)      # ConvWeighted(cout, cin, .., encode=True)
        for j, rk in enumerate(ist["resblock_kernel_sizes"]):
            g.adain_resblock1(f"{G}.resblocks.{i * nk + j}", cout, rk, st)
        if i + 1 < len(rates):
            sf0 = math.prod(rates[i + 1:])
            g.normal(f"{G}.noise_convs.{i}.weight", cout, sf0 * 2, nfft + 2)
            g.normal(f"{G}.noise_convs.{i}.bias", cout)
            g.adain_resblock1(f"{G}.noise_res.{i}", cout, 7, st)
        else:
            g.normal(f"{G}.noise_convs.{i}.weight", cout, 1, nfft + 2)
            g.normal(f"{G}.noise_convs.{i}.bias", cout)
            g.adain_resblock1(f"{G}.noise_res.{i}", cout, 11, st)
    g.conv_weighted(G + ".conv_post", nfft + 2, 7, c0 // (2 ** len(rates)))
    return g.P


def kokoro_inputs(n_phonemes=128, n_token=178, seed=1):
    """cfg2 inputs: token ids [1, T] with BOS/EOS 0, style ref_s [1,256] (SURVEY.md section 8d)."""
    g = torch.Generator().manual_seed(seed)
    ids = torch.randint(1, n_token, (n_phonemes,), generator=g)
    ids = torch.cat([torch.zeros(1, dtype=torch.long), ids, torch.zeros(1, dtype=torch.long)])[None]
    ref_s = torch.randn(1, 256, generator=torch.Generator().manual_seed(seed + 1))
    return ids, ref_s


def kokoro_noise(n_samples, seed=3):
    """Injected randomness for SineGen: rand_ini [1,9] U[0,1), noise [1,n,9] N(0,1)."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand(1, 9, generator=g), torch.randn(1, n_samples, 9, generator=g)


# ============================================================================= codecs

def _fan(g, name, *shape, fan_in):
    return g.normal(name, *shape, std=1.0 / math.sqrt(fan_in))


FINAL_GAIN_DIV = 1.0e6     # keeps the pre-tanh signal O(0.5) so the tanh is not saturated in parity tests


def snac_weights(cfg, seed=6, encoder=False):
    """Parameter tree of codec/models/snac/snac.py:SNAC (quantizer + decoder; ``encoder=True`` adds the encoder and the quantizers'
    in_proj), random values.  weight_v ~ N(0, 1/fan_in), weight_g = ||v|| (so the effective weight is v), Snake alpha ~ U(0.5, 1.5)."""
    g = _Gen(seed)
    gen = g.g

    def wn(pre, shape, fan_in, except_dim=0, bias=None):
        v = _fan(g, pre + ".weight_v", *shape, fan_in=fan_in)
        axes = tuple(i for i in range(3) if i != except_dim)
        g.P[pre + ".weight_g"] = _bf16(torch.sqrt((v * v).sum(dim=axes, keepdim=True)))
        if bias:
            g.normal(pre + ".bias", bias, std=0.05)

    def alpha(name, c):
        g.P[name] = _bf16(0.5 + torch.rand(1, c, 1, generator=gen))

    latent = cfg["encoder_dim"] * (2 ** len(cfg["encoder_rates"]))
    cd = cfg["codebook_dim"]
    for i, _ in enumerate(cfg["vq_strides"]):
        q = f"quantizer.quantizers.{i}"
        g.normal(q + ".codebook.weight", cfg["codebook_size"], cd, std=1.0)
        wn(q + ".out_proj", (latent, 1, cd), cd, bias=latent)
    pre = "decoder.model.layers"
    li = 0
    wn(f"{pre}.{li}", (latent, 7, 1), 7, bias=latent); li += 1
    ch = cfg["decoder_dim"]
    wn(f"{pre}.{li}", (ch, 1, latent), latent, bias=ch); li += 1
    for i, stride in enumerate(cfg["decoder_rates"]):
        cin, cout = ch // (2 ** i), ch // (2 ** (i + 1))
        bp = f"{pre}.{li}.block.layers"; li += 1
        bi = 0
        alpha(f"{bp}.{bi}.alpha", cin); bi += 1
        wn(f"{bp}.{bi}", (cin, 2 * stride, cout), cin * 2, bias=cout); bi += 1          # (in, K, out); ~2 taps hit each output
        if cfg["noise"]:
            wn(f"{bp}.{bi}.linear", (cout, 1, cout), cout); bi += 1
        for _d in (1, 3, 9):
            rp = f"{bp}.{bi}.block.layers"; bi += 1
            alpha(rp + ".0.alpha", cout)
            wn(rp + ".1", (cout, 7, 1) if cfg["depthwise"] else (cout, 7, cout), 7 if cfg["depthwise"] else 7 * cout, bias=cout)
            alpha(rp + ".2.alpha", cout)
            wn(rp + ".3", (cout, 1, cout), cout, bias=cout)
    alpha(f"{pre}.{li}.alpha", cout); li += 1
    wn(f"{pre}.{li}", (1, 7, cout), 7 * cout * FINAL_GAIN_DIV, bias=1)
    if encoder:                                                   # snac/layers.py:133-158 (drawn AFTER the decode-side tensors: those keep their values)
        for i, _ in enumerate(cfg["vq_strides"]):
            wn(f"quantizer.quantizers.{i}.in_proj", (cd, 1, latent), latent, bias=cd)
        pre = "encoder.block.layers"
        d = cfg["encoder_dim"]
        wn(f"{pre}.0", (d, 7, 1), 7, bias=d)
        li = 1
        for stride in cfg["encoder_rates"]:
            bp = f"{pre}.{li}.block.layers"; li += 1
            for bi in range(3):
                rp = f"{bp}.{bi}.block.layers"
                alpha(rp + ".0.alpha", d)
                wn(rp + ".1", (d, 7, 1) if cfg["depthwise"] else (d, 7, d), 7 if cfg["depthwise"] else 7 * d, bias=d)
                alpha(rp + ".2.alpha", d)
                wn(rp + ".3", (d, 1, d), d, bias=d)
            alpha(f"{bp}.3.alpha", d)
            wn(f"{bp}.4", (2 * d, 2 * stride, d), 2 * stride * d, bias=2 * d)
            d *= 2
        wn(f"{pre}.{li}", (d, 7, 1) if cfg["depthwise"] else (d, 7, d), 7 if cfg["depthwise"] else 7 * d, bias=d)
    return g.P


def snac_codes(cfg, t_fine, batch=1, seed=6):
    """cfg5 SNAC inputs: codes[l] int64 [B, t_fine / stride_l] (t_fine must be a multiple of max stride)."""
    gen = torch.Generator().manual_seed(seed)
    return [torch.randint(0, cfg["codebook_size"], (batch, t_fine // s), generator=gen) for s in cfg["vq_strides"]]


def snac_noises(cfg, batch=1, seed=7):
    """Injected NoiseBlock draws: one N(0,1) per (batch, channel) per decoder block (snac/layers.py:261-267 quirk)."""
    gen = torch.Generator().manual_seed(seed)
    return [torch.randn(batch, 1, cfg["decoder_dim"] // (2 ** (i + 1)), generator=gen) for i in range(len(cfg["decoder_rates"]))]


def dac_weights(cfg, seed=8, encoder=True):
    """Parameter tree of codec/models/descript/dac.py:DAC (quantizer + decoder; ``encoder=True`` adds the encoder and the quantizers'
    in_proj), random values by the recipe of ``snac_weights``: weight_v ~ N(0, 1/fan_in), weight_g = ||v|| rounded to bf16 (so the folded
    weight is NOT 16-bit exact and the split-plane weight path runs), Snake alpha ~ U(0.5, 1.5) in the reference's [1, 1, C] layout.
    Transposed convs are (out, K, in) with the norm per input channel (nn/layers.py:89-92)."""
    g = _Gen(seed)
    gen = g.g

    def wn(pre, shape, fan_in, except_dim=0, bias=None):
        v = _fan(g, pre + ".weight_v", *shape, fan_in=fan_in)
        axes = tuple(i for i in range(3) if i != except_dim)
        g.P[pre + ".weight_g"] = _bf16(torch.sqrt((v * v).sum(dim=axes, keepdim=True)))
        if bias:
            g.normal(pre + ".bias", bias, std=0.05)

    def alpha(name, c):
        g.P[name] = _bf16(0.5 + torch.rand(1, 1, c, generator=gen))

    def res_units(bp, first, c):
        for i in range(3):
            rp = f"{bp}.{first + i}.block.layers"
            alpha(rp + ".0.alpha", c)
            wn(rp + ".1", (c, 7, c), 7 * c, bias=c)
            alpha(rp + ".2.alpha", c)
            wn(rp + ".3", (c, 1, c), c, bias=c)

    latent = cfg.get("latent_dim") or cfg["encoder_dim"] * (2 ** len(cfg["encoder_rates"]))
    cds = [cfg["codebook_dim"]] * cfg["n_codebooks"] if isinstance(cfg["codebook_dim"], int) else list(cfg["codebook_dim"])
    for i, cd in enumerate(cds):
        q = f"quantizer.quantizers.{i}"
        g.normal(q + ".codebook.weight", cfg["codebook_size"], cd, std=1.0)
        wn(q + ".out_proj", (latent, 1, cd), cd, bias=latent)
    pre = "decoder.model.layers"
    ch = cfg["decoder_dim"]
    wn(f"{pre}.0", (ch, 7, latent), 7 * latent, bias=ch)
    for i, stride in enumerate(cfg["decoder_rates"]):
        cin, cout = ch // (2 ** i), ch // (2 ** (i + 1))
        bp = f"{pre}.{i + 1}.block.layers"
        alpha(f"{bp}.0.alpha", cin)
        wn(f"{bp}.1", (cout, 2 * stride, cin), cin * 2, except_dim=2, bias=cout)         # ~2 taps hit each output
        res_units(bp, 2, cout)
    n = len(cfg["decoder_rates"])
    alpha(f"{pre}.{n + 1}.alpha", cout)
    wn(f"{pre}.{n + 2}", (1, 7, cout), 7 * cout * FINAL_GAIN_DIV, bias=1)
    if encoder:                                                   # drawn AFTER the decode-side tensors: those keep their values
        for i, cd in enumerate(cds):
            wn(f"quantizer.quantizers.{i}.in_proj", (cd, 1, latent), latent, bias=cd)
        pre = "encoder.block.layers"
        d = cfg["encoder_dim"]
        wn(f"{pre}.0", (d, 7, 1), 7, bias=d)
        for i, stride in enumerate(cfg["encoder_rates"]):
            bp = f"{pre}.{i + 1}.block.layers"
            res_units(bp, 0, d)
            alpha(f"{bp}.3.alpha", d)
            wn(f"{bp}.4", (2 * d, 2 * stride, d), 2 * stride * d, bias=2 * d)
            d *= 2
        n = len(cfg["encoder_rates"])
        alpha(f"{pre}.{n + 1}.alpha", d)
        wn(f"{pre}.{n + 2}", (latent, 3, d), 3 * d, bias=latent)
    return g.P


BIGVGAN_FINAL_GAIN = 0.01  # conv_post's gain: keeps the pre-tanh signal of the deep unit-gain stack mostly inside the unsaturated range


def bigvgan_weights(cfg, seed=9):
    """Parameter tree of codec/models/bigvgan/bigvgan.py:BigVGAN (``cfg`` a BigVGANConfig), without the resampling filters (the model
    computes them, as the reference's constructor does).  Unit-gain convs by the recipe of ``dac_weights`` (weight_v ~ N(0, 1/fan_in),
    weight_g = ||v|| rounded to bf16), transposed convs (out, K, in) with the norm per input channel (conv.py:91); SnakeBeta alpha / beta
    ~ 0.1 N(0, 1) for snake_logscale (exp ~ 1) and U(0.5, 1.5) otherwise; conv_post scaled by BIGVGAN_FINAL_GAIN."""
    from .codec.models.bigvgan import param_shapes
    g = _Gen(seed)
    for name, shape in param_shapes(cfg).items():
        leaf = name.rsplit(".", 1)[-1]
        if leaf == "filter" or leaf == "weight_g":
            continue
        if leaf == "weight_v":
            pre = name[: -len(".weight_v")]
            tr = pre.startswith("ups.")
            cout, k, cin = shape
            fan_in = cin * 2 if tr else cin * k                      # a transposed conv with K = 2 u hits each output with ~2 taps
            v = _fan(g, name, *shape, fan_in=fan_in)
            norm = torch.sqrt((v * v).sum(dim=(0, 1) if tr else (1, 2), keepdim=True))
            g.P[pre + ".weight_g"] = _bf16(norm * (BIGVGAN_FINAL_GAIN if pre == "conv_post" else 1.0))
        elif leaf == "bias":
            g.normal(name, *shape, std=0.05)
        elif cfg.snake_logscale:
            g.normal(name, *shape, std=0.1)
        else:
            g.P[name] = _bf16(0.5 + torch.rand(*shape, generator=g.g))
    return g.P


def mimi_weights(cfg, seed=5, encoder=False):
    """Parameter tree of codec/models/mimi/mimi.py:Mimi (decode side; ``encoder=True`` adds the SEANet encoder, the encoder transformer, the
    down-sampling conv and the quantisers' input projections), random values at the mimi_202407 shapes."""
    g = _Gen(seed)
    gen = g.g
    d, nf = cfg["dimension"], cfg["nfilters"]
    for name, nq in (("rvq_first", 1), ("rvq_rest", cfg["nq"] - 1)):
        for li in range(nq):
            cb = f"quantizer.{name}.vq.layers.{li}.codebook"
            g.normal(cb + ".embedding_sum", cfg["bins"], cfg["qdim"], std=1.0)
            g.P[cb + ".cluster_usage"] = _bf16(0.5 + 1.5 * torch.rand(cfg["bins"], generator=gen))
        _fan(g, f"quantizer.{name}.output_proj.weight", d, 1, cfg["qdim"], fan_in=cfg["qdim"] * (1 if nq == 1 else 4))
    s = cfg["upsample_stride"]
    _fan(g, "upsample.convtr.convtr.convtr.weight", d, 2 * s, 1, fan_in=2)
    for li in range(cfg["num_layers"]):
        L = f"decoder_transformer.transformer.layers.{li}"
        g.layer_norm(L + ".norm1", d)
        g.layer_norm(L + ".norm2", d)
        _fan(g, L + ".self_attn.in_proj.weight", 3 * d, d, fan_in=d)
        _fan(g, L + ".self_attn.out_proj.weight", d, d, fan_in=d)
        _fan(g, L + ".gating.linear1.weight", cfg["dim_feedforward"], d, fan_in=d)
        _fan(g, L + ".gating.linear2.weight", d, cfg["dim_feedforward"], fan_in=cfg["dim_feedforward"])
        g.P[L + ".layer_scale_1.scale"] = _bf16(torch.full((d,), 0.3) + 0.1 * torch.rand(d, generator=gen))
        g.P[L + ".layer_scale_2.scale"] = _bf16(torch.full((d,), 0.3) + 0.1 * torch.rand(d, generator=gen))
    mult = 1 << len(cfg["ratios"])
    _fan(g, "decoder.init_conv1d.conv.conv.weight", mult * nf, cfg["ksize"], d, fan_in=cfg["ksize"] * d)
    g.normal("decoder.init_conv1d.conv.conv.bias", mult * nf, std=0.05)
    for li, r in enumerate(cfg["ratios"]):
        cin, cout = mult * nf, mult * nf // 2
        L = f"decoder.layers.{li}"
        _fan(g, L + ".upsample.convtr.convtr.weight", cout, 2 * r, cin, fan_in=2 * cin)
        g.normal(L + ".upsample.convtr.convtr.bias", cout, std=0.05)
        hid = cout // cfg["compress"]
        _fan(g, L + ".residuals.0.block.0.conv.conv.weight", hid, cfg["residual_ksize"], cout, fan_in=cfg["residual_ksize"] * cout)
        g.normal(L + ".residuals.0.block.0.conv.conv.bias", hid, std=0.05)
        _fan(g, L + ".residuals.0.block.1.conv.conv.weight", cout, 1, hid, fan_in=hid)
        g.normal(L + ".residuals.0.block.1.conv.conv.bias", cout, std=0.05)
        mult //= 2
    _fan(g, "decoder.final_conv1d.conv.conv.weight", 1, cfg["last_ksize"], nf, fan_in=cfg["last_ksize"] * nf)
    g.normal("decoder.final_conv1d.conv.conv.bias", 1, std=0.05)
    if encoder:                                                   # drawn AFTER the decode-side tensors, which keep their values
        _fan(g, "encoder.init_conv1d.conv.conv.weight", nf, cfg["ksize"], 1, fan_in=cfg["ksize"])
        g.normal("encoder.init_conv1d.conv.conv.bias", nf, std=0.05)
        c = nf
        for li, r in enumerate(reversed(cfg["ratios"])):
            L = f"encoder.layers.{li}"
            hid = c // cfg["compress"]
            _fan(g, L + ".residuals.0.block.0.conv.conv.weight", hid, cfg["residual_ksize"], c, fan_in=cfg["residual_ksize"] * c)
            g.normal(L + ".residuals.0.block.0.conv.conv.bias", hid, std=0.05)
            _fan(g, L + ".residuals.0.block.1.conv.conv.weight", c, 1, hid, fan_in=hid)
            g.normal(L + ".residuals.0.block.1.conv.conv.bias", c, std=0.05)
            _fan(g, L + ".downsample.conv.conv.weight", 2 * c, 2 * r, c, fan_in=2 * r * c)
            g.normal(L + ".downsample.conv.conv.bias", 2 * c, std=0.05)
            c *= 2
        _fan(g, "encoder.final_conv1d.conv.conv.weight", d, cfg["last_ksize"], c, fan_in=cfg["last_ksize"] * c)
        g.normal("encoder.final_conv1d.conv.conv.bias", d, std=0.05)
        for li in range(cfg["num_layers"]):
            L = f"encoder_transformer.transformer.layers.{li}"
            g.layer_norm(L + ".norm1", d)
            g.layer_norm(L + ".norm2", d)
            _fan(g, L + ".self_attn.in_proj.weight", 3 * d, d, fan_in=d)
            _fan(g, L + ".self_attn.out_proj.weight", d, d, fan_in=d)
            _fan(g, L + ".gating.linear1.weight", cfg["dim_feedforward"], d, fan_in=d)
            _fan(g, L + ".gating.linear2.weight", d, cfg["dim_feedforward"], fan_in=cfg["dim_feedforward"])
            g.P[L + ".layer_scale_1.scale"] = _bf16(torch.full((d,), 0.3) + 0.1 * torch.rand(d, generator=gen))
            g.P[L + ".layer_scale_2.scale"] = _bf16(torch.full((d,), 0.3) + 0.1 * torch.rand(d, generator=gen))
        _fan(g, "downsample.conv.conv.conv.weight", d, 2 * s, d, fan_in=2 * s * d)
        for name in ("rvq_first", "rvq_rest"):
            _fan(g, f"quantizer.{name}.input_proj.weight", cfg["qdim"], 1, d, fan_in=d)
    return g.P


def mimi_codes(cfg, t, batch=1, seed=5):
    return torch.randint(0, cfg["bins"], (batch, cfg["nq"], t), generator=torch.Generator().manual_seed(seed))


# ============================================================================= Whisper

def _f16(x):
    return x.to(torch.float16).to(torch.float32)


def whisper_encoder_weights(dims, seed=0):
    """Parameter tree of stt/models/whisper/whisper.py:AudioEncoder (fp16 checkpoint, cfg3): N(0, 0.02), LN gains 1."""
    g = _Gen(seed)
    d, nm = dims["n_audio_state"], dims["n_mels"]

    def n(name, *shape):
        g.P[name] = _f16(torch.randn(*shape, generator=g.g) * 0.02)

    n("encoder.conv1.weight", d, 3, nm); n("encoder.conv1.bias", d)
    n("encoder.conv2.weight", d, 3, d); n("encoder.conv2.bias", d)
    for i in range(dims["n_audio_layer"]):
        L = f"encoder.blocks.{i}"
        for nm_ in ("query", "value", "out"):
            n(f"{L}.attn.{nm_}.weight", d, d); n(f"{L}.attn.{nm_}.bias", d)
        n(f"{L}.attn.key.weight", d, d)
        g.layer_norm(L + ".attn_ln", d)
        g.layer_norm(L + ".mlp_ln", d)
        n(L + ".mlp1.weight", 4 * d, d); n(L + ".mlp1.bias", 4 * d)
        n(L + ".mlp2.weight", d, 4 * d); n(L + ".mlp2.bias", d)
    g.layer_norm("encoder.ln_post", d)
    return g.P


def whisper_audio(batch, n_samples=480000, seed=4):
    """cfg3 input: 0.1 * N(0,1) float32 [B, n]."""
    return 0.1 * torch.randn(batch, n_samples, generator=torch.Generator().manual_seed(seed))


def kokoro_to_torch_checkpoint(P):
    """Reference-tree (MLX layout) Kokoro weights -> the PyTorch-layout checkpoint the hub ships, i.e. the input that
    ``Model.sanitize`` (kokoro.py:179-276) converts: conv weights (out, in, K), LSTM ``weight_ih_l0[_reverse]`` names."""
    inv = {"Wx_forward": "weight_ih_l0", "Wh_forward": "weight_hh_l0", "bias_ih_forward": "bias_ih_l0", "bias_hh_forward": "bias_hh_l0",
           "Wx_backward": "weight_ih_l0_reverse", "Wh_backward": "weight_hh_l0_reverse", "bias_ih_backward": "bias_ih_l0_reverse",
           "bias_hh_backward": "bias_hh_l0_reverse"}
    out = {}
    for k, v in P.items():
        base, _, leaf = k.rpartition(".")
        if leaf in inv:
            out[f"{base}.{inv[leaf]}"] = v
        elif "weight_v" in k or ("noise_convs" in k and leaf == "weight") or "F0_proj.weight" in k or "N_proj.weight" in k:
            out[k] = v.transpose(1, 2).contiguous()
        else:
            out[k] = v
    return out


def whisper_decoder_weights(dims, seed=1):
    """Parameter tree of stt/models/whisper/whisper.py:TextDecoder (fp16 checkpoint): N(0, 0.02), LN gains 1."""
    g = _Gen(seed)
    d = dims["n_text_state"]

    def n(name, *shape, std=0.02):
        g.P[name] = _f16(torch.randn(*shape, generator=g.g) * std)

    n("decoder.token_embedding.weight", dims["n_vocab"], d, std=0.3)      # peaky logits so the decode rules see text/timestamp competition
    n("decoder.positional_embedding", dims["n_text_ctx"], d)
    for i in range(dims["n_text_layer"]):
        L = f"decoder.blocks.{i}"
        for a in ("attn", "cross_attn"):
            for nm_ in ("query", "value", "out"):
                n(f"{L}.{a}.{nm_}.weight", d, d); n(f"{L}.{a}.{nm_}.bias", d)
            n(f"{L}.{a}.key.weight", d, d)
        for ln in ("attn_ln", "cross_attn_ln", "mlp_ln"):
            g.layer_norm(f"{L}.{ln}", d)
        n(L + ".mlp1.weight", 4 * d, d); n(L + ".mlp1.bias", 4 * d)
        n(L + ".mlp2.weight", d, 4 * d); n(L + ".mlp2.bias", d)
    g.layer_norm("decoder.ln", d)
    g.P["decoder.token_embedding.weight"][50364:] *= 0.25      # damp timestamp logits (random weights would otherwise let the
    g.P["decoder.token_embedding.weight"] = _f16(g.P["decoder.token_embedding.weight"])   # 1501 timestamps out-vote every text token)
    return g.P


# ============================================================================= Qwen3-TTS

def qwen3_talker_weights(cfg, text_vocab=512, seed=11):
    """Parameter tree of tts/models/qwen3_tts/talker.py:Qwen3TTSTalkerForConditionalGeneration with the checkpoint's ``talker.``
    prefix; ``cfg`` is the flat dict of oracle/qwen3.py:TALKER.  bf16-exact values.  ``text_vocab`` shrinks the 151 936-row text
    embedding (prompt assembly only, not on the per-frame path); fan-in scaling keeps the residual stream O(1) through 28 layers
    and the logits wide enough (std ~ 2) that sampling is not uniform."""
    g = _Gen(seed)
    gen = g.g
    H, I, hd = cfg["hidden_size"], cfg["intermediate_size"], cfg["head_dim"]
    hq, hk = cfg["num_attention_heads"], cfg["num_key_value_heads"]

    def stack(pre, n_layers, H, I, hq, hk, hd):
        for i in range(n_layers):
            L = f"{pre}.layers.{i}"
            _fan(g, L + ".self_attn.q_proj.weight", hq * hd, H, fan_in=H)
            _fan(g, L + ".self_attn.k_proj.weight", hk * hd, H, fan_in=H)
            _fan(g, L + ".self_attn.v_proj.weight", hk * hd, H, fan_in=H)
            _fan(g, L + ".self_attn.o_proj.weight", H, hq * hd, fan_in=4 * hq * hd)
            g.P[L + ".self_attn.q_norm.weight"] = _bf16(1.0 + 0.1 * torch.randn(hd, generator=gen))
            g.P[L + ".self_attn.k_norm.weight"] = _bf16(1.0 + 0.1 * torch.randn(hd, generator=gen))
            g.P[L + ".input_layernorm.weight"] = _bf16(1.0 + 0.1 * torch.randn(H, generator=gen))
            g.P[L + ".post_attention_layernorm.weight"] = _bf16(1.0 + 0.1 * torch.randn(H, generator=gen))
            _fan(g, L + ".mlp.gate_proj.weight", I, H, fan_in=H)
            _fan(g, L + ".mlp.up_proj.weight", I, H, fan_in=H)
            _fan(g, L + ".mlp.down_proj.weight", H, I, fan_in=4 * I)
        g.P[pre + ".norm.weight"] = _bf16(1.0 + 0.1 * torch.randn(H, generator=gen))

    stack("talker.model", cfg["num_hidden_layers"], H, I, hq, hk, hd)
    g.normal("talker.model.codec_embedding.weight", cfg["vocab_size"], H, std=1.0)
    g.normal("talker.model.text_embedding.weight", text_vocab, cfg["text_hidden_size"], std=1.0)
    _fan(g, "talker.text_projection.linear_fc1.weight", cfg["text_hidden_size"], cfg["text_hidden_size"], fan_in=cfg["text_hidden_size"])
    g.normal("talker.text_projection.linear_fc1.bias", cfg["text_hidden_size"], std=0.05)
    _fan(g, "talker.text_projection.linear_fc2.weight", H, cfg["text_hidden_size"], fan_in=cfg["text_hidden_size"] / 4)
    g.normal("talker.text_projection.linear_fc2.bias", H, std=0.05)
    _fan(g, "talker.codec_head.weight", cfg["vocab_size"], H, fan_in=H / 4)
    cH, cI = cfg["cp_hidden_size"], cfg["cp_intermediate_size"]
    stack("talker.code_predictor.model", cfg["cp_num_hidden_layers"], cH, cI, cfg["cp_num_attention_heads"], cfg["cp_num_key_value_heads"],
          cfg["cp_head_dim"])
    for k in range(cfg["num_code_groups"] - 1):
        g.normal(f"talker.code_predictor.model.codec_embedding.{k}.weight", cfg["cp_vocab_size"], H, std=1.0)
        _fan(g, f"talker.code_predictor.lm_head.{k}.weight", cfg["cp_vocab_size"], cH, fan_in=cH / 4)
    return g.P


def qwen3_tokenizer_weights(cfg, seed=12, encoder=None):
    """Parameter tree of speech_tokenizer.py:Qwen3TTSSpeechTokenizer (decode side, MLX names after ``sanitize``); ``cfg`` is the
    flat dict of oracle/qwen3.py:TOKENIZER_DECODER.  bf16-exact values.  ``encoder`` = the flat dict of oracle/qwen3.py:TOKENIZER_ENCODER
    adds the speech-tokenizer encoder (``encoder_model.*``, the names of Qwen3TTSSpeechTokenizerEncoder.sanitize): Mimi's encode side at
    those shapes, drawn from its own stream (the decoder's tensors keep their values)."""
    g = _Gen(seed)
    gen = g.g
    cd, ld, hs = cfg["codebook_dim"], cfg["latent_dim"], cfg["hidden_size"]
    nsem, nq = cfg["num_semantic_quantizers"], cfg["num_quantizers"]
    D = "decoder."
    for name, n in (("rvq_first", nsem), ("rvq_rest", nq - nsem)):
        for li in range(n):
            g.normal(f"{D}quantizer.{name}.vq.layers.{li}.codebook.embed.weight", cfg["codebook_size"], cd // 2, std=1.0)
        _fan(g, f"{D}quantizer.{name}.output_proj.weight", cd, 1, cd // 2, fan_in=(cd // 2) * max(n, 1))
    _fan(g, D + "pre_conv.conv.weight", ld, 3, cd, fan_in=3 * cd)
    g.normal(D + "pre_conv.conv.bias", ld, std=0.05)
    T = D + "pre_transformer"
    _fan(g, T + ".input_proj.weight", hs, ld, fan_in=ld)
    g.normal(T + ".input_proj.bias", hs, std=0.05)
    _fan(g, T + ".output_proj.weight", ld, hs, fan_in=hs)
    g.normal(T + ".output_proj.bias", ld, std=0.05)
    nh, hd, I = cfg["num_attention_heads"], cfg["head_dim"], cfg["intermediate_size"]
    for i in range(cfg["num_hidden_layers"]):
        L = f"{T}.layers.{i}"
        for n in "qkv":
            _fan(g, L + f".self_attn.{n}_proj.weight", nh * hd, hs, fan_in=hs)
        _fan(g, L + ".self_attn.o_proj.weight", hs, nh * hd, fan_in=nh * hd)
        _fan(g, L + ".mlp.gate_proj.weight", I, hs, fan_in=hs)
        _fan(g, L + ".mlp.up_proj.weight", I, hs, fan_in=hs)
        _fan(g, L + ".mlp.down_proj.weight", hs, I, fan_in=I)
        g.P[L + ".input_layernorm.weight"] = _bf16(1.0 + 0.1 * torch.randn(hs, generator=gen))
        g.P[L + ".post_attention_layernorm.weight"] = _bf16(1.0 + 0.1 * torch.randn(hs, generator=gen))
        g.P[L + ".self_attn_layer_scale.scale"] = _bf16(0.3 + 0.1 * torch.rand(hs, generator=gen))
        g.P[L + ".mlp_layer_scale.scale"] = _bf16(0.3 + 0.1 * torch.rand(hs, generator=gen))
    g.P[T + ".norm.weight"] = _bf16(1.0 + 0.1 * torch.randn(hs, generator=gen))
    for i, f in enumerate(cfg["upsampling_ratios"]):
        U = f"{D}upsample.{i}"
        _fan(g, U + ".0.conv.weight", ld, f, ld, fan_in=ld)
        g.normal(U + ".0.conv.bias", ld, std=0.05)
        _fan(g, U + ".1.dwconv.conv.weight", ld, 7, 1, fan_in=7)
        g.normal(U + ".1.dwconv.conv.bias", ld, std=0.05)
        g.P[U + ".1.norm.weight"] = _bf16(1.0 + 0.1 * torch.randn(ld, generator=gen))
        g.normal(U + ".1.norm.bias", ld, std=0.05)
        _fan(g, U + ".1.pwconv1.weight", 4 * ld, ld, fan_in=ld)
        g.normal(U + ".1.pwconv1.bias", 4 * ld, std=0.05)
        _fan(g, U + ".1.pwconv2.weight", ld, 4 * ld, fan_in=4 * ld)
        g.normal(U + ".1.pwconv2.bias", ld, std=0.05)
        g.P[U + ".1.gamma"] = _bf16(0.3 + 0.1 * torch.rand(ld, generator=gen))
    dd = cfg["decoder_dim"]
    _fan(g, D + "decoder.0.conv.weight", dd, 7, ld, fan_in=7 * ld)
    g.normal(D + "decoder.0.conv.bias", dd, std=0.05)
    cin = dd
    for bi, r in enumerate(cfg["upsample_rates"]):
        cout = cin // 2
        B_ = f"{D}decoder.{bi + 1}.block"
        g.P[B_ + ".0.alpha"] = _bf16(0.2 * torch.randn(cin, generator=gen))
        g.P[B_ + ".0.beta"] = _bf16(0.2 * torch.randn(cin, generator=gen))
        _fan(g, B_ + ".1.conv.weight", cout, 2 * r, cin, fan_in=2 * cin)
        g.normal(B_ + ".1.conv.bias", cout, std=0.05)
        for ui in range(3):
            U = f"{B_}.{ui + 2}"
            for a in ("act1", "act2"):
                g.P[f"{U}.{a}.alpha"] = _bf16(0.2 * torch.randn(cout, generator=gen))
                g.P[f"{U}.{a}.beta"] = _bf16(0.2 * torch.randn(cout, generator=gen))
            _fan(g, U + ".conv1.conv.weight", cout, 7, cout, fan_in=7 * cout * 2)
            g.normal(U + ".conv1.conv.bias", cout, std=0.05)
            _fan(g, U + ".conv2.conv.weight", cout, 1, cout, fan_in=cout * 4)
            g.normal(U + ".conv2.conv.bias", cout, std=0.05)
        cin = cout
    n_blocks = len(cfg["upsample_rates"])
    g.P[f"{D}decoder.{n_blocks + 1}.alpha"] = _bf16(0.2 * torch.randn(cin, generator=gen))
    g.P[f"{D}decoder.{n_blocks + 1}.beta"] = _bf16(0.2 * torch.randn(cin, generator=gen))
    _fan(g, f"{D}decoder.{n_blocks + 2}.conv.weight", 1, 7, cin, fan_in=7 * cin * 16)
    g.normal(f"{D}decoder.{n_blocks + 2}.conv.bias", 1, std=0.02)
    if encoder is not None:
        keep = ("encoder.", "encoder_transformer.", "downsample.", "quantizer.")
        g.P.update({"encoder_model." + k: v for k, v in mimi_weights(encoder, seed=seed + 1, encoder=True).items() if k.startswith(keep)})
    return g.P


def qwen3_codes(cfg, t, batch=1, seed=13):
    """codes [B, 16, T] (first code > 0 so that the valid-length rule of speech_tokenizer.py:1113-1116 keeps every frame)."""
    return torch.randint(1, cfg["codebook_size"], (batch, cfg["num_quantizers"], t), generator=torch.Generator().manual_seed(seed))


def qwen3_speaker_encoder_weights(cfg, seed=14):
    """Parameter tree of tts/models/qwen3_tts/speaker_encoder.py:Qwen3TTSSpeakerEncoder with the checkpoint's ``speaker_encoder.``
    prefix, MLX conv layout [out, K, in]; ``cfg`` is a dict of oracle/qwen3.py:SPEAKER_ENCODER's keys.  bf16-exact values, weights
    scaled by 1/sqrt(fan-in) so that every block's activations stay O(1), biases N(0, 0.05)."""
    g = _Gen(seed)
    ch, ks, sc = cfg["enc_channels"], cfg["enc_kernel_sizes"], cfg["enc_res2net_scale"]
    A, S, E = cfg["enc_attention_channels"], cfg["enc_se_channels"], cfg["enc_dim"]

    def conv(name, cout, k, cin):
        g.normal(name + ".weight", cout, k, cin, std=1.0 / math.sqrt(k * cin))
        g.normal(name + ".bias", cout, std=0.05)

    p = "speaker_encoder."
    conv(p + "blocks.0.conv", ch[0], ks[0], cfg["mel_dim"])
    for i in range(1, len(ch) - 1):
        b = f"{p}blocks.{i}"
        conv(b + ".tdnn1.conv", ch[i], 1, ch[i - 1])
        for j in range(sc - 1):
            conv(f"{b}.res2net_block.blocks.{j}.conv", ch[i] // sc, ks[i], ch[i] // sc)
        conv(b + ".tdnn2.conv", ch[i], 1, ch[i])
        conv(b + ".se_block.conv1", S, 1, ch[i])
        conv(b + ".se_block.conv2", ch[i], 1, S)
    conv(p + "mfa.conv", ch[-1], ks[-1], sum(ch[1:-1]))
    conv(p + "asp.tdnn.conv", A, 1, 3 * ch[-1])
    conv(p + "asp.conv", ch[-1], 1, A)
    conv(p + "fc", E, 1, 2 * ch[-1])
    return g.P


def vocos_backbone_weights(bb, seed=11, prefix="backbone."):
    """MLX-layout parameters of a ``codec.models.vocos.VocosBackbone``: convs and linears ~ N(0, 1/fan_in) (unit gain), biases 0.05 N(0, 1),
    LayerNorm gains 1 + 0.1 N(0, 1); AdaLayerNorm's scale linear gives 1 + small per condition (weights 0.1 / E N(0, 1), bias 1), its shift
    linear small values; ``gamma`` the constructor's value.  bf16-exact weights, so the tensor-core path holds them exactly."""
    g = _Gen(seed)
    for name, shape in bb.param_shapes(prefix).items():
        leaf = name.rsplit(".", 1)[-1]
        if leaf == "gamma":
            g.const(name, bb.layer_scale_init_value, *shape)
        elif ".scale." in name or ".shift." in name:
            g.normal(name, *shape, std=0.1 / shape[-1] if leaf == "weight" else 0.05)
            if name.endswith(".scale.bias"):
                g.P[name] = g.P[name] + 1.0
        elif leaf == "bias":
            g.normal(name, *shape, std=0.05)
        elif len(shape) == 1:
            g.P[name] = _bf16(1.0 + 0.1 * torch.randn(*shape, generator=g.g))
        else:
            _fan(g, name, *shape, fan_in=math.prod(shape[1:]))
    return g.P


def vocos_head_weights(head, seed=12, prefix="head."):
    """ISTFTHead's linear at unit gain: its input is LayerNorm output (~unit variance), so the log-magnitudes are ~N(-0.5, 1) and well under
    1 % of the bins reach exp(.) > 100 -- the clip does not hide errors -- and the phases ~N(0, 1)."""
    g = _Gen(seed)
    (wn, ws), (bn, bs) = head.param_shapes(prefix).items()
    _fan(g, wn, *ws, fan_in=ws[1])
    b = 0.05 * torch.randn(*bs, generator=g.g)
    b[: head.n_fft // 2 + 1] -= 0.5
    g.P[bn] = _bf16(b)
    return g.P


def vocos_weights(config: dict, seed=11) -> dict:
    """Released-size synthetic parameters for ``Vocos.from_hparams(config)`` (the reference's YAML-shaped dict)."""
    from .codec.models.vocos import ISTFTHead, VocosBackbone
    bb = VocosBackbone(**config["backbone"]["init_args"], device="cpu")
    hd = ISTFTHead(**config["head"]["init_args"], device="cpu")
    P = vocos_backbone_weights(bb, seed)
    P.update(vocos_head_weights(hd, seed + 1))
    return P


def encodec_weights(config: dict, seed=15) -> dict:
    """MLX-layout parameters of ``codec.models.encodec.Encodec(config)`` (float32, as the released checkpoints are): convs ~ N(0, 1/fan_in)
    (unit gain; the residual branch's last conv and the shortcut at 1/sqrt(2) so that a block keeps the scale), biases N(0, 0.05^2),
    GroupNorm gains 1 + 0.1 N(0, 1); LSTM Wx and Wh ~ N(0, 0.5^2 / H), bias N(0, 0.1^2) -- gate pre-activations of order 1, neither
    saturated nor vanishing; code book q: rows of nearly equal norm (so that the nearest code is decided by direction and every code is
    used), 0.15 * 0.8^q per element, shrinking with the residual it quantises."""
    from .codec.models.encodec import param_shapes
    g = torch.Generator().manual_seed(seed)
    P = {}
    for name, shape in param_shapes(config).items():
        leaf = name.rsplit(".", 1)[-1]
        if leaf == "embed":
            q = int(name.split(".")[2])
            e = torch.randn(*shape, generator=g)
            e = e / e.norm(dim=1, keepdim=True) * math.sqrt(shape[1]) * (1 + 0.05 * torch.randn(shape[0], 1, generator=g))
            P[name] = 0.15 * 0.8 ** q * e
        elif leaf in ("Wx", "Wh"):
            P[name] = 0.5 / math.sqrt(shape[1]) * torch.randn(*shape, generator=g)
        elif leaf == "bias":
            P[name] = (0.1 if name.endswith(("Wx", "lstm")) or ".lstm." in name else 0.05) * torch.randn(*shape, generator=g)
        elif ".norm." in name:
            P[name] = 1.0 + 0.1 * torch.randn(*shape, generator=g)
        else:
            gain = 1 / math.sqrt(2) if (".block.3." in name or ".shortcut." in name) else 1.0
            P[name] = gain / math.sqrt(shape[1] * shape[2]) * torch.randn(*shape, generator=g)
    return P


# reference test configuration of Soprano's LM (tts/tests/test_models.py TestSoprano), 12 layers
SOPRANO_LM = {"hidden_size": 512, "num_hidden_layers": 12, "num_attention_heads": 8, "num_key_value_heads": 4, "intermediate_size": 1024,
              "vocab_size": 32000, "head_dim": 64, "rms_norm_eps": 1e-5, "rope_theta": 10000.0, "max_position_embeddings": 4096,
              "tie_word_embeddings": False, "model_type": "qwen3"}


def soprano_weights(model, seed=21, logit_std=4.0) -> dict:
    """Sanitized parameters of a ``tts.models.soprano.Model``: the Qwen3 LM (``language_model.*``, fan-in scaled bf16-exact values, a head
    whose logits have a spread of about ``logit_std`` so that top-p filtering bites) and the decoder (``decoder.decoder.*``,
    ``decoder.head.*``)."""
    c = model.config
    g = _Gen(seed)
    gen = g.g
    H, I, hd, hq, hk = c.hidden_size, c.intermediate_size, c.head_dim, c.num_attention_heads, c.num_key_value_heads
    for i in range(c.num_hidden_layers):
        L = f"language_model.layers.{i}"
        _fan(g, L + ".self_attn.q_proj.weight", hq * hd, H, fan_in=H)
        _fan(g, L + ".self_attn.k_proj.weight", hk * hd, H, fan_in=H)
        _fan(g, L + ".self_attn.v_proj.weight", hk * hd, H, fan_in=H)
        _fan(g, L + ".self_attn.o_proj.weight", H, hq * hd, fan_in=4 * hq * hd)
        for n, d in ((".self_attn.q_norm.weight", hd), (".self_attn.k_norm.weight", hd), (".input_layernorm.weight", H),
                     (".post_attention_layernorm.weight", H)):
            g.P[L + n] = _bf16(1.0 + 0.1 * torch.randn(d, generator=gen))
        _fan(g, L + ".mlp.gate_proj.weight", I, H, fan_in=H)
        _fan(g, L + ".mlp.up_proj.weight", I, H, fan_in=H)
        _fan(g, L + ".mlp.down_proj.weight", H, I, fan_in=4 * I)
    g.P["language_model.norm.weight"] = _bf16(1.0 + 0.1 * torch.randn(H, generator=gen))
    g.normal("language_model.embed_tokens.weight", c.vocab_size, H, std=1.0)
    _fan(g, "language_model.lm_head.weight", c.vocab_size, H, fan_in=H / logit_std ** 2)
    g.P.update(vocos_backbone_weights(model.decoder.decoder, seed=seed + 1, prefix="decoder.decoder."))
    g.P.update(vocos_head_weights(model.decoder.head, seed=seed + 2, prefix="decoder.head."))
    return g.P
