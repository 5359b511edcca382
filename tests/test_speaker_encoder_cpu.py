"""Speaker-encoder checks that need no GPU: the kernels build for sm_90a without spills, and a hub-layout checkpoint (PyTorch conv
weights [out, in, K]) loads to the same packed weights as the MLX-layout one."""
import os
import re
import subprocess

import torch

from mlx_audio_b200 import build
from oracle import qwen3 as Q

KERNELS = ("spk_logmel_kernel", "spk_reflect_pad_kernel", "spk_res2net_kernelILi4", "spk_res2net_kernelILi1", "spk_channel_stats_kernel",
           "spk_se_gate_kernel", "spk_se_apply_kernel", "spk_gemv_kernel", "spk_asp_act_kernel", "spk_asp_pool_kernel")


def test_speaker_kernels_compile_without_spills(tmp_path):
    assert "speaker.cu" in build.SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "speaker.cu"), "-o", str(tmp_path / "speaker.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    props = re.findall(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    for k in KERNELS:
        hits = [(int(s), int(l)) for name, s, l in props if k in name]
        assert hits == [(0, 0)], (k, hits)


def _packed(enc):
    out = {"b0": enc.b0[0].w, "mfa": enc.mfa[0].w, "asp_wx": enc.asp_wx.w, "asp_wms": enc.asp_wms, "asp_conv": enc.asp_conv.w,
           "fc_w": enc.fc_w, "fc_b": enc.fc_b}
    for i, blk in enumerate(enc.blocks):
        for k in ("res_w", "res_b", "se_w1", "se_b1", "se_w2", "se_b2"):
            out[f"{i}.{k}"] = blk[k]
        out[f"{i}.tdnn1"], out[f"{i}.tdnn2"] = blk["tdnn1"].w, blk["tdnn2"].w
    return out


def test_hub_checkpoint_loads_like_mlx_layout():
    """Released shapes: Model.sanitize + Qwen3TTSSpeakerEncoder.sanitize turn every [out, in, K] conv of a hub checkpoint into the MLX
    layout (the reference's shape heuristic decides, as in speaker_encoder.py:309-332), so both dicts pack identically."""
    from mlx_audio_b200 import synth
    from mlx_audio_b200.tts.models.qwen3_tts import Model, Qwen3TTSSpeakerEncoderConfig
    from mlx_audio_b200.tts.models.qwen3_tts.speaker_encoder import Qwen3TTSSpeakerEncoder
    cfg = dict(Q.SPEAKER_ENCODER)
    mlx = synth.qwen3_speaker_encoder_weights(cfg, seed=3)
    hub = {k: (v.permute(0, 2, 1).contiguous() if v.dim() == 3 else v) for k, v in mlx.items()}
    hub["speaker_encoder.blocks.0.conv.position_ids"] = torch.arange(4)            # dropped by Model.sanitize
    a = Qwen3TTSSpeakerEncoder(Qwen3TTSSpeakerEncoderConfig(**cfg), "cpu")
    a.load_weights(Qwen3TTSSpeakerEncoder.sanitize(Model.sanitize(hub)))
    b = Qwen3TTSSpeakerEncoder(Qwen3TTSSpeakerEncoderConfig(**cfg), "cpu")
    b.load_weights(Qwen3TTSSpeakerEncoder.sanitize(mlx))
    pa, pb = _packed(a), _packed(b)
    assert pa.keys() == pb.keys()
    for k in pa:
        assert pa[k].shape == pb[k].shape and torch.equal(pa[k], pb[k]), k
    assert tuple(pa["0.res_w"].shape) == (7, 3, 64, 64) and tuple(pa["asp_wms"].shape) == (128, 3072) and tuple(pa["fc_w"].shape) == (1024, 3072)
    # the conv weights the reference packs: blocks.1.res2net_block.blocks.0 [64, 3, 64] (MLX) is stage 0 with taps first
    w = mlx["speaker_encoder.blocks.1.res2net_block.blocks.0.conv.weight"]
    assert torch.equal(pa["0.res_w"][0], w.permute(1, 2, 0))
