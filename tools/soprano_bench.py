"""Soprano on the GPU: decode tokens/s and audio-s/s at B = 1 and with 4 and 16 sentences batched, prefill and decoder time per 10 s of
audio, and the mlx-lm sampler kernel against a torch sort-based restatement (both replayed from CUDA graphs, alternated in the same process).  Synthetic bf16 LM weights
at the reference's test configuration (hidden 512, 12 layers, vocabulary 32 000) and the released decoder (dim 768, n_fft 2048, hop 512).

    python tools/soprano_bench.py [--steps 256] [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    return q or torch.cuda.get_device_name()


def timed(fn, reps):
    out = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append(time.perf_counter() - t0)
    return statistics.median(out)


def torch_sampler(logits, u, temperature, top_p):
    """make_sampler(temperature, top_p) on raw logits with torch ops: sort, exp, cumsum, mask, softmax, inverse CDF."""
    srt, idx = torch.sort(logits, dim=-1, stable=True)
    cum = torch.cumsum(torch.exp(srt).double(), dim=-1)
    keep = torch.empty_like(cum, dtype=torch.bool).scatter_(-1, idx, cum > 1 - top_p)
    y = (logits * (1 / temperature)).masked_fill(~keep, float("-inf")).double()
    w = torch.softmax(y, dim=-1).cumsum(-1)
    return torch.searchsorted(w, u[:, None].double()).clamp(max=logits.shape[1] - 1)[:, 0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=256)
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("soprano_bench: needs a CUDA device")
    from mlx_audio_b200 import ops, synth
    from mlx_audio_b200.tts.models.soprano import DecoderConfig, Model, ModelConfig
    m = Model(ModelConfig.from_dict({**synth.SOPRANO_LM, "decoder_config": DecoderConfig()}), device="cuda")
    m.load_weights(list(synth.soprano_weights(m).items()))
    m._stop_token_id = None                                          # run every row to max_tokens
    res = {"gpu": gpu_info(), "steps": a.steps}
    prompt = list(range(2, 42))                                      # a 40-token prompt
    for B in (1, 4, 16):
        rows = [prompt] * B
        m.generate_from_ids(rows, max_tokens=a.steps, seed=0)          # warm-up + graph capture
        t = timed(lambda: m.generate_from_ids(rows, max_tokens=a.steps, seed=0), a.reps)
        tp = timed(lambda: m.generate_from_ids(rows, max_tokens=0, seed=0), a.reps)
        tok_s = B * a.steps / (t - tp)
        res[f"B{B}"] = {"call_ms": round(t * 1e3, 2), "prefill_ms": round(tp * 1e3, 2), "decode_step_ms": round((t - tp) / a.steps * 1e3, 4),
                        "tokens_per_s": round(tok_s, 1), "audio_s_per_s": round(tok_s * 2048 / 32000, 1)}
    L = 10 * 32000 // 2048 + 1                                       # hidden states for 10 s of audio
    h = torch.randn(1, L, 512, device="cuda")
    m.decoder.waveform(h)
    res["decoder_ms_per_10s"] = round(timed(lambda: m.decoder.waveform(h), a.reps * 4) * 1e3, 3)
    # sampler: kernel vs torch restatement, alternated; each as a CUDA graph of 100 calls timed with events, so the figure is device time
    # without the host wrapper (the decode step replays the kernel the same way)
    def graph_of(fn):
        fn()
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(100):
                fn()
        return g

    def replay_us(g):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        g.replay()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) * 1e3 / 100

    for B in (1, 16):
        lg = torch.randn(B, 32000, device="cuda") * 4 - 8
        u = torch.rand(B, 1, device="cuda")
        out = torch.empty(B, dtype=torch.int64, device="cuda")
        gk = graph_of(lambda: ops.lm_sample_mlx(lg, temperature=0.3, top_p=0.95, u=u, out=out))
        gt = graph_of(lambda: torch_sampler(lg, u[:, 0], 0.3, 0.95))
        k_t, t_t = [], []
        for _ in range(10):
            k_t.append(replay_us(gk))
            t_t.append(replay_us(gt))
        k = statistics.median(k_t)
        res[f"sampler_B{B}_us"] = {"kernel": round(k, 2), "torch_sort": round(statistics.median(t_t), 2),
                                   "share_of_decode_step": round(k / (res[f"B{B}"]["decode_step_ms"] * 1e3), 3)}
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
