"""SHA-256 digests of what Kokoro's generator-group launches of the fused conv kernel write at the benchmarked shape (bench.py cfg2:
128 phonemes, F = 390 frames, synthetic checkpoint seed 0, inputs seed 1, device noise seed 1234).

Every `ops.conv_fused` launch of one eager `Model.forward_ids` that holds three problems (the k = 3 / 7 / 11 AdaINResBlock1 branches of
a generator stage: c1 and c2 for dilations 1, 3, 5, two stages = 12 launches) is digested right after it runs: each problem's output
rows and the (sum, sumsq) bins it accumulated.  The fused kernel's results do not depend on its schedule (fixed product order, fixed-order
split-K and statistics reductions, integer statistics atomics), so a change to the kernel's pipeline must reproduce these bytes.

Run on an H100 from the repository root:  python tests/golden/make_fused_group_digest.py
"""
from __future__ import annotations

import hashlib
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
OUT = os.path.join(HERE, "fused_group_digest.json")


def _label(q) -> str:
    dil = q.shifts[1] - q.shifts[0] if q.taps > 1 else 1
    return f"L{q.L} {q.Cin}->{q.N} k{q.taps} d{dil}"


def generator_group_digests(dev="cuda:0") -> list:
    import torch
    from mlx_audio_b200 import ops, synth
    from mlx_audio_b200.configs import KOKORO_82M
    from mlx_audio_b200.tts.models.kokoro import Model, ModelConfig

    P = synth.kokoro_weights(KOKORO_82M, seed=0)
    model = Model(ModelConfig.from_dict(KOKORO_82M), device=dev).load_weights(list(P.items()))
    model.seed(1234)
    ids, ref_s = synth.kokoro_inputs(128, seed=1)
    out = []
    orig = ops.conv_fused

    def digesting(problems):
        ys = orig(problems)
        if isinstance(problems, ops.FusedProblem) or len(problems) != 3:
            return ys
        torch.cuda.synchronize()
        h = hashlib.sha256()
        for pr in problems:
            h.update(pr.out.contiguous().cpu().numpy().tobytes())
            if pr.p.stats_out:
                st = next(t for t in pr.keep if isinstance(t, torch.Tensor) and t.data_ptr() == pr.p.stats_out)
                h.update(st.cpu().numpy().tobytes())
        out.append({"launch": " + ".join(_label(pr.p) for pr in problems), "sha256": h.hexdigest()})
        return ys

    ops.conv_fused = digesting
    try:
        with torch.no_grad():
            model.forward_ids(ids[0].to(dev), ref_s.to(dev))
        torch.cuda.synchronize()
    finally:
        ops.conv_fused = orig
    return out


if __name__ == "__main__":
    d = generator_group_digests()
    with open(OUT, "w") as f:
        json.dump(d, f, indent=1)
        f.write("\n")
    print(f"{len(d)} launches -> {OUT}")
