"""Compile-time guard for the continuous-batching kernels: the three attention / cache kernels that take per-row cache positions and a
slot map (lm.cu, attn_prefill.cu) and the slot-advance kernel build for sm_90a with the library's flags, and ptxas reports no spills."""
import os
import re
import subprocess

import pytest

from mlx_audio_b200 import build

KERNELS = {"lm.cu": ["qknorm_rope_cache_kernel", "attn_decode_kernel", "slot_advance_kernel"],
           "attn_prefill.cu": ["attn_prefill_kernel"]}


@pytest.mark.parametrize("src", sorted(KERNELS))
def test_session_kernels_compile_without_spills(tmp_path, src):
    assert src in build.SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, src), "-o", str(tmp_path / "k.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    props = re.findall(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout)
    for name in KERNELS[src]:
        found = [p for p in props if name in p[0]]
        assert found, (name, r.stdout)
        for mangled, stack, st, ld in found:
            assert (int(st), int(ld)) == (0, 0), (mangled, stack, st, ld)
