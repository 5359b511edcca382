"""Compile-time guard for the incremental Mimi kernels (mimi_stream.cu): they build for sm_90a with the library's flags and ptxas reports no
register spills for any of them."""
import os
import re
import subprocess

from mlx_audio_b200 import build

KERNELS = ("conv_stream_kernel", "convtr_stream_kernel", "convtr_stream_dw_kernel", "ring_rope_kv_kernel", "ring_attn_kernel",
           "stream_advance_kernel")


def test_mimi_stream_kernels_compile_without_spills(tmp_path):
    assert "mimi_stream.cu" in build.SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "mimi_stream.cu"), "-o", str(tmp_path / "mimi_stream.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    found = {}
    for m in re.finditer(r"Function properties for (\S+)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", r.stdout):
        for k in KERNELS:
            if re.search(rf"\d{k}E", m.group(1)):
                found[k] = (int(m.group(3)), int(m.group(4)))
    assert sorted(found) == sorted(KERNELS), r.stdout
    assert all(v == (0, 0) for v in found.values()), found
