"""Compile-time guard for the streaming-state kernel (stream.cu): it builds for sm_90a with the library's flags and ptxas reports no
spills -- it is a plain row-range copy / add, with nothing that should need local memory."""
import os
import re
import subprocess

from mlx_audio_b200 import build


def test_stream_rows_kernel_compiles_without_spills(tmp_path):
    assert "stream.cu" in build.SOURCES
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", os.path.join(build.CSRC, "stream.cu"), "-o", str(tmp_path / "stream.o")]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    m = re.search(r"Function properties for (\S*stream_rows_kernel\S*)\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads",
                  r.stdout)
    assert m, r.stdout
    assert (int(m.group(2)), int(m.group(3)), int(m.group(4))) == (0, 0, 0), m.group(0)
