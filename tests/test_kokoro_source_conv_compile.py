"""Compile-time guard for Kokoro's harmonic-source conv kernel (csrc/conv.cu: kokoro_source_conv_kernel), which no numerical test
can see: its 8 x 8 register tile per thread must not spill, and both instantiations (K = 12 / stride 6, K = 1) must fit two 256-thread
CTAs on an SM, as their launch bounds ask."""
import os
import re
import subprocess

import pytest

from mlx_audio_b200 import build

SRC = os.path.join(build.CSRC, "conv.cu")
KERNEL = "kokoro_source_conv_kernel"
THREADS = 256


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("conv") / "conv.o")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", SRC, "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return r.stdout


def test_source_conv_registers_and_spills(ptxas_log):
    pat = re.compile(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                     r"ptxas info\s*: Used (\d+) registers")
    props = [(m.group(1), int(m.group(4)), int(m.group(2)), int(m.group(3))) for m in pat.finditer(ptxas_log) if KERNEL in m.group(1)]
    assert len(props) == 2, f"expected two instantiations of {KERNEL}, found {len(props)}"
    for name, regs, stores, loads in props:
        assert stores == 0 and loads == 0, f"{name} spills {stores} / {loads} bytes"
        assert 2 * THREADS * regs <= 65536, f"{name}: {regs} registers x {THREADS} threads do not fit two CTAs on an SM"
