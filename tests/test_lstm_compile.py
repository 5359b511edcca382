"""Compile-time guard for the BiLSTM recurrence kernel (csrc/lstm.cu): what ptxas makes of it, which no numerical test can see.

- W_h lives in registers (128 per thread): the kernel must not spill, and one 256-thread CTA must fit an SM (256 * registers <= 64 K).
- Each lane reads only its own 16 columns of h per step, as 4 LDS.128.  More than 8 in the kernel means a return to reading the whole h
  per gate row, which multiplies the shared-memory traffic of every step.
"""
import os
import re
import subprocess

import pytest

from mlx_audio_b200 import build

SRC = os.path.join(build.CSRC, "lstm.cu")
KERNEL = "lstm_bidir_kernel"
THREADS = 256


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("lstm") / "lstm.o")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", SRC, "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return obj, r.stdout


def test_lstm_registers_and_spills(compiled):
    _, log = compiled
    pat = re.compile(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                     r"ptxas info\s*: Used (\d+) registers")
    props = [(int(m.group(4)), int(m.group(2)), int(m.group(3))) for m in pat.finditer(log) if KERNEL in m.group(1)]
    assert len(props) == 1, "no ptxas register / spill report for the LSTM kernel"
    regs, stores, loads = props[0]
    assert stores == 0 and loads == 0, f"the LSTM kernel spills {stores} / {loads} bytes"
    assert THREADS * regs <= 65536, f"{regs} registers x {THREADS} threads do not fit one CTA on an SM"


def test_lstm_reads_each_lanes_columns_only(compiled):
    obj, _ = compiled
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    funcs = [f for f in re.split(r"\n\s*Function : ", sass) if f.startswith("_Z") and KERNEL in f.split("\n", 1)[0]]
    assert len(funcs) == 1, f"{KERNEL} not found in the SASS"
    n = len(re.findall(r"\bLDS\.128\b", funcs[0]))
    assert 0 < n <= 8, f"the LSTM kernel has {n} LDS.128"
