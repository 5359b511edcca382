"""Compile-time guard for the persistent ALBERT kernel (csrc/albert.cu): what ptxas makes of it, which no numerical test can see.

- Its wgmmas must stay asynchronous.  ptxas silently serialises wgmma when the MMA issue sits on a path it cannot prove warp-uniform
  (warning C7520) or when it runs out of registers for the in-flight accumulators (C7512).  Results are unchanged either way.
- The production kernel must not spill.
- It launches one CTA of THREADS threads per SM: its register count must leave that CTA resident (THREADS * registers <= 64 K).
"""
import os
import re
import subprocess

import pytest

from mlx_audio_b200 import build

SRC = os.path.join(build.CSRC, "albert.cu")
PROD = "albert_kernelILb0EE"             # the timeline build (ILb1EE) is a profiling aid


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("albert") / "albert.o")
    cmd = [build._nvcc(), *build.NVCC_FLAGS, "-c", SRC, "-o", obj]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    assert r.returncode == 0, r.stdout
    return obj, r.stdout


def _properties(log):
    """{mangled kernel name: (registers, spill store bytes, spill load bytes)} from the ptxas -v log."""
    pat = re.compile(r"Function properties for (\S+)\n\s*\d+ bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                     r"ptxas info\s*: Used (\d+) registers")
    return {m.group(1): (int(m.group(4)), int(m.group(2)), int(m.group(3))) for m in pat.finditer(log)}


def _kernel_sass(obj, key):
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    sass = subprocess.run([cuobjdump, "-sass", obj], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, check=True).stdout
    funcs = re.split(r"\n\s*Function : ", sass)
    mine = [f for f in funcs if f.startswith("_Z") and key in f.split("\n", 1)[0]]
    assert len(mine) == 1, f"{key} not found in the SASS"
    return mine[0]


def test_albert_wgmma_is_not_serialised(compiled):
    obj, log = compiled
    serialised = [l for l in log.splitlines() if re.search(r"\(C75(20|12)\)", l) and "albert_kernel" in l]
    assert not serialised, "ptxas serialises the wgmmas of the ALBERT kernel:\n" + "\n".join(serialised)
    sass = _kernel_sass(obj, PROD)
    assert len(re.findall(r"\bHGMMA\.", sass)) > 0


def test_albert_registers_and_spills(compiled):
    _, log = compiled
    props = [v for name, v in _properties(log).items() if PROD in name]
    assert len(props) == 1, "no ptxas register / spill report for the production ALBERT kernel"
    regs, stores, loads = props[0]
    assert stores == 0 and loads == 0, f"the ALBERT kernel spills {stores} / {loads} bytes"
    threads = int(re.search(r"constexpr int THREADS = (\d+);", open(SRC).read()).group(1))
    assert threads * regs <= 65536, f"{regs} registers x {threads} threads do not fit one CTA on an SM"
