"""Compile-time guard for the fused conv kernel: what ptxas makes of it, which no numerical test can see.

- Its wgmmas must compile into an asynchronous pipeline.  ptxas silently serialises wgmma (every HGMMA followed by a wait for it)
  when the MMA issue sits on a path it cannot prove warp-uniform (warning C7520) or when it runs out of registers for the in-flight
  accumulators (C7512).  Results are unchanged either way.
- Spills must not grow.  The target is zero; the worker loops still spill a few bytes at their 128-register budget (the cold `sinf`
  fallback of the Snake sine and per-tile bookkeeping), so this checks the current bound, and the bound only ever goes down.
- The kernel must launch at exactly REG_LAUNCH registers per thread: the setmaxnreg re-allocation between the warpgroups is balanced
  against that count, and a kernel compiled below it would leave the worker warpgroups waiting for registers that never come free.
"""
import os
import re
import subprocess

import pytest

from mlx_audio_b200 import build

SRC = os.path.join(build.CSRC, "conv_fused.cu")
# (spill stores, spill loads) in bytes per instantiation: DBG = false is the production kernel, DBG = true the timeline build
SPILL_BOUND = {"conv_fused_kernelILb0E": (44, 44), "conv_fused_kernelILb1E": (128, 156)}
VARIANTS = 4 * 2                      # mma_tile instantiations per kernel: NB = 1..4 x (bf16, fp16)


@pytest.fixture(scope="module")
def compiled(tmp_path_factory):
    obj = str(tmp_path_factory.mktemp("conv_fused") / "conv_fused.o")
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


@pytest.mark.parametrize("key", sorted(SPILL_BOUND))
def test_conv_fused_wgmma_is_pipelined(compiled, key):
    obj, log = compiled
    serialised = [l for l in log.splitlines() if re.search(r"\(C75\d\d\)", l) and "serialized" in l and key in l]
    assert not serialised, f"ptxas serialises the wgmmas of {key}:\n" + "\n".join(serialised)
    sass = _kernel_sass(obj, key)
    hgmma = len(re.findall(r"\bHGMMA\.", sass))
    waits = len(re.findall(r"\bWARPGROUP\.DEPBAR\b", sass))
    assert hgmma > 0
    # per variant: one wait per tap step (for the previous step's group) and the drain at the end of the tile
    assert waits <= 2 * VARIANTS, f"{waits} WARPGROUP.DEPBAR for {hgmma} HGMMA in {VARIANTS} variants: the wgmma issue is serialised"


@pytest.mark.parametrize("key", sorted(SPILL_BOUND))
def test_conv_fused_registers_and_spills(compiled, key):
    _, log = compiled
    props = [v for name, v in _properties(log).items() if key in name]
    assert len(props) == 1, f"no ptxas register / spill report for {key}"
    regs, stores, loads = props[0]
    max_stores, max_loads = SPILL_BOUND[key]
    assert stores <= max_stores and loads <= max_loads, f"{key} spills {stores} / {loads} bytes (bound {max_stores} / {max_loads})"
    reg_launch = int(re.search(r"constexpr int REG_LAUNCH = (\d+);", open(SRC).read()).group(1))
    assert regs == reg_launch, f"{key} compiled to {regs} registers; the setmaxnreg budget assumes {reg_launch}"
