"""The solver step's head and vector kernels keep their accumulators and in-flight loads in registers: ptxas reports no
spill stores for either, and the built library gives them no local memory.  No GPU needed: ptxas -v on the source,
cuobjdump -res-usage on the library."""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, "pymde_b200", "libmde_b200.so")
SRC = os.path.join(REPO, "pymde_b200", "csrc", "mde_solver.cu")
KERNELS = ("step_head_kernel", "step_vec_kernel")


def _tool(name):
    for c in (shutil.which(name), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", name)):
        if c and os.path.exists(c):
            return c
    return None


def test_step_kernels_do_not_spill():
    nvcc = _tool("nvcc")
    if nvcc is None:
        pytest.skip("needs nvcc")
    with tempfile.TemporaryDirectory() as tmp:
        out = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v",
                              "-c", SRC, "-o", os.path.join(tmp, "s.o")], capture_output=True, text=True, check=True)
    # ptxas prints, per entry: "Function properties for NAME" then "N bytes stack frame, S bytes spill stores, ..."
    found = re.findall(r"Function properties for (\S+)\n.*?(\d+) bytes spill stores", out.stderr)
    step = [(fn, int(sp)) for fn, sp in found if any(k in fn for k in KERNELS)]
    assert len(step) == 2, step
    for fn, spill in step:
        assert spill == 0, (fn, spill)


def test_built_step_kernels_use_no_local_memory():
    tool = _tool("cuobjdump")
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*(?:%s)\S*):\s*\n\s*(.*)" % "|".join(KERNELS), out)
    assert len(found) == 2, [f for f, _ in found]
    for fn, usage in found:
        assert "LOCAL:0 " in usage, (fn, usage)
