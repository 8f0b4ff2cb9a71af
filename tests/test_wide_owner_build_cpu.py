"""The wide owner kernels (deterministic mode at 5 <= m <= 512) keep their rows in registers: no instantiation may
spill or have a stack frame.  Read from the built library with cuobjdump; no GPU needed."""
import os
import re
import shutil
import subprocess

import pytest

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(REPO, "pymde_b200", "libmde_b200.so")


def _cuobjdump():
    for c in (shutil.which("cuobjdump"), os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")):
        if c and os.path.exists(c):
            return c
    return None


def test_wide_owner_kernels_have_no_spills_or_stack():
    tool = _cuobjdump()
    if tool is None or not os.path.exists(LIB):
        pytest.skip("needs the built library and cuobjdump")
    out = subprocess.run([tool, "-res-usage", LIB], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"Function (\S*(?:distortion_wide_owner_kernel|wide_owner_combine_kernel)\S*):\s*\n\s*(.*)", out)
    # 12 (G, CPL, VW) shapes x MODE 0 and 2, and the segment combine kernel
    assert len(found) == 25, [f for f, _ in found]
    for fn, usage in found:
        assert "STACK:0 " in usage and "LOCAL:0 " in usage, (fn, usage)
