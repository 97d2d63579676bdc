"""The wgmma conv-GEMM kernels keep their epilogue in registers.  Beside the 128 fp32 accumulators of a 256-channel tile the
consumer warps have little room, and values the epilogue spills to local memory miss the small L1 left beside the
pipeline stages: the epilogue then waits on L2 round trips.  Whether that happens is a compiler decision (the per-row
column base of epilogue_tile, gemm_epilogue.cuh, is what prevents it with CUDA 12.9), so it is checked on the built
library: the stack frame of every gemm_wgmma_kernel instance, from cuobjdump's resource usage.  Needs no GPU."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EM_LN = 4                      # the fused-LayerNorm epilogue instance: its three passes over the row keep 32 bytes spilled
STACK_BUDGET = {EM_LN: 32}     # bytes per thread; every other instance: none


def _cuobjdump():
    for cand in (os.path.join(os.path.dirname(os.environ.get("NVCC", "")), "cuobjdump"), "/usr/local/cuda/bin/cuobjdump",
                 shutil.which("cuobjdump") or ""):
        if cand and os.path.isfile(cand):
            return cand
    return None


def test_gemm_kernels_do_not_spill():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    import __graft_entry__ as g
    g.build()
    out = subprocess.run([tool, "-res-usage", g.OUT], capture_output=True, text=True, check=True).stdout
    found = re.findall(r"gemm_wgmma_kernelILi(\d+)ELi(\d+)ELi(\d+)E\S*\s+REG:(\d+) STACK:(\d+)", out)
    assert len(found) == 36, f"expected the 36 gemm_wgmma_kernel instances, found {len(found)}"
    over = [(f"bn{bn}/mode{mode}/prec{prec}", int(stack)) for bn, mode, prec, _, stack in found
            if int(stack) > STACK_BUDGET.get(int(mode), 0)]
    assert not over, f"stack frame (spilled registers) above budget: {over}"
