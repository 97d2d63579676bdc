"""The residual epilogues of the 256-channel wgmma conv-GEMM keep their global loads in flight.  Each consumer thread reads
64 residual pairs per tile (32 column groups, two rows).  When each pair is consumed a few instructions after its load
issues, the thread waits out one HBM round trip per column group, in series; on H100 80GB HBM3 that was most of the time
the residual + LayerNorm tiles held an SM beyond their MMAs (DESIGN.md §5).  epilogue_tile (gemm_epilogue.cuh) loads them
through a ring of registers several column groups ahead, and reads the adaLN shift / scale of the LayerNorm pass from
shared memory.  Whether the loads stay ahead is a compiler decision, so it is checked on the built library: in the SASS of
every 256-channel EM_LN / EM_RESID / EM_SILU_OUT instance, the epilogue issues exactly the 64 residual pair loads, and
the median distance from one of them to the first instruction that reads its registers is far above the 7-11
instructions of loads consumed where they are issued.  Needs no GPU."""
import os
import re
import shutil
import statistics
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EM_LN, EM_RESID, EM_SILU_OUT = 4, 5, 6
RESID_PAIRS = 64               # per thread and tile: 2 rows x 32 column groups
# instructions from a residual load to its first use.  A column group of these epilogues is ~75-100 instructions and the
# loads run 8 groups ahead: the median is 630-780 with CUDA 12.9.  Consumed where issued, it was 7 (EM_LN) and 11.
MIN_MEDIAN_DISTANCE = 200

_INS = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;")
_REG = re.compile(r"\bR(\d+)\b")


def _cuobjdump():
    for cand in (os.path.join(os.path.dirname(os.environ.get("NVCC", "")), "cuobjdump"), "/usr/local/cuda/bin/cuobjdump",
                 shutil.which("cuobjdump") or ""):
        if cand and os.path.isfile(cand):
            return cand
    return None


def _functions(sass):
    out = {}
    for chunk in re.split(r"\n\s*Function : ", sass)[1:]:
        name, body = chunk.split("\n", 1)
        out[name.strip()] = [m.group(1) for m in map(_INS.match, body.split("\n")) if m]
    return out


def _operands(ins):
    """(opcode, operands) of one SASS instruction, without its predicate guard"""
    if ins.startswith("@"):
        ins = ins.split(None, 1)[1]
    parts = ins.split(None, 1)
    return parts[0], (parts[1].split(",") if len(parts) > 1 else [])


def _first_use(ins, i, regs):
    """instructions from ins[i] to the first later one that reads any of regs (straight-line order)"""
    for d, x in enumerate(ins[i + 1:], 1):
        op, ops = _operands(x)
        srcs = ops if op.startswith(("ST", "RED", "ATOM")) else ops[1:]
        if any(int(r) in regs for s in srcs for r in _REG.findall(s)):
            return d
    return None


def test_residual_loads_run_ahead_of_their_use():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    import __graft_entry__ as g
    g.build()
    sass = subprocess.run([tool, "-sass", g.OUT], capture_output=True, text=True, check=True).stdout
    checked, bad = [], []
    for name, ins in _functions(sass).items():
        m = re.search(r"gemm_wgmma_kernelILi(\d+)ELi(\d+)ELi(\d+)E", name)
        if not m or int(m.group(1)) != 256 or int(m.group(2)) not in (EM_LN, EM_RESID, EM_SILU_OUT):
            continue
        inst = f"bn256/mode{m.group(2)}/prec{m.group(3)}"
        checked.append(inst)
        # the epilogue follows the second named warpgroup barrier: the first orders stage_epi_vectors, the second
        # opens epilogue_tile
        bars = [i for i, x in enumerate(ins) if re.match(r"BAR\.SYNC\S* R\d+, 0x80", x)]
        assert len(bars) >= 2, f"{inst}: named barriers of stage_epi_vectors / epilogue_tile not found"
        dist = []
        for i in range(bars[1], len(ins)):
            op, ops = _operands(ins[i])
            if op.startswith("LDG.E.64"):
                rd = int(_REG.search(ops[0]).group(1))
                dist.append(_first_use(ins, i, {rd, rd + 1}))
        if len(dist) != RESID_PAIRS:
            bad.append(f"{inst}: {len(dist)} 8-byte global loads in the epilogue, expected the {RESID_PAIRS} residual "
                       "pairs only (the LayerNorm modulate loop reads shift / scale from shared memory)")
            continue
        used = [d for d in dist if d is not None]
        med = statistics.median(used) if used else 0
        if med < MIN_MEDIAN_DISTANCE:
            bad.append(f"{inst}: residual loads consumed a median {med} instructions after issue "
                       f"(< {MIN_MEDIAN_DISTANCE})")
    assert len(checked) == 5, f"expected the 5 256-channel residual instances, found {checked}"
    assert not bad, "\n".join(bad)
