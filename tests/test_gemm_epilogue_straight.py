"""The epilogue of the 256-channel wgmma conv-GEMM runs as straight-line code.  Each SM runs one CTA whose two consumer
warpgroups drain their accumulators while no MMA issues, so every instruction a column group issues is tensor-core idle
time.  epilogue_wide (gemm_epilogue.cuh) forms one base pointer per row and plane, does no column bounds work (256-channel
tiles run for N % 256 == 0 only) and turns kernel-uniform choices into predicates once per tile or row.  Whether the
compiler keeps it so is checked on the built library, for the four instances the benchmark's default workload runs
(QKV: mode 3 / prec 0, conv_1: 1 / 1, O: 4 / 0, conv_2: 4 / 1):
  * column chains: the stores of one plane of one row, [R + imm] with imm stepping by one column group (32 bytes for fp32
    pairs, 16 for 2-byte words).  Between two stores of a chain there is no 64-bit null test of a pointer
    (ISETP .EX against RZ) and no integer min / max;
  * at most one integer min per row in the epilogue (the row clamp of the loads);
  * at most MAX_BRA_PER_ROW branches per row between the first and the last store of the epilogue;
  * the column-group period shrank by at least 30 %: the median distance between two stores of a chain (and, in the
    residual instances, between consecutive residual loads).  The parent commit's code formed every address per column
    group, so it had no chains; its period is the median distance between a store and the same plane's store of the next
    column group, counted in stores (CUDA 12.9):
        instance         parent: store / residual load    this code: store / residual load
        mode 3 / prec 0  53 / -                           12 / -
        mode 1 / prec 1  78 / -                           28 / -
        mode 4 / prec 0  121 / 88                         26 / 32
        mode 4 / prec 1  121 / 88                         26 / 32
Needs no GPU."""
import os
import re
import shutil
import statistics
import subprocess

import pytest

# (mode, prec) -> the parent commit's column-group period: the median instructions between two stores of a column chain
# (store) and between consecutive residual loads (load), as measured by _metrics on its SASS
PARENT_PERIOD = {(3, 0): {"store": 53}, (1, 1): {"store": 78}, (4, 0): {"store": 121, "load": 88},
                 (4, 1): {"store": 121, "load": 88}}
MAX_SHARE = 0.7                # the period must shrink by at least 30 %
MAX_BRA_PER_ROW = 12           # CUDA 12.9 builds 17 in QKV (RoPE: one per 64-column head and body), 5-6 elsewhere

_INS = re.compile(r"^\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*;")
_ADDR = re.compile(r"\[(R\d+)\.64(?:\+(0x[0-9a-f]+))?\]")
_MIN = re.compile(r"^(?:@!?U?P\w+\s+)?(VIMNMX|VIADDMNMX|IMNMX)")
_NULL_TEST = re.compile(r"ISETP\S*\.EX\b.*\bRZ\b")


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


def _opcode(ins):
    return (ins.split(None, 1)[1] if ins.startswith("@") else ins).split(None, 1)[0]


def _metrics(ins):
    """Column-loop figures of one 256-channel instance's epilogue (from the second named warpgroup barrier on: the first
    orders stage_epi_vectors, the second opens epilogue_tile)"""
    bars = [i for i, x in enumerate(ins) if re.match(r"BAR\.SYNC\S* R\d+, 0x80", x)]
    assert len(bars) >= 2, "named barriers of stage_epi_vectors / epilogue_tile not found"
    ep = ins[bars[1]:]
    stores = []                                        # (position, base register, offset, column-group stride)
    for i, x in enumerate(ep):
        op = _opcode(x)
        if op.startswith("STG"):
            m = _ADDR.search(x)
            if m:
                stores.append((i, m.group(1), int(m.group(2) or "0", 16), 32 if op.startswith("STG.E.64") else 16))
    # chains: each store to the store of the next column group through the same base register
    links = []
    for k, (i, reg, off, step) in enumerate(stores):
        for i2, reg2, off2, step2 in stores[k + 1:]:
            if reg2 == reg and step2 == step and off2 == off + step:
                links.append((i, i2))
                break
    loads = [i for i, x in enumerate(ep) if _opcode(x).startswith("LDG.E.64")]
    first, last = stores[0][0], stores[-1][0]
    return {
        "store": statistics.median(i2 - i for i, i2 in links) if links else None,
        "load": statistics.median(b - a for a, b in zip(loads, loads[1:])) if len(loads) > 1 else None,
        "null_tests": sum(1 for i, i2 in links for x in ep[i + 1:i2] if _NULL_TEST.search(x)),
        "mins_in_chains": sum(1 for i, i2 in links for x in ep[i + 1:i2] if _MIN.match(x)),
        "mins": sum(1 for x in ep[first:last] if _MIN.match(x)),
        "bra": sum(1 for x in ep[first:last] if _opcode(x).startswith("BRA")),
        "links": len(links),
    }


def _instances(sass):
    out = {}
    for name, ins in _functions(sass).items():
        m = re.search(r"gemm_wgmma_kernelILi(\d+)ELi(\d+)ELi(\d+)E", name)
        if m and int(m.group(1)) == 256 and (int(m.group(2)), int(m.group(3))) in PARENT_PERIOD:
            out[(int(m.group(2)), int(m.group(3)))] = _metrics(ins)
    return out


def test_wide_epilogue_is_straight_line():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump (CUDA toolkit) not found")
    import __graft_entry__ as g
    g.build()
    sass = subprocess.run([tool, "-sass", g.OUT], capture_output=True, text=True, check=True).stdout
    found = _instances(sass)
    assert sorted(found) == sorted(PARENT_PERIOD), f"expected the instances {sorted(PARENT_PERIOD)}, found {sorted(found)}"
    bad = []
    for key, got in sorted(found.items()):
        inst = f"bn256/mode{key[0]}/prec{key[1]}"
        if got["links"] < 64:
            bad.append(f"{inst}: {got['links']} column-chain store pairs, expected at least one chain per row")
        if got["null_tests"]:
            bad.append(f"{inst}: {got['null_tests']} 64-bit pointer null tests inside the column chains")
        if got["mins_in_chains"] or got["mins"] > 2:
            bad.append(f"{inst}: {got['mins']} integer min / max between the epilogue's first and last store, "
                       f"{got['mins_in_chains']} inside the column chains (the row clamp needs one per row)")
        if got["bra"] > 2 * MAX_BRA_PER_ROW:
            bad.append(f"{inst}: {got['bra']} branches between the epilogue's first and last store "
                       f"(> {MAX_BRA_PER_ROW} per row)")
        for kind, parent in PARENT_PERIOD[key].items():
            if got[kind] is None or got[kind] > MAX_SHARE * parent:
                bad.append(f"{inst}: column-group period ({kind}) {got[kind]} instructions, parent {parent} "
                           f"(must be <= {MAX_SHARE * parent:.0f})")
    assert not bad, "\n".join(bad)


if __name__ == "__main__":                # python tests/test_gemm_epilogue_straight.py <sass dump>: print the figures
    import sys
    for k, v in sorted(_instances(open(sys.argv[1]).read()).items()):
        print(k, v)
