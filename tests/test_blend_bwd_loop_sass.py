"""Static check of the blend backward's splat loop (no GPU), in the SASS of the default instantiation
blend_bwd_kernel<false,false,false> (blend_bwd.cu):
  * the loop -- the block that holds the MUFU.EX2s, up to its back-branch -- evaluates two splats per iteration in at
    most LOOP_MAX instructions;
  * the flush after the reduce-scatter is the id, the factor, the address, one multiply and the RED: no lane-bit
    arithmetic (SHF / LOP3 / ISETP re-deriving the owner's slot) between the loop's last SHFL and its REDG;
  * the per-splat factor table is gone: every variant but DEPTH's fits in SMEM_MAX bytes of shared memory per CTA."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
LOOP_MAX = 330    # two splats per iteration (323 as built with nvcc 12.9; one splat per iteration took 188)
SMEM_MAX = 20 * 1024
DEFAULT = "blend_bwd_kernelILb0ELb0ELb0E"


def _build():
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    from brush_b200 import build
    build.build()
    return os.path.join(ROOT, "brush_b200", "csrc", "_obj", "blend_bwd.o")


def _loop(obj):
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, timeout=600).stdout
    ins, cur = [], None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+([^;]*);", line)
        if m and cur and DEFAULT in cur:
            ins.append((int(m.group(1), 16), m.group(2).strip()))
    assert ins, "no SASS for the default blend_bwd_kernel"
    first_ex2 = next(i for i, (_, t) in enumerate(ins) if "MUFU.EX2" in t)
    for end in range(first_ex2, len(ins)):
        m = re.search(r"\bBRA\s+(?:!?U?P\w+,\s*)?(0x[0-9a-f]+)", ins[end][1])
        if m and int(m.group(1), 16) <= ins[first_ex2][0]:
            start = next(i for i, (a, _) in enumerate(ins) if a == int(m.group(1), 16))
            return [t for _, t in ins[start:end + 1]]
    raise AssertionError("no back-branch after the loop's first MUFU.EX2")


def _op(text):
    return re.sub(r"^@!?U?P\w+\s+", "", text).split()[0]


def test_splat_loop_instruction_budget():
    loop = _loop(_build())
    ops = [_op(t) for t in loop]
    assert sum(op.startswith("MUFU.EX2") for op in ops) == 4, "two splats per iteration, two pixels each"
    assert len(loop) <= LOOP_MAX, (len(loop), LOOP_MAX)


def test_flush_has_no_lane_arithmetic():
    ops = [_op(t) for t in _loop(_build())]
    last_shfl = max(i for i, op in enumerate(ops) if op.startswith("SHFL"))
    reds = [i for i, op in enumerate(ops) if op.startswith("REDG")]
    assert len(reds) == 1, ops[last_shfl:]
    tail = ops[last_shfl + 1:reds[0]]
    bad = [op for op in tail if op.startswith(("SHF", "LOP3", "ISETP", "LEA.HI", "SEL"))]
    assert not bad, tail


def test_no_factor_table_in_shared_memory():
    obj = _build()
    txt = open(obj + ".ptxas.txt").read()
    found = 0
    for m in re.finditer(r"Compiling entry function '(\S+)'[^\n]*\n(?:[^\n]*\n){0,2}?[^\n]*Used \d+ registers[^\n]*?(\d+) bytes smem", txt):
        name, smem = m.group(1), int(m.group(2))
        if "blend_bwd_kernel" not in name:
            continue
        found += 1
        depth = re.search(r"blend_bwd_kernelILb[01]ELb[01]ELb([01])E", name).group(1) == "1"
        if not depth:
            assert smem <= SMEM_MAX, (name, smem)
    assert found >= 4, txt[:2000]
