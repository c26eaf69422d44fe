"""Static check of the blend kernels' row staging (no GPU): in the SASS of every blend_{fwd,bwd}_kernel the bulk copies
of a batch issue back to back from uniform registers, at most ISSUE_MAX instructions apart, with no per-row ELECT
waterfall (blend_common.cuh, issue_rows_tma)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
ISSUE_MAX = 10   # instructions per staged row (9 as built with nvcc 12.9; 14 for the per-lane ELECT waterfall)


@pytest.mark.parametrize("unit", ["blend_fwd", "blend_bwd"])
def test_row_issue_instruction_count(unit):
    if not os.path.exists(CUOBJDUMP):
        pytest.skip("cuobjdump not available")
    from brush_b200 import build
    build.build()
    obj = os.path.join(ROOT, "brush_b200", "csrc", "_obj", unit + ".o")
    out = subprocess.run([CUOBJDUMP, "-sass", obj], capture_output=True, text=True, timeout=600).stdout
    kernels = {}
    cur = None
    for line in out.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1)
            kernels[cur] = []
            continue
        m = re.match(r"\s+/\*[0-9a-f]{4}\*/\s+(?:@!?U?P\w+\s+)?([A-Z0-9_.]+)", line)
        if m and cur:
            kernels[cur].append(m.group(1))
    assert kernels
    for name, ops in kernels.items():
        at = [i for i, op in enumerate(ops) if op.startswith("UBLKCP")]
        assert len(at) >= 32, (name, len(at))
        gaps = [b - a for a, b in zip(at, at[1:])]
        # the unrolled rows of one batch: consecutive copies of one staging site
        rows = sorted(gaps)[: len(gaps) * 3 // 4]
        assert max(rows) <= ISSUE_MAX, (name, sorted(gaps)[:40])
        # a waterfall elects a lane for every copy
        assert sum(op.startswith("ELECT") for op in ops) * 8 < len(at), name
