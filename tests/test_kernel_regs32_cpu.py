"""Register guard for the 32-row instantiation of the decode kernel (CPU only: nvcc + cuobjdump, ~1 minute).
tools/spill_report.py prints it with the suffix _r32; the bounds of the 16-row kernel's (test_kernel_regs_cpu.py)."""
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(shutil.which("nvcc") is None or shutil.which("cuobjdump") is None, reason="needs the CUDA toolkit")
def test_32_row_phase_functions_do_not_spill():
    out = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "spill_report.py")], capture_output=True, text=True,
                         timeout=600)
    assert out.returncode == 0, out.stderr[-2000:]
    rows = {}
    for line in out.stdout.splitlines():
        m = re.match(r"(\w+)\s+n_ins\s+(\d+)\s+maxR\s+(-?\d+)\s+STL\s+(\d+)\s+LDL\s+(\d+)", line)
        if m:
            rows[m.group(1)] = tuple(int(m.group(i)) for i in (2, 3, 4, 5))
    # the 32-row GEMM phase inlines its activation staging (decode_engine.cu, stage_acts): gemm_phase_r32 covers both
    assert "stage_acts_r32" not in rows, out.stdout
    for fn in ("gemm_phase_r32", "attn_item_r32", "attn_scores_r32"):
        n_ins, max_r, stl, ldl = rows[fn]
        assert stl == 0 and ldl == 0, f"{fn} spills (STL {stl}, LDL {ldl}):\n{out.stdout}"
    assert rows["producer_loop_r32"][1] < 40
    assert rows["kernel_r32"][2] <= 12, out.stdout
