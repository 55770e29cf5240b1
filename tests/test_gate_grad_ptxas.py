"""Compiler invariants of lb2_segment_dot's kernels: every instantiation of k_segment_dot_chunks (vector / scalar rows, with / without
the second operand) and k_segment_dot_reduce compiles for sm_90a without a stack frame or spills.  The chunk kernel keeps a chunk's row
indices and several rows' loads in registers; a spill would put them in local memory, on the path of every row."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


def test_segment_dot_kernels_have_no_stack_frame_and_no_spills(tmp_path):
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip("nvcc not available")
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "lidiff_b200", "csrc", "gate_grad.cu"), "-o", str(tmp_path / "gate_grad.o")],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    log = r.stdout + r.stderr
    found = re.findall(r"Function properties for (\S*k_segment_dot\S*)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, "
                       r"(\d+) bytes spill loads", log)
    assert len(found) == 5, log                              # 4 chunk kernels + the reduction
    for name, *counts in found:
        assert counts == ["0", "0", "0"], (name, counts)
