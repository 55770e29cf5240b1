"""Compiler invariants of the multi-CTA farthest point sampling kernels: k_fps_coop and k_fps_cluster keep every point they own and
its running distance in registers under __launch_bounds__(1024, 1), so at most 64 registers per thread.  A stack frame or a spill
would move those arrays to local memory and silently undo that design without changing a result."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
KERNELS = {"k_fps_coop": "_Z10k_fps_coopPKdiiPiP7FpsBestPj", "k_fps_cluster": "_Z13k_fps_clusterPKdPKliiPi"}


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "dense.o"
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "lidiff_b200", "csrc", "dense.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_no_stack_frame_and_no_spills(ptxas_log, kernel):
    m = re.search(rf"Function properties for {KERNELS[kernel]}\s*\n\s*(\d+) bytes stack frame, "
                  r"(\d+) bytes spill stores, (\d+) bytes spill loads\s*\n[^\n]*Used (\d+) registers", ptxas_log)
    assert m, f"no ptxas report for {kernel}"
    assert m.groups()[:3] == ("0", "0", "0"), f"{kernel}: {m.group(0)}"
    assert int(m.group(4)) <= 64, f"{kernel}: {m.group(4)} registers, above the 64 of a 1024-thread CTA"
