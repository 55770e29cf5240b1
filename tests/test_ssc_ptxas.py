"""Compiler invariants of csrc/ssc.cu: no scene-completion grid kernel has a stack frame or spills (the scan's 64 counts per thread
are read twice rather than held, and every other kernel keeps a handful of words in registers)."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
KERNELS = ["k_ssc_count_labels", "k_ssc_count_bits", "k_ssc_scan", "k_ssc_offsets", "k_ssc_emit", "k_ssc_voxelize", "k_ssc_confusion"]


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "ssc.o"
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "lidiff_b200", "csrc", "ssc.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


@pytest.mark.parametrize("kernel", KERNELS)
def test_no_stack_frame_and_no_spills(ptxas_log, kernel):
    m = re.search(rf"Function properties for _Z\d+{kernel}\w*\s*\n\s*(\d+) bytes stack frame, "
                  r"(\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    assert m, f"no ptxas report for {kernel}"
    assert m.groups() == ("0", "0", "0"), f"{kernel}: {m.group(0)}"
