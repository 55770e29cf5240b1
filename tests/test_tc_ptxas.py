"""Compiler invariants of the wgmma convolution kernels: every k_spconv_tc<NC> compiles for sm_90a without a stack frame or
spills, and without the ptxas advisories that mean its wgmma are serialised (C7520) or that ptxas had to inject warpgroup.arrive /
warpgroup.wait (C7519 / C7517).  Any of these costs the kernel a large share of its speed without changing a result."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")


@pytest.fixture(scope="module")
def ptxas_log(tmp_path_factory):
    if not (os.path.exists(NVCC) or shutil.which(NVCC)):
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "spconv_tc.o"
    r = subprocess.run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "lidiff_b200", "csrc", "spconv_tc.cu"), "-o", str(out)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return r.stdout + r.stderr


def test_no_serialised_or_patched_wgmma(ptxas_log):
    for code in ("C7517", "C7519", "C7520"):
        assert code not in ptxas_log, f"ptxas advisory {code}:\n{ptxas_log}"


@pytest.mark.parametrize("nc", [32, 64, 96, 128])
def test_no_stack_frame_and_no_spills(ptxas_log, nc):
    m = re.search(rf"Function properties for _ZN2tc11k_spconv_tcILi{nc}EEEvNS_6ParamsE\s*\n\s*(\d+) bytes stack frame, "
                  r"(\d+) bytes spill stores, (\d+) bytes spill loads", ptxas_log)
    assert m, f"no ptxas report for k_spconv_tc<{nc}>"
    assert m.groups() == ("0", "0", "0"), f"k_spconv_tc<{nc}>: {m.group(0)}"
