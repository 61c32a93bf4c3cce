"""What ptxas makes of the flagship residual-layer kernel (pwg_fc.cu), checked without a GPU: its wgmma chains must not be
serialized (remarks C7510 / C7520: every tensor-core instruction would wait for the previous one) and it must not spill."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parakeet_b200", "csrc")
KERNEL = "pwg_layer_fc_kernel"


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


@pytest.fixture(scope="module")
def ptxas_report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    out = tmp_path_factory.mktemp("ptxas") / "pwg_fc.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(CSRC, "pwg_fc.cu"), "-o", str(out)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _kernel_block(report):
    """The ptxas lines from the kernel's 'Compiling entry function' line up to the next entry function."""
    lines = report.splitlines()
    start = [i for i, ln in enumerate(lines) if "Compiling entry function" in ln and KERNEL in ln]
    assert start, f"ptxas reported no entry function {KERNEL}"
    block = []
    for ln in lines[start[0] + 1:]:
        if "Compiling entry function" in ln:
            break
        block.append(ln)
    return block


def test_pwg_layer_fc_wgmma_not_serialized(ptxas_report):
    remarks = [ln for ln in ptxas_report.splitlines() if re.search(r"C75[12]0", ln) and KERNEL in ln]
    assert not remarks, "\n".join(remarks)


def test_pwg_layer_fc_no_spills(ptxas_report):
    block = _kernel_block(ptxas_report)
    spills = [ln for ln in block if "spill" in ln]
    assert spills, "ptxas -v printed no spill line for the kernel"
    for ln in spills:
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        assert m and m.group(1) == "0" and m.group(2) == "0", ln
    assert any("0 bytes stack frame" in ln for ln in block), "\n".join(block)
