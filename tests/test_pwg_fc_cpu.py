"""What ptxas makes of the frame-rate Parallel WaveGAN residual layer kernel (pwg_fc.cu), without a GPU: no spills, no wgmma
serialization, and its shared memory within the H100's 227 KB opt-in limit per block."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parakeet_b200", "csrc")
KERNEL = "pwg_layer_fc_kernel"
SMEM_OPTIN_LIMIT = 227 * 1024         # cudaDevAttrMaxSharedMemoryPerBlockOptin on the H100
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand) and os.access(cand, os.X_OK):
            return cand
    return None


@pytest.fixture(scope="module")
def nvcc():
    n = _nvcc()
    if n is None:
        pytest.skip("nvcc not available")
    return n


@pytest.fixture(scope="module")
def kernel_block(nvcc, tmp_path_factory):
    """ptxas -v lines of the kernel's entry function."""
    out = tmp_path_factory.mktemp("ptxas") / "pwg_fc.o"
    r = subprocess.run([nvcc] + ARCH + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "pwg_fc.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    lines = r.stderr.splitlines()
    start = [i for i, ln in enumerate(lines) if "Compiling entry function" in ln and KERNEL in ln]
    assert start, f"ptxas reported no entry function {KERNEL}"
    block = []
    for ln in lines[start[0] + 1:]:
        if "Compiling entry function" in ln:
            break
        block.append(ln)
    return lines, block


def test_layer_kernel_no_spills(kernel_block):
    _, block = kernel_block
    spills = [re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln) for ln in block]
    spills = [m for m in spills if m]
    assert spills and all(m.group(1) == "0" and m.group(2) == "0" for m in spills), "\n".join(block)
    assert any("0 bytes stack frame" in ln for ln in block), "\n".join(block)


def test_layer_kernel_no_wgmma_serialization(kernel_block):
    lines, _ = kernel_block
    remarks = [ln for ln in lines if re.search(r"C75(10|12|20)", ln) and KERNEL in ln]
    assert not remarks, "\n".join(remarks)


def test_layer_kernel_shared_memory_within_optin_limit(nvcc, kernel_block, tmp_path):
    """The dynamic shared memory the host asks for at launch, plus any static shared memory, fits one block."""
    _, block = kernel_block
    m = [re.search(r"(\d+) bytes smem", ln) for ln in block]
    static = sum(int(x.group(1)) for x in m if x)
    probe = tmp_path / "probe.cu"
    probe.write_text('#include <stdio.h>\n#include "pwg_fc.cu"\nint main() { printf("%d\\n", pk::fc::kFcSmem); return 0; }\n')
    exe = tmp_path / "probe"
    r = subprocess.run([nvcc] + ARCH + ["-I", CSRC, str(probe), os.path.join(CSRC, "pk_common.cu"), "-o", str(exe)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    dynamic = int(subprocess.run([str(exe)], check=True, capture_output=True, text=True, timeout=60).stdout)
    assert dynamic > 0 and static + dynamic <= SMEM_OPTIN_LIMIT, (static, dynamic)
