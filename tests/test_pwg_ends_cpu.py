"""What ptxas makes of every instantiation of the frame-rate Parallel WaveGAN residual layer kernel (pwg_fc.cu: the first layer,
which computes first_conv itself, the middle layers, and the last layer, which runs the tail), without a GPU: no spills, a
0-byte stack frame, no wgmma serialization, and shared memory within the H100's 227 KB opt-in limit per block."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parakeet_b200", "csrc")
KERNEL = "pwg_layer_fc_kernel"
MODES = {"0": "first", "1": "middle", "2": "last"}       # template argument of the kernel (FcMode)
SMEM_OPTIN_LIMIT = 227 * 1024
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
def ptxas(nvcc, tmp_path_factory):
    """All ptxas -v lines, and the lines of each instantiation's entry function by mode name."""
    out = tmp_path_factory.mktemp("ptxas_ends") / "pwg_fc.o"
    r = subprocess.run([nvcc] + ARCH + ["-Xptxas", "-v", "-c", os.path.join(CSRC, "pwg_fc.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    lines = r.stderr.splitlines()
    blocks = {}
    for i, ln in enumerate(lines):
        m = re.search(KERNEL + r"ILi(\d)E", ln)
        if "Compiling entry function" in ln and m:
            block = []
            for nxt in lines[i + 1:]:
                if "Compiling entry function" in nxt:
                    break
                block.append(nxt)
            blocks[MODES[m.group(1)]] = block
    return lines, blocks


@pytest.fixture(scope="module")
def dynamic_smem(nvcc, tmp_path_factory):
    d = tmp_path_factory.mktemp("probe_ends")
    probe = d / "probe.cu"
    probe.write_text('#include <stdio.h>\n#include "pwg_fc.cu"\nint main() { printf("%d\\n", pk::fc::kFcSmem); return 0; }\n')
    exe = d / "probe"
    r = subprocess.run([nvcc] + ARCH + ["-I", CSRC, str(probe), os.path.join(CSRC, "pk_common.cu"), "-o", str(exe)],
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-4000:]
    return int(subprocess.run([str(exe)], check=True, capture_output=True, text=True, timeout=60).stdout)


def test_every_mode_is_instantiated(ptxas):
    _, blocks = ptxas
    assert sorted(blocks) == sorted(MODES.values()), sorted(blocks)


@pytest.mark.parametrize("mode", list(MODES.values()))
def test_mode_no_spills_no_stack(ptxas, mode):
    _, blocks = ptxas
    block = blocks[mode]
    spills = [re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln) for ln in block]
    spills = [m for m in spills if m]
    assert spills and all(m.group(1) == "0" and m.group(2) == "0" for m in spills), "\n".join(block)
    assert any("0 bytes stack frame" in ln for ln in block), "\n".join(block)


def test_no_wgmma_serialization_in_any_mode(ptxas):
    lines, _ = ptxas
    remarks = [ln for ln in lines if re.search(r"C75(10|12|20)", ln) and KERNEL in ln]
    assert not remarks, "\n".join(remarks)


@pytest.mark.parametrize("mode", list(MODES.values()))
def test_mode_shared_memory_within_optin_limit(ptxas, dynamic_smem, mode):
    """Every mode launches with the same dynamic shared memory (kFcSmem); with its static shared memory it fits one block."""
    _, blocks = ptxas
    m = [re.search(r"(\d+) bytes smem", ln) for ln in blocks[mode]]
    static = sum(int(x.group(1)) for x in m if x)
    assert dynamic_smem > 0 and static + dynamic_smem <= SMEM_OPTIN_LIMIT, (static, dynamic_smem)
