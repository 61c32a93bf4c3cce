"""WaveFlow density direction (ConditionalWaveFlow.forward, WaveFlowLoss) without a GPU: the oracle against vectors the
reference's own code produced, the oracle's forward / inverse identity, what ptxas makes of the new layer kernel, the C-ABI
struct layouts and the input errors of the host class."""
import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest
import torch

from conftest import rel_err
from parakeet_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_executed_waveflow_forward.npz")
VECTORS = {"a": (64, 4), "b": (128, 5)}          # tag: (channels, parameter seed)
TOL = 2e-6        # to rounding: the reference sums the layers' skips with stack + sum, the oracle one at a time


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


@pytest.mark.parametrize("tag", sorted(VECTORS))
def test_oracle_forward_and_loss_equal_executed_reference(g, tag):
    from oracle import waveflow as owf
    from oracle import waveflow_forward as owff
    channels, seed = VECTORS[tag]
    folded = owf.fold_weight_norm(owf.synth_params(seed, channels=channels))
    audio, mel = torch.from_numpy(g[f"{tag}_audio"]), torch.from_numpy(g[f"{tag}_mel"])
    with torch.no_grad():
        z, log_det = owff.waveflow_forward(folded, audio, mel)
    ref_z = torch.from_numpy(g[f"{tag}_z"])
    assert tuple(z.shape) == tuple(ref_z.shape) == (audio.shape[0], audio.shape[1] // 16 * 16)
    assert rel_err(z, ref_z) <= TOL
    assert tuple(log_det.shape) == (1,)
    assert rel_err(log_det, torch.from_numpy(g[f"{tag}_log_det"])) <= TOL
    for sigma in (1.0, 0.7):
        loss = owff.waveflow_loss(z, log_det, sigma)
        assert tuple(loss.shape) == (1,)
        assert rel_err(loss, torch.from_numpy(g[f"{tag}_loss_sigma{sigma}"])) <= TOL, sigma


def test_vector_a_covers_trim_and_width():
    """Vector (a) prunes audio that is shorter than its condition and not a multiple of n_group; W = 351 > 2 x 128."""
    z = np.load(GOLD)
    assert z["a_audio"].shape == (2, 22 * 256 - 5) and z["a_z"].shape == (2, 351 * 16)
    assert z["b_audio"].shape == (1, 22 * 256) and z["b_mel"].shape == (1, 80, 22)
    assert os.path.getsize(GOLD) < 1 << 20


def test_oracle_forward_inverse_identity():
    """inverse(forward(audio).z, untrimmed condition) == pruned audio, with the non-zero output_proj of synth_params."""
    from oracle import waveflow as owf
    from oracle import waveflow_forward as owff
    folded = owf.fold_weight_norm(owf.synth_params(4))
    assert float(folded["decoder.3.output_proj.weight"].abs().max()) > 0
    gen = torch.Generator().manual_seed(12)
    mel = torch.randn(1, 80, 9, generator=gen) * 0.5 - 3
    audio = (torch.rand(1, 9 * 256 - 11, generator=gen) * 2 - 1) * 0.5
    with torch.no_grad():
        z, _ = owff.waveflow_forward(folded, audio, mel)
        cond = owf.encoder(folded, mel, 2, trim_conv_artifact=False)
        back = owf.waveflow_inverse(folded, z, cond, 8, 8, 16)
    pruned = audio[:, :audio.shape[1] // 16 * 16]
    assert back.shape == pruned.shape
    assert rel_err(back, pruned) < 1e-4


# ------------------------------------------------------------------------------------------------ ptxas on the new kernel
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
    out = tmp_path_factory.mktemp("ptxas") / "waveflow_layer.o"
    r = subprocess.run([nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-Xptxas", "-v", "-c",
                        os.path.join(ROOT, "parakeet_b200", "csrc", "waveflow_layer.cu"), "-o", str(out)],
                       capture_output=True, text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    return r.stderr


def _kernel(channels):
    return f"waveflow_forward_layer_kernelILi{channels}E"


def _spills(report, kernel):
    lines = report.splitlines()
    start = [i for i, ln in enumerate(lines) if "Compiling entry function" in ln and kernel in ln]
    assert start, f"ptxas reported no entry function {kernel}"
    for ln in lines[start[0] + 1:]:
        assert "Compiling entry function" not in ln, f"no spill line for {kernel}"
        m = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", ln)
        if m:
            return int(m.group(1)), int(m.group(2))


@pytest.mark.parametrize("channels", [64, 128])
def test_forward_layer_wgmma_not_serialized(ptxas_report, channels):
    remarks = [ln for ln in ptxas_report.splitlines() if re.search(r"C75[12]0", ln) and _kernel(channels) in ln]
    assert not remarks, "\n".join(remarks)


def test_forward_layer_64_no_spills_and_no_register_serialization(ptxas_report):
    assert _spills(ptxas_report, _kernel(64)) == (0, 0)
    remarks = [ln for ln in ptxas_report.splitlines() if re.search(r"C751\d", ln) and "serialized" in ln and _kernel(64) in ln]
    assert not remarks, "\n".join(remarks)


def test_forward_layer_128_spill_bound(ptxas_report):
    """The 128-channel instantiation holds the 128 GEMM1 accumulators and 64 z registers at once and spills, exactly as the
    inverse's waveflow_flow_kernel<128> does (DESIGN.md section 7); the measured 384 / 592 bytes are pinned as an upper bound."""
    stores, loads = _spills(ptxas_report, _kernel(128))
    assert stores <= 384 and loads <= 592, (stores, loads)


# ------------------------------------------------------------------------------------------------ C-ABI
def test_forward_structs_match_ctypes(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    mirrors = {"pk_waveflow_forward_layer_args": _lib.WaveflowForwardLayerArgs,
               "pk_waveflow_forward_tail_args": _lib.WaveflowForwardTailArgs}
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "parakeet_b200.h"', "int main(void) {"]
    for cname, cls in mirrors.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    seen = 0
    for line in out.splitlines():
        cname, field, value = line.split()
        cls = mirrors[cname]
        expect = ctypes.sizeof(cls) if field == "size" else getattr(cls, field).offset
        assert int(value) == expect, (cname, field, value, expect)
        seen += 1
    assert seen == sum(len(c._fields_) + 1 for c in mirrors.values())


def test_new_entry_points_are_declared():
    names = _lib.exported_symbols()
    for s in ("pk_waveflow_forward_layer", "pk_waveflow_forward_tail", "pk_waveflow_nll"):
        assert s in names


# ------------------------------------------------------------------------------------------------ host input errors
def _model(channels=64, n_mels=80):
    from parakeet_b200.models import ConditionalWaveFlow
    return ConditionalWaveFlow([16, 16], 8, 8, 16, channels, n_mels, (3, 3), device="cpu")


def test_forward_cpu_tensors_raise_pkerror():
    with pytest.raises(_lib.PkError):
        _model()(torch.zeros(1, 4 * 256), torch.zeros(1, 80, 4))


def test_forward_audio_longer_than_condition_raises_valueerror():
    with pytest.raises(ValueError):
        _model()(torch.zeros(1, 4 * 256 + 1), torch.zeros(1, 80, 4))
    with pytest.raises(ValueError):
        _model().decoder_forward(torch.zeros(1, 100), torch.zeros(1, 80, 99))


@pytest.mark.parametrize("channels,n_mels", [(192, 80), (64, 64), (128, 132)])
def test_forward_outside_the_fused_configs_raises_notimplemented(channels, n_mels):
    with pytest.raises(NotImplementedError):
        _model(channels, n_mels)(torch.zeros(1, 4 * 256), torch.zeros(1, n_mels, 4))


def test_loss_cpu_tensors_raise_pkerror():
    from parakeet_b200.models import WaveFlowLoss
    with pytest.raises(_lib.PkError):
        WaveFlowLoss(1.0)(torch.zeros(1, 16), torch.zeros(1))
