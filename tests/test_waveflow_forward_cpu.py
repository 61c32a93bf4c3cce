"""WaveFlow density direction (ConditionalWaveFlow.forward, WaveFlowLoss) without a GPU: the oracle against vectors the
reference's own code produced, the oracle's forward / inverse identity, what ptxas makes of the new layer kernel, the C-ABI
struct layouts and the input errors of the host class."""
import ctypes
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import _ptxas
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
def _kernel(channels):
    return _ptxas.entry(_ptxas.report("waveflow_layer.cu"), f"waveflow_forward_layer_kernelILi{channels}E")


@_ptxas.needs_nvcc
@pytest.mark.parametrize("channels", [64, 128])
def test_forward_layer_wgmma_not_serialized(channels):
    """Only the 128-channel instantiation serializes its wgmma, for lack of registers (C7512, DESIGN.md section 7)."""
    allowed = {64: set(), 128: {"C7512"}}[channels]
    e = _kernel(channels)
    assert e["codes"] & _ptxas.SERIALIZED <= allowed, e


@_ptxas.needs_nvcc
def test_forward_layer_64_no_spills_and_no_register_serialization():
    e = _kernel(64)
    assert (e["spill_stores"], e["spill_loads"]) == (0, 0), e
    assert e["codes"] <= {"C7519"}, e              # no remark but the injected warpgroup.arrive, which serializes nothing


@_ptxas.needs_nvcc
def test_forward_layer_128_spill_bound():
    """The 128-channel instantiation holds the 128 GEMM1 accumulators and 64 z registers at once and spills, exactly as the
    inverse's waveflow_flow_kernel<128> does (DESIGN.md section 7); the measured 384 / 592 bytes are pinned as an upper bound."""
    e = _kernel(128)
    assert e["spill_stores"] <= 384 and e["spill_loads"] <= 592, e


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
