"""What ptxas makes of every instantiation of the frame-rate Parallel WaveGAN residual layer kernel (pwg_fc.cu: the first layer,
which computes first_conv itself, the middle layers, and the last layer, which runs the tail), without a GPU: no spills, a
0-byte stack frame, no wgmma serialization, and shared memory within the H100's 227 KB opt-in limit per block."""
import re

import pytest

import _ptxas

KERNEL = "pwg_layer_fc_kernel"
MODES = {"first": 0, "middle": 1, "last": 2}             # template argument of the kernel (FcMode)
SMEM_OPTIN_LIMIT = 227 * 1024                             # cudaDevAttrMaxSharedMemoryPerBlockOptin on the H100

pytestmark = _ptxas.needs_nvcc


def _entry(mode):
    return _ptxas.entry(_ptxas.report("pwg_fc.cu"), f"{KERNEL}ILi{MODES[mode]}E")


def test_every_mode_is_instantiated():
    names = [e["name"] for e in _ptxas.report("pwg_fc.cu")["entries"] if KERNEL in e["name"]]
    assert sorted(int(re.search(KERNEL + r"ILi(\d)E", n).group(1)) for n in names) == sorted(MODES.values()), names


@pytest.mark.parametrize("mode", list(MODES))
def test_mode_no_spills_no_stack(mode):
    e = _entry(mode)
    assert (e["stack"], e["spill_stores"], e["spill_loads"]) == (0, 0, 0), e


def test_no_wgmma_serialization_in_any_mode():
    entries = [e for e in _ptxas.report("pwg_fc.cu")["entries"] if KERNEL in e["name"]]
    assert entries and not any(e["codes"] & _ptxas.SERIALIZED for e in entries), entries


@pytest.mark.parametrize("mode", list(MODES))
def test_mode_shared_memory_within_optin_limit(mode):
    """Every mode launches with the same dynamic shared memory (kFcSmem); with its static shared memory it fits one block."""
    static, dynamic = _entry(mode)["smem"], _ptxas.fc_dynamic_smem()
    assert dynamic > 0 and static + dynamic <= SMEM_OPTIN_LIMIT, (static, dynamic)
