"""The CUDA sources keep one owner for launch setup and for the helpers every kernel file uses, checked on the source text: the
dynamic shared-memory limit and occupancy are handled only by pk::prepare_kernel (pk_common.cu), which remembers them per device,
and each shared device / host helper has exactly one definition."""
import glob
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "parakeet_b200", "csrc")


def _sources():
    paths = sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) +
                   glob.glob(os.path.join(CSRC, "*.h")))
    assert paths, CSRC
    out = {}
    for p in paths:
        with open(p) as f:
            out[os.path.basename(p)] = f.read()
    return out


SOURCES = _sources()


@pytest.mark.parametrize("call", ["cudaFuncSetAttribute", "cudaOccupancyMaxActiveBlocksPerMultiprocessor"])
def test_launch_setup_only_in_pk_common(call):
    users = sorted(name for name, text in SOURCES.items() if re.search(rf"\b{call}\b", text))
    assert users == ["pk_common.cu"], users


@pytest.mark.parametrize("pattern", [r"\battr_set\b", r"\bonce_flag\b", r"\bcall_once\b", r"\bmax_resident\b", r"\bsized_for\b"])
def test_no_process_wide_launch_caches(pattern):
    users = sorted(name for name, text in SOURCES.items() if re.search(pattern, text))
    assert not users, users


@pytest.mark.parametrize("name, home", [
    ("split2", "pk_sm90.cuh"),
    ("ex2_approx", "pk_sm90.cuh"),
    ("rcp_approx", "pk_sm90.cuh"),
    ("warp_sum", "pk_sm90.cuh"),
    ("sigmoidf_", "pk_sm90.cuh"),
    ("ld_acquire_gpu", "pk_sm90.cuh"),
    ("red_release_gpu_inc", "pk_sm90.cuh"),
    ("warp_max", "pk_sm90.cuh"),
    ("ld_split", "pk_sm90.cuh"),
    ("block_sum_tree", "pk_sm90.cuh"),
    ("aligned16", "pk_host.h"),
    ("fold_gate_bias", "pk_host.h"),
    ("nblk", "pk_host.h"),
    ("grid_stride_blocks", "pk_host.h"),
])
def test_helper_defined_once(name, home):
    # a definition: return type, the name, its parameter list and an opening brace (calls end in ';' or sit inside expressions)
    definition = re.compile(rf"^[ \t]*(?:static |inline |__device__ |__forceinline__ )*[\w:]+[ \t]+{name}\([^;{{]*\)[ \t]*\{{",
                            re.MULTILINE)
    where = [(fname, len(definition.findall(text))) for fname, text in SOURCES.items() if definition.search(text)]
    assert where == [(home, 1)], where


def test_log2e_constant_defined_once():
    where = sorted(name for name, text in SOURCES.items() if re.search(r"constexpr float kLog2e\b", text))
    assert where == ["pk_host.h"], where


def test_launch_macros_defined_once():
    # the stream cast, the launch tail and the grid-stride loop live in pk_host.h / pk_sm90.cuh under one name each
    stream_cast = re.compile(r"^[ \t]*#[ \t]*define[ \t]+\w+[^\n]*static_cast<cudaStream_t>", re.MULTILINE)
    launch_tail = re.compile(r"^[ \t]*#[ \t]*define[ \t]+\w+(?:\([^)]*\))?[ \t]*\\?\s*PK_CHECK_CUDA\(cudaGetLastError\(\)\)", re.MULTILINE)
    grid_stride = re.compile(r"^[ \t]*#[ \t]*define[ \t]+\w+\([^)]*\)[ \t]*\\?\s*for \(long long", re.MULTILINE)
    for pattern, home in ((stream_cast, "pk_host.h"), (launch_tail, "pk_host.h"), (grid_stride, "pk_sm90.cuh")):
        where = [(name, len(pattern.findall(text))) for name, text in SOURCES.items() if pattern.search(text)]
        assert where == [(home, 1)], (pattern.pattern, where)


def test_merged_entry_points_are_gone():
    # the causal mask, the guided attention loss and the gradient clip are arguments of these three, not entry points of their own
    with open(os.path.join(ROOT, "include", "parakeet_b200.h")) as f:
        header = f.read()
    for name, variant in (("pk_masked_softmax", "_ex"), ("pk_softmax_bwd", "_guided"), ("pk_adam", "_clip")):
        assert re.search(rf"\b{name}\(", header), name
        gone = name + variant
        assert not re.search(rf"\b{gone}\b", header), gone
        assert not [f for f, text in SOURCES.items() if re.search(rf"\b{gone}\b", text)], gone
