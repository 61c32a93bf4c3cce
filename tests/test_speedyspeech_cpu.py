"""SpeedySpeech without a GPU: the oracle against vectors the reference's own code produced, the state-dict tree, Paddle's
padding="same" rule, what ptxas makes of the residual-block kernel, the C-ABI struct layout and the host errors."""
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
GOLD = os.path.join(ROOT, "tests", "golden", "ref_executed_speedyspeech.npz")
TOL = 2e-6
KERNEL = "ss_residual_block_kernel"


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


def _cfg(tag):
    from oracle import speedyspeech as oss
    return {"small": (oss.SMALL_CFG, 6, 7), "shipped": (oss.SHIPPED_CFG, 7, None)}[tag]


@pytest.mark.parametrize("tag", ["small", "shipped"])
def test_oracle_inference_equals_executed_reference(g, tag):
    from oracle import speedyspeech as oss
    cfg, seed, tone_size = _cfg(tag)
    p = oss.synth_params(seed, cfg, tone_size=tone_size)
    text = torch.from_numpy(g[f"{tag}_inf_text"])
    with torch.no_grad():
        mel = oss.inference(p, cfg, text)
    assert tuple(mel.shape) == g[f"{tag}_inf_mel"].shape and rel_err(mel, torch.from_numpy(g[f"{tag}_inf_mel"])) < TOL


def test_oracle_tones_wrapper_and_batched_forward_equal_executed_reference(g):
    from oracle import speedyspeech as oss
    cfg, seed, tone_size = _cfg("small")
    p = oss.synth_params(seed, cfg, tone_size=tone_size)
    text, tones = torch.from_numpy(g["small_inf_text"]), torch.from_numpy(g["small_inf_tones"])
    mu, sigma = torch.from_numpy(g["small_wr_mu"]), torch.from_numpy(g["small_wr_sigma"])
    with torch.no_grad():
        mel = oss.inference(p, cfg, text, tones)
        logmel = oss.inference_denorm(p, cfg, text, tones, mu, sigma)
        dec, pred = oss.forward(p, cfg, torch.from_numpy(g["small_fwd_text"]), torch.from_numpy(g["small_fwd_tones"]),
                                torch.from_numpy(g["small_fwd_durations"]))
    assert tuple(mel.shape) == g["small_inf_tone_mel"].shape and rel_err(mel, torch.from_numpy(g["small_inf_tone_mel"])) < TOL
    assert rel_err(logmel, torch.from_numpy(g["small_wr_logmel"])) < TOL
    assert (g["small_fwd_text"] == 0).any(), "the batched vector must hold padded tokens"
    assert tuple(dec.shape) == g["small_fwd_decoded"].shape and rel_err(dec, torch.from_numpy(g["small_fwd_decoded"])) < TOL
    assert rel_err(pred, torch.from_numpy(g["small_fwd_pred_durations"])) < TOL
    assert os.path.getsize(GOLD) < 1 << 20


@pytest.mark.parametrize("tag", ["small", "shipped"])
def test_state_dict_keys_and_shapes_equal_reference_tree(g, tag):
    from parakeet_b200.models import SpeedySpeech
    cfg, _, tone_size = _cfg(tag)
    sd = SpeedySpeech(40, tone_size=tone_size, device="cpu", **cfg).state_dict()
    assert sorted(sd) == list(g[f"{tag}_keys"])
    assert [",".join(map(str, sd[k].shape)) for k in g[f"{tag}_keys"]] == list(g[f"{tag}_shapes"])


@pytest.mark.parametrize("d", [1, 3, 27])
def test_paddle_same_rule_known_answers(d):
    from parakeet_b200.models.speedyspeech import paddle_same_conv
    assert paddle_same_conv(1, d) == (1, 0, 0)
    assert paddle_same_conv(3, d) == (1, 1, 1)
    assert paddle_same_conv(4, d) == (1, 1, 2)


# ------------------------------------------------------------------------------------------------ ptxas on the kernel
@_ptxas.needs_nvcc
def test_residual_block_kernel_no_spills_and_no_wgmma_serialization():
    e = _ptxas.entry(_ptxas.report("speedyspeech.cu"), KERNEL)
    assert not e["codes"] & _ptxas.SERIALIZED, e
    assert (e["stack"], e["spill_stores"], e["spill_loads"]) == (0, 0, 0), e


# ------------------------------------------------------------------------------------------------ C-ABI
def test_args_struct_matches_ctypes(tmp_path):
    gcc = shutil.which("gcc")
    if gcc is None:
        pytest.skip("no C compiler")
    cls, cname = _lib.SsResidualBlockArgs, "pk_ss_residual_block_args"
    lines = ['#include <stddef.h>', '#include <stdio.h>', '#include "parakeet_b200.h"', "int main(void) {",
             f'  printf("size %zu\\n", sizeof({cname}));']
    lines += [f'  printf("{f} %zu\\n", offsetof({cname}, {f}));' for f, _ in cls._fields_]
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run([gcc, "-std=c99", "-Wall", "-Werror", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    got = dict(line.split() for line in out if line)
    assert int(got.pop("size")) == ctypes.sizeof(cls)
    assert {k: int(v) for k, v in got.items()} == {f: getattr(cls, f).offset for f, _ in cls._fields_}
    assert "pk_ss_residual_block" in _lib.exported_symbols()


# ------------------------------------------------------------------------------------------------ host errors
def _model(**kw):
    from oracle import speedyspeech as oss
    from parakeet_b200.models import SpeedySpeech
    return SpeedySpeech(40, device="cpu", **dict(oss.SMALL_CFG, **kw))


@pytest.mark.parametrize("field", ["encoder_hidden_size", "duration_predictor_hidden_size", "decoder_hidden_size"])
def test_hidden_size_other_than_128_raises_at_construction(field):
    with pytest.raises(_lib.PkError):
        _model(**{field: 256})


def test_training_mode_forward_raises():
    m = _model()
    m.train()
    with pytest.raises(_lib.PkError):
        m.inference(torch.ones(5, dtype=torch.int64))


def test_cpu_tensors_raise():
    m = _model().eval()
    with pytest.raises(_lib.PkError):
        m.inference(torch.ones(5, dtype=torch.int64))
    with pytest.raises(_lib.PkError):
        m(torch.ones(1, 5, dtype=torch.int64), None, torch.ones(1, 5, dtype=torch.int64))


def test_tones_without_tone_size_raise():
    m = _model().eval()
    with pytest.raises(_lib.PkError):
        m.inference(torch.ones(5, dtype=torch.int64), torch.ones(5, dtype=torch.int64))
