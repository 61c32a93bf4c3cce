"""WaveFlow training step without a GPU: the oracle's gradients (autograd through the density direction with weight norm in the
graph) against finite differences and between fp32 and fp64, the zero-output_proj structure of the reference's initialisation,
what ptxas makes of csrc/waveflow_train.cu, the C-ABI declarations, and the step's argument checks."""
import os

import pytest
import torch

import _ptxas

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(n_flows=2, n_layers=2, n_group=8)


def _setup(seed=4, channels=16, frames=3, batch=2, zero_output_proj=False):
    from oracle import waveflow as owf
    p = owf.synth_params(seed, upsample_factors=(4, 4), channels=channels, n_mels=8, **CFG)
    if zero_output_proj:
        p = {k: (torch.zeros_like(v) if "output_proj" in k else v) for k, v in p.items()}
    g = torch.Generator().manual_seed(seed + 100)
    mel = torch.randn(batch, 8, frames, generator=g) * 0.5 - 1
    audio = (torch.rand(batch, frames * 16 - 3, generator=g) * 2 - 1) * 0.5
    return p, audio, mel


def _rel_l2(a, b):
    return float((a.double() - b.double()).norm() / max(float(b.double().norm()), 1e-300))


def test_oracle_gradients_match_finite_differences():
    from oracle import waveflow_train as owt
    p, audio, mel = _setup()
    loss, grads = owt.train_grads(p, audio, mel, **CFG)
    assert set(grads) == set(p)
    g = torch.Generator().manual_seed(1)
    for k in ["encoder.0.weight_v", "encoder.1.weight_g", "decoder.0.input_proj.bias", "decoder.1.resnet.1.conv.weight_v",
              "decoder.0.resnet.0.condition_proj.weight_g", "decoder.1.resnet.0.out_proj.bias", "decoder.0.output_proj.weight"]:
        d = torch.randn(p[k].shape, generator=g, dtype=torch.float64)
        eps = 1e-6
        lp = owt.train_grads({**p, k: p[k].double() + eps * d}, audio, mel, **CFG)[0]
        lm = owt.train_grads({**p, k: p[k].double() - eps * d}, audio, mel, **CFG)[0]
        fd = float(lp - lm) / (2 * eps)
        an = float((grads[k] * d).sum())
        assert abs(fd - an) <= 1e-6 * max(1.0, abs(an)), (k, fd, an)


def test_oracle_fp32_vs_fp64_gap():
    """Recorded gap of the fp32 oracle to the fp64 one (the arbiter of the GPU tolerances): every tensor within 1e-4 relative L2
    at this size (measured: < 1e-5 on most tensors)."""
    from oracle import waveflow_train as owt
    p, audio, mel = _setup(channels=32, frames=4)
    l64, g64 = owt.train_grads(p, audio, mel, **CFG)
    l32, g32 = owt.train_grads(p, audio, mel, dtype=torch.float32, **CFG)
    assert abs(float(l32) - float(l64)) <= 1e-5 * abs(float(l64))
    # input_proj.weight_v: weight norm over ONE input element makes w = g * sign(v), so its gradient is zero up to rounding
    zero = {k for k in g64 if float(g64[k].norm()) < 1e-12}
    assert zero == {k for k in g64 if k.endswith("input_proj.weight_v")}
    assert all(float(g32[k].norm()) < 1e-6 for k in zero)
    gaps = {k: _rel_l2(g32[k], g64[k]) for k in g64 if k not in zero}
    worst = max(gaps, key=gaps.get)
    print(f"oracle fp32 vs fp64: worst {worst} {gaps[worst]:.2e}, median {sorted(gaps.values())[len(gaps) // 2]:.2e}")
    assert gaps[worst] < 1e-4, (worst, gaps[worst])


def test_oracle_zero_output_proj_gradients():
    """The reference zero-initialises output_proj: the flows start as the identity, so only output_proj receives a gradient."""
    from oracle import waveflow_train as owt
    p, audio, mel = _setup(zero_output_proj=True)
    _, grads = owt.train_grads(p, audio, mel, **CFG)
    for k, g in grads.items():
        if "output_proj" in k:
            assert float(g.abs().max()) > 0, k
        else:
            assert float(g.abs().max()) == 0.0, k


# ------------------------------------------------------------------------------------------------ ptxas on the new kernels
def _backward_layer(channels):
    return _ptxas.entry(_ptxas.report("waveflow_train.cu"), f"waveflow_backward_layer_kernelILi{channels}E")


@_ptxas.needs_nvcc
def test_waveflow_train_glue_kernels_do_not_spill():
    glue = [e for e in _ptxas.report("waveflow_train.cu")["entries"] if "backward_layer" not in e["name"]]
    assert len(glue) >= 12
    assert all((e["spill_stores"], e["spill_loads"]) == (0, 0) for e in glue), glue


@_ptxas.needs_nvcc
@pytest.mark.parametrize("channels", [64, 128])
def test_backward_layer_wgmma_not_serialized(channels):
    """No C75xx remark at all: neither serialization (_ptxas.SERIALIZED) nor an injected warpgroup.arrive (C7519)."""
    e = _backward_layer(channels)
    assert not e["codes"], e


# upper bounds: 0 bytes for both instantiations when this test was written (168 registers each, no stack frame)
SPILL_BOUND = {64: (0, 0), 128: (0, 0)}


@_ptxas.needs_nvcc
@pytest.mark.parametrize("channels", [64, 128])
def test_backward_layer_spill_bound(channels):
    e = _backward_layer(channels)
    assert e["spill_stores"] <= SPILL_BOUND[channels][0] and e["spill_loads"] <= SPILL_BOUND[channels][1], e


# ------------------------------------------------------------------------------------------------ C-ABI and host checks
NEW = ["pk_waveflow_backward_layer", "pk_waveflow_train_gather_split", "pk_waveflow_train_input_fwd", "pk_waveflow_train_update",
       "pk_waveflow_train_tail_fwd", "pk_waveflow_forward_tail_bwd", "pk_waveflow_train_input_bwd", "pk_waveflow_train_outer_sum",
       "pk_waveflow_upsample_bwd", "pk_waveflow_train_cond_gather", "pk_waveflow_train_cond_scatter", "pk_waveflow_train_loss"]


def test_new_entry_points_declared_exported_and_bound_from_header():
    """Each entry point is declared, exported, and bound with the argtypes derived from its header prototype."""
    from parakeet_b200 import _lib
    declared = set(_lib.exported_symbols())
    assert set(NEW) <= declared
    for name in NEW:
        assert _lib.PROTOTYPES[name].argtypes, name
    if os.path.exists(_lib.LIB_PATH):
        L = _lib.lib()
        for name in NEW:
            assert hasattr(L, name), name
            assert list(getattr(L, name).argtypes) == _lib.PROTOTYPES[name].argtypes, name


def _model(channels=64, n_mels=80, n_layers=2, device="cpu"):
    from parakeet_b200.models import ConditionalWaveFlow
    return ConditionalWaveFlow([16, 16], 2, n_layers, 16, channels, n_mels, (3, 3), device=device)


def test_cpu_model_raises_pkerror():
    from parakeet_b200._lib import PkError
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    with pytest.raises(PkError):
        WaveFlowTrainStep(_model())


@pytest.mark.parametrize("kw", [dict(channels=192), dict(n_mels=64), dict(n_mels=136), dict(n_layers=1), dict(n_layers=9)])
def test_ineligible_configs_raise_not_implemented(kw):
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    with pytest.raises(NotImplementedError):
        WaveFlowTrainStep(_model(**kw))


# ------------------------------------------------------------------------------------------------ pinned to the reference's code
GOLD = os.path.join(ROOT, "tests", "golden", "ref_executed_waveflow_train.npz")


def golden_setup():
    """The vector scripts/make_golden_ref.py waveflow_train recorded from the reference's own ConditionalWaveFlow + WaveFlowLoss."""
    import numpy as np
    from oracle import waveflow as owf
    g = np.load(GOLD)
    p = owf.synth_params(6, n_flows=2, n_layers=8, channels=64)
    return g, p, torch.from_numpy(g["audio"]), torch.from_numpy(g["mel"]), dict(n_flows=2, n_layers=8, n_group=16)


def _sampled(t):
    t = t.reshape(-1)
    return t[::max(1, t.numel() // 4096)]


def test_oracle_gradients_equal_executed_reference():
    from oracle import waveflow_train as owt
    g, p, audio, mel, cfg = golden_setup()
    loss, grads = owt.train_grads(p, audio, mel, dtype=torch.float32, **cfg)
    assert abs(float(loss) - float(g["loss"][0])) <= 1e-6 * abs(float(g["loss"][0]))
    assert {k[len("grad/"):] for k in g.files if k.startswith("grad/")} == set(p)
    for k in p:
        ref = torch.from_numpy(g["grad/" + k])
        if k.endswith("input_proj.weight_v"):           # zero up to rounding in both (w = g * sign(v))
            assert float(ref.norm()) < 1e-6 and float(grads[k].norm()) < 1e-6, k
            continue
        assert _rel_l2(_sampled(grads[k]), ref) <= 1e-5, k
        assert abs(float(grads[k].double().norm()) - float(g["gradnorm/" + k])) <= 1e-5 * float(g["gradnorm/" + k]), k
