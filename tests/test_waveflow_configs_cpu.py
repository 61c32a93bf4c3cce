"""ConditionalWaveFlow's config range without a GPU: the configs the constructor refuses, which layer path each accepted config
takes, pk_waveflow_flow's refusal of one-layer flows, the oracle against the reference's own code at a config away from the
shipped one (tests/golden/ref_executed_waveflow_configs.npz, scripts/make_golden_ref.py waveflow_configs), and the oracle's
forward / inverse identity at the configs tests/test_gpu_waveflow_configs.py runs."""
import ctypes
import os

import numpy as np
import pytest
import torch

from conftest import rel_err
from parakeet_b200 import _lib

GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_executed_waveflow_configs.npz")
GOLD_CFG = dict(upsample_factors=(8, 32), n_flows=4, n_layers=8, n_group=8, channels=128, n_mels=128)
GOLD_SEED = 7
TOL = 2e-6        # the oracle's forward against the executed reference (as tests/test_waveflow_forward_cpu.py)


def _model(channels=64, n_mels=80, n_layers=3, n_flows=2, n_group=16):
    from parakeet_b200.models import ConditionalWaveFlow
    return ConditionalWaveFlow([16, 16], n_flows, n_layers, n_group, channels, n_mels, (3, 3), device="cpu", seed=9)


@pytest.mark.parametrize("channels,n_mels", [(192, 80), (256, 80), (64, 81), (128, 100)])
def test_constructor_refuses_configs_no_path_runs(channels, n_mels):
    """192 / 256 channels would need the two-GEMM path's fused epilogues past N = 256; n_mels 81 / 100 a condition row stride
    that is not a multiple of 16 bytes.  Both are refused when the model is built, not deep inside infer()."""
    with pytest.raises(NotImplementedError):
        _model(channels, n_mels)


def test_from_pretrained_refuses_configs_no_path_runs(tmp_path):
    from parakeet_b200.models import ConditionalWaveFlow
    cfg = {"model": {"upsample_factors": [16, 16], "n_flows": 2, "n_layers": 2, "n_group": 16, "channels": 64, "kernel_size": [3, 3]},
           "data": {"n_mels": 100}}
    with pytest.raises(NotImplementedError):
        ConditionalWaveFlow.from_pretrained(cfg, str(tmp_path / "missing"), device="cpu")


@pytest.mark.parametrize("channels", [64, 128])
@pytest.mark.parametrize("n_mels", [64, 72, 128, 136])
def test_constructor_accepts_and_routes(channels, n_mels):
    """64 and 128 channels are accepted at every n_mels that is a multiple of 8; the fused kernels take 64 < n_mels <= 128, the
    two-GEMM row loop the rest."""
    assert _model(channels, n_mels)._eligible() == (64 < n_mels <= 128)


def test_eligible_needs_two_to_eight_layers():
    """A one-layer flow would race on pk_waveflow_flow's ring (the next row's input_proj lands in layer 0's ring during the
    layer-step whose neighbouring tiles still read that slot); more than 8 layers need width dilations past 128."""
    for n_layers in range(1, 10):
        assert _model(n_layers=n_layers)._eligible() == (2 <= n_layers <= 8), n_layers


def test_one_layer_forward_raises_notimplemented():
    with pytest.raises(NotImplementedError):
        _model(n_layers=1)(torch.zeros(1, 4 * 256), torch.zeros(1, 80, 4))


def test_flow_kernel_refuses_one_layer():
    """The argument check runs before any launch: a complete argument struct with n_layers = 1 returns -1 and says why."""
    L = _lib.lib()
    B, W, C, M, G = 1, 8, 64, 80, 16
    a = _lib.WaveflowFlowArgs()
    a.batch, a.width, a.channels, a.n_mels, a.n_group = B, W, C, M, G
    keep = []

    def buf(nbytes):
        b = ctypes.create_string_buffer(nbytes)
        keep.append(b)
        return ctypes.cast(b, ctypes.c_void_p)
    for name in ("cond_rows", "ring_hi", "ring_lo", "cond_hi", "cond_lo", "w1_hi", "w1_lo", "w2_hi", "w2_lo", "bias1", "bias2",
                 "in_w", "in_b", "out_w", "out_b", "z", "x", "skip", "flags"):
        setattr(a, name, buf(4096))
    a.flags_len = 1 << 20
    for n_layers, reason in ((1, b"ring"), (0, b"ring"), (9, b"2..8")):
        a.n_layers = n_layers
        assert L.pk_waveflow_flow(ctypes.byref(a), None) == -1, n_layers
        msg = L.pk_last_error()
        assert b"n_layers" in msg and reason in msg, msg


# ------------------------------------------------------------------------------------------------ oracle vs executed reference
@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


def _gold_params():
    from oracle import waveflow as owf
    return owf.fold_weight_norm(owf.synth_params(GOLD_SEED, **GOLD_CFG))


def test_golden_vector_covers_the_config(g):
    """W = 284 for the inverse and 319 for the forward (both > 2 x 128: the widest taps read live columns); the audio is not a
    multiple of n_group.  The mel has 128 bands."""
    assert g["mel"].shape == (2, 128, 10) and g["z"].shape == (2, (10 * 8 - 8) * 32 - 32)
    assert g["z"].shape[1] // 8 == 284 and g["x"].shape == g["z"].shape
    assert g["audio"].shape == (2, 10 * 256 - 5) and g["fwd_z"].shape == (2, (10 * 256 - 5) // 8 * 8)
    assert os.path.getsize(GOLD) < 1 << 20


def test_oracle_equals_executed_reference_at_a_non_default_config(g):
    from oracle import waveflow as owf
    from oracle import waveflow_forward as owff
    folded = _gold_params()
    c = GOLD_CFG
    mel, z, audio = (torch.from_numpy(g[k]) for k in ("mel", "z", "audio"))
    with torch.no_grad():
        x = owf.infer(folded, mel, z, n_up=2, n_flows=c["n_flows"], n_layers=c["n_layers"], n_group=c["n_group"])
        fz, log_det = owff.waveflow_forward(folded, audio, mel, n_up=2, n_flows=c["n_flows"], n_layers=c["n_layers"], n_group=c["n_group"])
    assert tuple(x.shape) == g["x"].shape and rel_err(x, torch.from_numpy(g["x"])) < 1e-5
    assert tuple(fz.shape) == g["fwd_z"].shape and rel_err(fz, torch.from_numpy(g["fwd_z"])) <= TOL
    assert rel_err(log_det, torch.from_numpy(g["fwd_log_det"])) <= TOL
    for sigma in (1.0, 0.7):
        assert rel_err(owff.waveflow_loss(fz, log_det, sigma), torch.from_numpy(g[f"loss_sigma{sigma}"])) <= TOL, sigma


# ------------------------------------------------------------------------------------------------ oracle forward / inverse
@pytest.mark.parametrize("ups,n_flows,n_layers,n_group,channels,n_mels", [
    ((16, 16), 4, 1, 16, 64, 72),
    ((16, 16), 4, 5, 8, 128, 128),
    ((8, 32), 16, 2, 16, 64, 96),
    ((16, 16), 4, 3, 8, 128, 136),
])
def test_oracle_forward_inverse_identity_at_other_configs(ups, n_flows, n_layers, n_group, channels, n_mels):
    """inverse(forward(audio).z, untrimmed condition) == pruned audio (as test_oracle_forward_inverse_identity) at the layer
    counts, flow counts, n_group, upsample factors and mel bands the GPU config tests use.  n_flows is a multiple of 4: the
    reference's WaveFlow.inverse permutes the condition starting from the unpermuted one, so it inverts forward only when the
    flows' permutations compose to the identity (with 2 flows they compose to a swap of the two halves)."""
    from oracle import waveflow as owf
    from oracle import waveflow_forward as owff
    folded = owf.fold_weight_norm(owf.synth_params(12, upsample_factors=ups, n_flows=n_flows, n_layers=n_layers, n_group=n_group,
                                                   channels=channels, n_mels=n_mels))
    gen = torch.Generator().manual_seed(13)
    mel = torch.randn(1, n_mels, 5, generator=gen) * 0.5 - 3
    audio = (torch.rand(1, 5 * 256 - 11, generator=gen) * 2 - 1) * 0.5
    with torch.no_grad():
        z, _ = owff.waveflow_forward(folded, audio, mel, n_up=2, n_flows=n_flows, n_layers=n_layers, n_group=n_group)
        cond = owf.encoder(folded, mel, 2, trim_conv_artifact=False)
        back = owf.waveflow_inverse(folded, z, cond, n_flows, n_layers, n_group)
    pruned = audio[:, :audio.shape[1] // n_group * n_group]
    assert back.shape == pruned.shape
    assert rel_err(back, pruned) < 1e-4
