"""ConditionalWaveFlow on the GPU across the config range the model accepts, against the fp64 oracles: the fused inverse
(pk_waveflow_flow) at every condition K-step count, n_group 8, other layer and flow counts, other upsample factors and more
tiles per layer-step than resident CTAs; the two-GEMM row loop that one-layer and out-of-range configs take; the density
direction, a round trip and the training step off the default config; and the CUDA model against the reference's own code at
a non-default config (tests/golden/ref_executed_waveflow_configs.npz).

Unless a case says otherwise: B = 3, 28 mel frames, upsample 16 x 16 -> 6 896 samples, W = 431 columns at n_group 16 (every
width dilation up to 128 reaches live columns on both sides, the last 256-column tile is partial)."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3          # audio and z: max-abs error / max-abs reference
LOGDET_TOL = 1e-3   # relative
LOSS_TOL = 1e-4     # relative
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_executed_waveflow_configs.npz")


def _model(cuda, seed, ups=(16, 16), n_flows=2, n_layers=8, n_group=16, channels=64, n_mels=80):
    """-> (CUDA model, fp64 weight-norm-folded oracle parameters, oracle config)."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    p = owf.synth_params(seed, upsample_factors=ups, n_flows=n_flows, n_layers=n_layers, n_group=n_group, channels=channels, n_mels=n_mels)
    m = ConditionalWaveFlow(list(ups), n_flows, n_layers, n_group, channels, n_mels, (3, 3), device=cuda)
    m.set_state_dict(p)
    folded = owf.fold_weight_norm({k: v.double() for k, v in p.items()})
    return m, folded, dict(n_up=len(ups), n_flows=n_flows, n_layers=n_layers, n_group=n_group)


def _noise(seed, batch, n_mels, frames, ups=(16, 16)):
    """mel (B, n_mels, frames) and the noise z (B, T_c) of infer: each transposed conv of the upsampler trims f samples."""
    g = torch.Generator().manual_seed(seed)
    t_c = frames
    for f in ups:
        t_c = t_c * f - f
    return torch.randn(batch, n_mels, frames, generator=g) * 0.5 - 3, torch.randn(batch, t_c, generator=g)


def _oracle_infer(folded, cfg, mel, z):
    from oracle import waveflow as owf
    with torch.no_grad():
        return owf.infer(folded, mel.double(), z.double(), **cfg)


def _check_infer(cuda, m, folded, cfg, mel, z):
    ref = _oracle_infer(folded, cfg, mel, z)
    out = m.infer(mel.to(cuda), z=z.to(cuda))
    assert tuple(out.shape) == tuple(ref.shape)
    err = rel_err(out, ref)
    assert err < TOL, err


# ------------------------------------------------------------------------------------------------ 1-5: the fused inverse
@pytest.mark.parametrize("channels", [64, 128])
@pytest.mark.parametrize("n_mels", [72, 96, 128])
def test_inverse_condition_ksteps(cuda, channels, n_mels):
    """The last condition K-chunk holds n_mels - 64 bands: cond_ksteps_last = 1, 2, 4 K-steps of 16 at n_mels 72 / 96 / 128,
    and at 72 the TMA box reads zero fill past the last band."""
    m, folded, cfg = _model(cuda, 60 + n_mels // 8 + channels, channels=channels, n_mels=n_mels)
    assert m._eligible()
    mel, z = _noise(61 + n_mels, 3, n_mels, 28)
    _check_infer(cuda, m, folded, cfg, mel, z)


@pytest.mark.parametrize("channels", [64, 128])
def test_inverse_n_group_8(cuda, channels):
    """n_group 8: 7 row steps per flow, the completion counters sized for them, the condition rows addressed through the
    8-row permutations of 8 flows; W = 862."""
    m, folded, cfg = _model(cuda, 70 + channels, n_flows=8, n_layers=4, n_group=8, channels=channels)
    assert m._eligible()
    mel, z = _noise(71, 3, 80, 28)
    assert z.shape[1] // 8 == 862
    _check_infer(cuda, m, folded, cfg, mel, z)


@pytest.mark.parametrize("n_layers", [2, 3, 5])
def test_inverse_layer_counts(cuda, n_layers):
    """The dataflow's layer-steps are (row, layer) pairs: the write of the next row's input_proj into layer 0's ring comes
    n_layers - 1 = 1, 2, 4 layer-steps after layer 0's last read of that slot."""
    m, folded, cfg = _model(cuda, 80 + n_layers, n_layers=n_layers)
    assert m._eligible()
    mel, z = _noise(81 + n_layers, 3, 80, 28)
    _check_infer(cuda, m, folded, cfg, mel, z)


@pytest.mark.parametrize("n_flows,channels", [(4, 128), (16, 64)])
def test_inverse_flow_counts(cuda, n_flows, channels):
    """The permutations switch from reversal to half reversal at n_flows // 2, so the composed condition-row map of every
    flow differs from the 8-flow one."""
    m, folded, cfg = _model(cuda, 90 + n_flows, n_flows=n_flows, n_layers=3, channels=channels)
    assert m._eligible()
    mel, z = _noise(91 + n_flows, 3, 80, 28)
    _check_infer(cuda, m, folded, cfg, mel, z)


def test_inverse_upsample_8_32(cuda):
    """pk_waveflow_upsample at factors 8 and 32 (W = 430): the upsampled condition alone, then the whole inverse."""
    from oracle import waveflow as owf
    ups = (8, 32)
    m, folded, cfg = _model(cuda, 95, ups=ups, n_layers=8)
    assert m._eligible()
    mel, z = _noise(96, 3, 80, 28, ups=ups)
    with torch.no_grad():
        cond = owf.encoder(folded, mel.double(), 2)
    assert rel_err(m.encode(mel.to(cuda)), cond) < 1e-5
    _check_infer(cuda, m, folded, cfg, mel, z)


# ------------------------------------------------------------------------------------------------ 6-7: many tiles, both paths
def _many_tiles(cuda, m, folded, cfg, seed):
    """B = 16, 145 frames: W = 2303, 9 tiles of 256 per utterance, 144 per layer-step (more than the H100's 132 CTAs at one per
    SM).  Utterances 0 and 15 against the oracle run on each alone; utterance 5 alone is bit-identical to its row of the
    batch; the eager call, the captured call and a replay are bit-identical."""
    mel, z = _noise(seed, 16, m.n_mels, 145)
    assert z.shape[1] // 16 == 2303
    mel_c, z_c = mel.to(cuda), z.to(cuda)
    replays = m._graphs.replays
    y0 = m.infer(mel_c, z=z_c).clone()                                # eager
    y1 = m.infer(mel_c, z=z_c).clone()                                # capture
    y2 = m.infer(mel_c, z=z_c).clone()                                # replay
    assert m._graphs.replays >= replays + 2
    assert torch.isfinite(y0).all() and torch.equal(y0, y1) and torch.equal(y0, y2)
    one = m.infer(mel_c[5:6].contiguous(), z=z_c[5:6].contiguous())
    assert torch.equal(one[0], y0[5])
    for b in (0, 15):
        ref = _oracle_infer(folded, cfg, mel[b:b + 1], z[b:b + 1])
        err = rel_err(y0[b:b + 1], ref)
        assert err < TOL, (b, err)


@pytest.mark.parametrize("n_layers", [2, 8])
def test_inverse_more_tiles_than_resident_ctas(cuda, n_layers):
    m, folded, cfg = _model(cuda, 100 + n_layers, n_layers=n_layers, channels=128)
    assert m._eligible()
    _many_tiles(cuda, m, folded, cfg, 101 + n_layers)


@pytest.mark.parametrize("channels", [64, 128])
def test_two_gemm_path_one_layer(cuda, channels):
    """A one-layer flow is not eligible for pk_waveflow_flow and runs the two-GEMM row loop."""
    m, folded, cfg = _model(cuda, 110 + channels, n_layers=1, channels=channels)
    assert not m._eligible()
    mel, z = _noise(111, 3, 80, 28)
    _check_infer(cuda, m, folded, cfg, mel, z)


def test_two_gemm_path_one_layer_many_tiles(cuda):
    m, folded, cfg = _model(cuda, 115, n_layers=1, channels=128)
    assert not m._eligible()
    _many_tiles(cuda, m, folded, cfg, 116)


@pytest.mark.parametrize("channels", [64, 128])
def test_two_gemm_path_136_mels(cuda, channels):
    """n_mels 136 is past the fused kernels' 128: the condition GEMM of the row loop runs with K = 136."""
    m, folded, cfg = _model(cuda, 120 + channels, n_layers=3, channels=channels, n_mels=136)
    assert not m._eligible()
    mel, z = _noise(121, 3, 136, 28)
    _check_infer(cuda, m, folded, cfg, mel, z)


# ------------------------------------------------------------------------------------------------ 8-9: the density direction
def _audio(seed, batch, n_mels, frames, samples):
    g = torch.Generator().manual_seed(seed)
    mel = torch.randn(batch, n_mels, frames, generator=g) * 0.5 - 3
    return (torch.rand(batch, samples, generator=g) * 2 - 1) * 0.5, mel


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


@pytest.mark.parametrize("channels,n_mels,n_layers,n_group", [(64, 72, 2, 16), (64, 128, 5, 16), (128, 72, 5, 8), (128, 128, 2, 8)])
def test_forward_and_loss(cuda, channels, n_mels, n_layers, n_group):
    """pk_waveflow_forward_layer / _tail at 4 flows, 2 or 5 layers, n_mels 72 (1 condition K-step, zero fill) and 128 (4),
    n_group 16 and 8; audio of 28 * 256 - 7 samples (W = 447 at n_group 16, 895 at 8)."""
    from oracle import waveflow_forward as owff
    from parakeet_b200.models import WaveFlowLoss
    m, folded, cfg = _model(cuda, 130 + n_layers + n_mels, n_flows=4, n_layers=n_layers, n_group=n_group, channels=channels, n_mels=n_mels)
    assert m._eligible()
    audio, mel = _audio(131 + n_mels, 3, n_mels, 28, 28 * 256 - 7)
    with torch.no_grad():
        ref_z, ref_ld = owff.waveflow_forward(folded, audio.double(), mel.double(), **cfg)
    z, log_det = m(audio.to(cuda), mel.to(cuda))
    assert tuple(z.shape) == tuple(ref_z.shape)
    err = rel_err(z, ref_z)
    assert err < TOL, err
    assert _rel(log_det, ref_ld) < LOGDET_TOL
    for sigma in (1.0, 0.7):
        assert _rel(WaveFlowLoss(sigma)(z, log_det), owff.waveflow_loss(ref_z, ref_ld, sigma)) < LOSS_TOL, sigma


def test_round_trip_n_group_8_128_mels(cuda):
    """inverse(forward(audio).z, untrimmed condition) returns the audio at n_group 8, 128 mel bands and 128 channels (8 flows:
    the reference's inverse undoes its forward when the flows' permutations compose to the identity)."""
    m, _, _ = _model(cuda, 140, n_flows=8, n_layers=8, n_group=8, channels=128, n_mels=128)
    assert m._eligible()
    audio, mel = _audio(141, 3, 128, 28, 28 * 256)
    audio, mel = audio.to(cuda), mel.to(cuda)
    z, _ = m(audio, mel)
    back = m.inverse(z, m.encode(mel, trim_conv_artifact=False))
    assert back.shape == audio.shape
    err = rel_err(back, audio)
    assert err < TOL, err


# ------------------------------------------------------------------------------------------------ 10: the training step
@pytest.mark.parametrize("channels,n_mels,n_group", [(64, 72, 16), (64, 72, 8), (64, 128, 16), (64, 128, 8), (128, 96, 16)])
def test_training_step_condition_bands(cuda, channels, n_mels, n_group):
    """Loss and every gradient at n_mels != 80: the forward condition GEMM (K = n_mels), the condition-gradient GEMM
    (N = n_mels) and pk_waveflow_train_cond_gather / _scatter; 2 flows x 2 layers."""
    from oracle import waveflow as owf
    from oracle import waveflow_train as owt
    from parakeet_b200.models import ConditionalWaveFlow
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    from test_gpu_waveflow_training import _check_grads
    seed = 150 + n_mels + n_group + channels
    p = owf.synth_params(seed, n_flows=2, n_layers=2, n_group=n_group, channels=channels, n_mels=n_mels)
    m = ConditionalWaveFlow([16, 16], 2, 2, n_group, channels, n_mels, (3, 3), device=cuda)
    m.set_state_dict(p)
    assert m._eligible()
    audio, mel = _audio(seed + 1, 3, n_mels, 28, 28 * 256 - 7)
    step = WaveFlowTrainStep(m)
    loss = step.forward_backward_graphed(audio.to(cuda), mel.to(cuda))
    ref_loss, ref = owt.train_grads(p, audio, mel, n_flows=2, n_layers=2, n_group=n_group)
    _check_grads(step, p, ref, loss, ref_loss)


# ------------------------------------------------------------------------------------------------ against the executed reference
def test_cuda_vs_executed_reference_at_a_non_default_config(cuda):
    """The reference's own ConditionalWaveFlow at n_group 8, 128 mel bands, 4 flows x 8 layers, upsample 8 x 32 and 128
    channels: the inverse from a given z, forward z / log-det and WaveFlowLoss."""
    from test_waveflow_configs_cpu import GOLD_CFG, GOLD_SEED
    from parakeet_b200.models import WaveFlowLoss
    g = np.load(GOLD)
    m, _, _ = _model(cuda, GOLD_SEED, ups=GOLD_CFG["upsample_factors"], **{k: v for k, v in GOLD_CFG.items() if k != "upsample_factors"})
    assert m._eligible()
    mel, z, audio = (torch.from_numpy(g[k]).to(cuda) for k in ("mel", "z", "audio"))
    x = m.infer(mel, z=z)
    assert tuple(x.shape) == g["x"].shape
    err = rel_err(x, torch.from_numpy(g["x"]))
    assert err < TOL, err
    fz, log_det = m(audio, mel)
    assert tuple(fz.shape) == g["fwd_z"].shape
    err = rel_err(fz, torch.from_numpy(g["fwd_z"]))
    assert err < TOL, err
    assert _rel(log_det, g["fwd_log_det"][0]) < LOGDET_TOL
    for sigma in (1.0, 0.7):
        assert _rel(WaveFlowLoss(sigma)(fz, log_det), g[f"loss_sigma{sigma}"][0]) < LOSS_TOL, sigma
