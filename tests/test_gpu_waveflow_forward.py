"""ConditionalWaveFlow.forward (audio -> z, log-det: pk_waveflow_forward_layer + pk_waveflow_forward_tail) and WaveFlowLoss on
the GPU, against the vectors the reference's own code produced, against the oracle, and against the already-pinned inverse."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_executed_waveflow_forward.npz")


def _model(cuda, channels, seed, n_group=16, zero_output_proj=False):
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(seed, channels=channels, n_group=n_group)
    if zero_output_proj:                                   # the reference's initialisation (Constant(0.))
        params = {k: (torch.zeros_like(v) if "output_proj" in k else v) for k, v in params.items()}
    m = ConditionalWaveFlow([16, 16], 8, 8, n_group, channels, 80, (3, 3), device=cuda)
    m.set_state_dict(params)
    return m, owf.fold_weight_norm(params)


def _inputs(seed, batch, frames, samples):
    g = torch.Generator().manual_seed(seed)
    mel = torch.randn(batch, 80, frames, generator=g) * 0.5 - 3
    audio = (torch.rand(batch, samples, generator=g) * 2 - 1) * 0.5
    return audio, mel


def _rel(a, b):
    return abs(float(a) - float(b)) / max(abs(float(b)), 1e-30)


@pytest.mark.parametrize("tag,channels,seed", [("a", 64, 4), ("b", 128, 5)])
def test_forward_and_loss_vs_executed_reference(cuda, tag, channels, seed):
    from parakeet_b200.models import WaveFlowLoss
    g = np.load(GOLD)
    m, _ = _model(cuda, channels, seed)
    audio, mel = torch.from_numpy(g[f"{tag}_audio"]).to(cuda), torch.from_numpy(g[f"{tag}_mel"]).to(cuda)
    z, log_det = m(audio, mel)
    ref_z = torch.from_numpy(g[f"{tag}_z"])
    assert tuple(z.shape) == tuple(ref_z.shape) and tuple(log_det.shape) == (1,)
    assert rel_err(z, ref_z) < TOL
    assert _rel(log_det, g[f"{tag}_log_det"][0]) < 1e-3
    for sigma in (1.0, 0.7):
        loss = WaveFlowLoss(sigma)(z, log_det)
        assert tuple(loss.shape) == (1,)
        assert _rel(loss, g[f"{tag}_loss_sigma{sigma}"][0]) < 1e-4, sigma


@pytest.mark.parametrize("channels,seed", [(64, 4), (128, 5)])
def test_forward_vs_oracle_wide_rows(cuda, channels, seed):
    """B = 3, 28 frames, 28 * 256 - 7 samples: W = 447, every width dilation up to 128 reaches live columns on both sides and
    the last 128-column tile is partial."""
    from oracle import waveflow_forward as owff
    from parakeet_b200.models import WaveFlowLoss
    m, folded = _model(cuda, channels, seed)
    audio, mel = _inputs(31, 3, 28, 28 * 256 - 7)
    with torch.no_grad():
        ref_z, ref_ld = owff.waveflow_forward(folded, audio, mel)
    assert ref_z.shape[-1] // 16 == 447
    z, log_det = m(audio.to(cuda), mel.to(cuda))
    assert rel_err(z, ref_z) < TOL
    assert _rel(log_det, ref_ld) < 1e-3
    assert _rel(WaveFlowLoss(0.7)(z, log_det), owff.waveflow_loss(ref_z, ref_ld, 0.7)) < 1e-4
    # batch independence: one utterance alone gives its slice of the batch, bit for bit
    z1, _ = m(audio[1:2].to(cuda), mel[1:2].to(cuda))
    assert torch.equal(z1, z[1:2])


def test_zero_output_proj_is_the_identity(cuda):
    """The reference initialises output_proj to zero: every flow copies its input, the 8 permutations compose to the identity,
    so z is the pruned audio bit for bit and the log-det is exactly 0."""
    m, _ = _model(cuda, 64, 4, zero_output_proj=True)
    audio, mel = _inputs(32, 2, 20, 20 * 256 - 3)
    z, log_det = m(audio.to(cuda), mel.to(cuda))
    pruned = audio[:, :audio.shape[1] // 16 * 16]
    assert torch.equal(z.cpu(), pruned)
    assert float(log_det) == 0.0


def test_round_trip_through_the_inverse_at_the_training_shape(cuda):
    """The reference's training batch (examples/waveflow/config.py: 8 clips of 65 frames, hop 256) at the shipped 128 channels:
    inverse(forward(audio).z, untrimmed condition) returns the audio - the new kernels tied to the pinned inverse."""
    m, _ = _model(cuda, 128, 5)
    audio, mel = _inputs(33, 8, 65, 65 * 256)
    audio, mel = audio.to(cuda), mel.to(cuda)
    z, _ = m(audio, mel)
    back = m.inverse(z, m.encode(mel, trim_conv_artifact=False))
    assert back.shape == audio.shape
    assert rel_err(back, audio) < TOL


def test_eager_capture_and_replay_are_bit_identical(cuda):
    m, _ = _model(cuda, 64, 4)
    audio, mel = _inputs(34, 2, 12, 12 * 256)
    audio, mel = audio.to(cuda), mel.to(cuda)
    outs = [m(audio, mel) for _ in range(3)]                # eager, capture (+ replay), replay
    assert m._graphs.replays == 2
    for z, ld in outs[1:]:
        assert torch.equal(z, outs[0][0]) and torch.equal(ld, outs[0][1])
    # the upsampled-condition entry point computes the same
    z, ld = m.decoder_forward(audio, m.encode(mel, trim_conv_artifact=False))
    assert torch.equal(z, outs[0][0]) and torch.equal(ld, outs[0][1])


def test_n_group_8_vs_oracle(cuda):
    from oracle import waveflow_forward as owff
    m, folded = _model(cuda, 64, 4, n_group=8)
    audio, mel = _inputs(35, 2, 10, 10 * 256 - 1)
    with torch.no_grad():
        ref_z, ref_ld = owff.waveflow_forward(folded, audio, mel, n_group=8)
    z, log_det = m(audio.to(cuda), mel.to(cuda))
    assert rel_err(z, ref_z) < TOL
    assert _rel(log_det, ref_ld) < 1e-3
