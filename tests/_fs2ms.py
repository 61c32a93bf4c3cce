"""The multi-speaker FastSpeech2 training step restated on the oracle (torch-CPU fp32 + autograd): what the CUDA step is
checked against.  oracle.fastspeech2.fs2_forward already integrates spk_id (fastspeech2.py:395-401); this is
oracle.fastspeech2.train_step_grads with the speaker ids passed through, as FastSpeech2Updater.update_core passes them
(fastspeech2_updater.py:51-99: spk_id only, never spembs).  tests/golden/ref_executed_fs2ms_train.npz pins it to the
reference's own code (tests/test_fs2_multispeaker_training_cpu.py)."""
import torch

from oracle import fastspeech2 as ofs

NUM_SPEAKERS = 6


def cfg(spk_type, num_speakers=NUM_SPEAKERS):
    """The aishell3 / vctk model (conf/default.yaml: the ljspeech model + spk_embed_dim 256, concat)."""
    return dict(ofs.LJSPEECH_MODEL_CFG, num_speakers=num_speakers, spk_embed_dim=256, spk_embed_integration_type=spk_type)


def params(spk_type, seed=1, num_speakers=NUM_SPEAKERS):
    """Seeded Paddle-layout parameters with the speaker table / projection and no tone tensors."""
    p = ofs.add_speaker_tone_params(ofs.synth_params(seed), seed, spk_type=spk_type, num_speakers=num_speakers)
    return {k: v for k, v in p.items() if not k.startswith("tone_")}


def model(spk_type, p, device, num_speakers=NUM_SPEAKERS, **kw):
    from parakeet_b200.models import FastSpeech2
    m = FastSpeech2(80, 80, **cfg(spk_type, num_speakers), stop_gradient_from_pitch_predictor=True, device=device, **kw)
    m.set_state_dict(p)
    return m


def train_step_grads(p, spk_type, batch, spk_id, stop_gradient_from_pitch_predictor=True, stop_gradient_from_energy_predictor=False,
                     dropout=None, rates=None):
    """-> (losses dict, grads dict keyed like p, new BatchNorm running statistics); spk_id int64 (B,)."""
    q = {k: (v.clone().requires_grad_(True) if not k.endswith(ofs.BUFFER_SUFFIXES) else v.clone()) for k, v in p.items()}
    new_stats = {}
    out = ofs.fs2_forward(q, cfg(spk_type), batch["text"], batch["text_lengths"], batch["speech_lengths"], batch["durations"],
                          batch["pitch"], batch["energy"], train_bn=True, new_stats=new_stats,
                          stop_gradient_from_pitch_predictor=stop_gradient_from_pitch_predictor,
                          stop_gradient_from_energy_predictor=stop_gradient_from_energy_predictor, dropout=dropout, rates=rates,
                          spk_id=torch.as_tensor(spk_id, dtype=torch.int64))
    l1, dur, pitch, energy = ofs.fs2_loss(out[1], out[0], out[2], out[3], out[4], batch["speech"], batch["durations"], batch["pitch"],
                                          batch["energy"], batch["text_lengths"], batch["speech_lengths"])
    loss = l1 + dur + pitch + energy
    loss.backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in q.items() if not k.endswith(ofs.BUFFER_SUFFIXES)}
    losses = {k: float(v.detach()) for k, v in dict(l1_loss=l1, duration_loss=dur, pitch_loss=pitch, energy_loss=energy, loss=loss).items()}
    return losses, grads, new_stats
