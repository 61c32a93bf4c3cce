"""Oracle: ConditionalWaveFlow density direction (torch-CPU fp32 restatement).  TEST INFRASTRUCTURE ONLY.

Follows the reference parakeet/models/waveflow.py: ConditionalWaveFlow.forward :759-783 (the encoder WITHOUT the trim of
infer), WaveFlow._trim :617-625 and forward :627-672 (fold, every flow followed by the permutation of both x and the condition
along the height, unfold, log_det = sum of all logs), WaveFlowLoss :855-891.  Built on oracle.waveflow: its encoder,
create_perm and the full (non-incremental) flow_forward.
"""
import math

import torch

from .waveflow import create_perm, encoder, flow_forward


def waveflow_forward(p, audio, mel, n_up=2, n_flows=8, n_layers=8, n_group=16):
    """ConditionalWaveFlow.forward (:759-783): audio (B, T), mel (B, C, T') -> (z (B, T // n_group * n_group), log_det (1,))."""
    condition = encoder(p, mel, n_up, trim_conv_artifact=False)
    return decoder_forward(p, audio, condition, n_flows, n_layers, n_group)


def decoder_forward(p, audio, condition, n_flows, n_layers, n_group):
    """WaveFlow.forward (:627-672) on an upsampled condition (B, C, T_c >= T)."""
    assert condition.shape[-1] >= audio.shape[-1]
    pruned = audio.shape[-1] // n_group * n_group
    x, condition = audio[:, :pruned], condition[:, :, :pruned]
    B = x.shape[0]
    x = x.reshape(B, -1, n_group).transpose(1, 2).unsqueeze(1)                        # (B, 1, H, W)
    condition = condition.reshape(B, condition.shape[1], -1, n_group).transpose(2, 3)  # (B, C, H, W)
    perms = create_perm(n_group, n_flows)
    logs_list = []
    for i in range(n_flows):
        x, logs = flow_forward(p, f"decoder.{i}.", x, condition, n_layers, n_group)
        logs_list.append(logs)
        pi = torch.tensor(perms[i])
        x = x.index_select(2, pi)
        condition = condition.index_select(2, pi)
    z = x.squeeze(1).transpose(1, 2).reshape(B, -1)
    return z, torch.sum(torch.stack(logs_list)).reshape(1)


def waveflow_loss(z, log_det, sigma=1.0):
    """WaveFlowLoss (:855-891): (sum z^2 / (2 sigma^2) - log_det) / numel(z) + log(2 pi) / 2 + log(sigma), shape (1,)."""
    loss = (torch.sum(z * z) / (2 * sigma * sigma) - log_det) / z.numel()
    return (loss + 0.5 * math.log(2 * math.pi) + math.log(sigma)).reshape(1)
