"""Oracle: the WaveFlow training step (torch-CPU restatement).  TEST INFRASTRUCTURE ONLY.

Follows the reference examples/waveflow/train.py:95-118 (Experiment.train_batch): `z, log_det = model(wav, mel)`,
`loss = WaveFlowLoss(sigma)(z, log_det)`, `loss.backward()`, `paddle.optimizer.Adam`.  The gradients come from torch autograd
through oracle.waveflow_forward.waveflow_forward with the weight norm folded INSIDE the graph, so they are taken with respect
to the trainable tensors (`weight_g` / `weight_v` pairs, biases, `output_proj.*`, the encoder's Conv2DTranspose g / v / bias).
Adam is oracle.fastspeech2.adam_step (Paddle's update; β 0.9 / 0.999, ε 1e-8, no clipping).
"""
import torch

from .fastspeech2 import adam_step  # noqa: F401  (re-exported: the WaveFlow recipe's optimiser)
from .waveflow import fold_weight_norm
from .waveflow_forward import waveflow_forward, waveflow_loss


def n_upsample(p):
    return len({k.split(".")[1] for k in p if k.startswith("encoder.")})


def train_grads(p, audio, mel, n_flows, n_layers, n_group, sigma=1.0, dtype=torch.float64):
    """-> (loss (1,), {name: gradient}) for every tensor of `p`, computed in `dtype`."""
    params = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in p.items()}
    z, log_det = waveflow_forward(fold_weight_norm(params), audio.detach().to(dtype), mel.detach().to(dtype), n_up=n_upsample(p),
                                  n_flows=n_flows, n_layers=n_layers, n_group=n_group)
    loss = waveflow_loss(z, log_det, sigma)
    grads = torch.autograd.grad(loss, list(params.values()))
    return loss.detach(), {k: g.detach() for k, g in zip(params, grads)}
