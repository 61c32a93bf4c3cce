"""Oracle: the GE2E speaker encoder (torch-CPU restatement).  TEST INFRASTRUCTURE ONLY.

Follows the reference parakeet/models/lstm_speaker_encoder.py (`LSTMSpeakerEncoder`) and examples/ge2e/train.py:39-43,62-75
(`Ge2eExperiment.setup_model` / `train_batch`): `loss, eer = model(specs, speakers_per_batch)`, `loss.backward()`,
`do_gradient_ops()` (the gradients of similarity_weight / similarity_bias times 0.01), `Adam(1e-4, ClipGradByGlobalNorm(3))`.

The LSTM is written out gate by gate (Paddle's nn.LSTM: gate order i, f, g, o; `b_ih` and `b_hh` added separately; input
(B, T, I) batch-major; h of shape [num_layers, B, H]).  `forward` keeps the reference's reshape of the (N*M, C) embeddings to
`[num_speakers, -1, num_speakers]` (not [N, M, C]): at the recipe's N = 64, M = 10, C = 256 the loss runs on (64, 40, 64).
"""
import math

import torch

from .fastspeech2 import adam_step

# state-dict keys of one layer: Paddle 2.1's LayerList of RNN(LSTMCell) (emitted) and the flat form of later releases (accepted)
LSTM_PARTS = ("weight_ih", "weight_hh", "bias_ih", "bias_hh")


def lstm_key(layer, part):
    return f"lstm.{layer}.cell.{part}"


def synth_params(seed, n_mels, num_layers, hidden_size, output_size):
    """Seeded Paddle-layout state dict (uniform(+-1/sqrt(H)) like Paddle's LSTM init; Linear weight [in, out])."""
    g = torch.Generator().manual_seed(seed)
    k = 1.0 / math.sqrt(hidden_size)
    u = lambda *shape: (torch.rand(*shape, generator=g) * 2 - 1) * k
    p = {}
    for l in range(num_layers):
        i = n_mels if l == 0 else hidden_size
        p[lstm_key(l, "weight_ih")] = u(4 * hidden_size, i)
        p[lstm_key(l, "weight_hh")] = u(4 * hidden_size, hidden_size)
        p[lstm_key(l, "bias_ih")] = u(4 * hidden_size)
        p[lstm_key(l, "bias_hh")] = u(4 * hidden_size)
    p["linear.weight"] = u(hidden_size, output_size)
    p["linear.bias"] = u(output_size)
    p["similarity_weight"] = torch.tensor([10.0])
    p["similarity_bias"] = torch.tensor([-5.0])
    return p


# the two configurations of tests/golden/ref_executed_ge2e.npz: (n_mels, num_layers, hidden, output), (N, M, frames), seed
GOLDEN_CONFIGS = {"small": ((40, 3, 64, 64), (4, 3, 20), 61), "shipped": ((40, 3, 256, 256), (4, 5, 160), 62)}


def synth_utterances(seed, batch, frames, n_mels):
    """Seeded log-mel-like partials (B, T, n_mels)."""
    return torch.randn(batch, frames, n_mels, generator=torch.Generator().manual_seed(seed)) * 0.5


def synth_states(seed, num_layers, batch, hidden_size):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(num_layers, batch, hidden_size, generator=g) * 0.3, torch.randn(num_layers, batch, hidden_size, generator=g) * 0.3


def num_layers_of(p):
    return len([k for k in p if k.endswith(".cell.weight_ih")])


def lstm(p, x, h0=None, c0=None):
    """x (B, T, I) -> out (B, T, H), (h, c) each [L, B, H]."""
    L = num_layers_of(p)
    B, T, _ = x.shape
    H = p[lstm_key(0, "weight_hh")].shape[1]
    hs, cs = [], []
    for l in range(L):
        w_ih, w_hh = p[lstm_key(l, "weight_ih")], p[lstm_key(l, "weight_hh")]
        b_ih, b_hh = p[lstm_key(l, "bias_ih")], p[lstm_key(l, "bias_hh")]
        h = h0[l] if h0 is not None else x.new_zeros(B, H)
        c = c0[l] if c0 is not None else x.new_zeros(B, H)
        outs = []
        for t in range(T):
            gates = x[:, t] @ w_ih.t() + b_ih + h @ w_hh.t() + b_hh
            i, f, gg, o = gates.chunk(4, dim=1)
            i, f, gg, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(gg), torch.sigmoid(o)
            c = f * c + i * gg
            h = o * torch.tanh(c)
            outs.append(h)
        x = torch.stack(outs, 1)
        hs.append(h)
        cs.append(c)
    return x, (torch.stack(hs), torch.stack(cs))


def normalize(x, axis=1, eps=1e-12):
    """paddle F.normalize: x / max(||x||_2, eps)."""
    return x / x.norm(p=2, dim=axis, keepdim=True).clamp_min(eps)


def embed_sequences(p, utterances, initial_states=None, reduce=False):
    h0, c0 = initial_states if initial_states is not None else (None, None)
    _, (h, _) = lstm(p, utterances, h0, c0)
    embeds = torch.relu(h[-1] @ p["linear.weight"] + p["linear.bias"])
    normalized = normalize(embeds)
    if reduce:
        return normalize(normalized.mean(0), axis=0)
    return normalized


def embed_utterance(p, utterances, initial_states=None):
    return embed_sequences(p, utterances, initial_states, reduce=True)


def similarity_matrix(embeds, w, b):
    """embeds (N, M, C) -> (N*M, N): cosine to the inclusive centroids, the own speaker's entry replaced by the cosine to the
    exclusive centroid, then * w + b (lstm_speaker_encoder.py similarity_matrix; the scatter is an overwrite)."""
    N, M, C = embeds.shape
    incl = embeds.mean(1)
    incl = incl / incl.norm(p=2, dim=1, keepdim=True)
    excl = (embeds.sum(1, keepdim=True).expand(N, M, C) - embeds) / (M - 1)
    excl = excl / excl.norm(p=2, dim=2, keepdim=True)
    p1 = (embeds.reshape(-1, C) @ incl.t()).reshape(-1)
    p2 = (embeds.reshape(-1, C) * excl.reshape(-1, C)).sum(1)
    index = (torch.arange(N * M).reshape(N, M) * N + torch.arange(N).unsqueeze(-1)).reshape(-1)
    mask = torch.ones(N * M * N, dtype=embeds.dtype)
    mask[index] = 0
    own = torch.ones(N * M * N, dtype=embeds.dtype).index_put((index,), p2)
    s = p1 * mask + (1 - mask) * own
    return (s * w + b).reshape(N * M, N)


def loss(embeds, w, b):
    """-> (cross-entropy (scalar), similarity matrix (N*M, N)); target of row (j, i) is speaker j."""
    N, M = embeds.shape[:2]
    sim = similarity_matrix(embeds, w, b)
    target = torch.arange(N).unsqueeze(-1).expand(N, M).reshape(-1)
    return torch.nn.functional.cross_entropy(sim, target), sim


def forward(p, utterances, num_speakers, initial_states=None):
    """LSTMSpeakerEncoder.forward without the EER: -> (loss, similarity matrix).  The reshape is the reference's."""
    e = embed_sequences(p, utterances, initial_states)
    return loss(e.reshape(num_speakers, -1, num_speakers), p["similarity_weight"], p["similarity_bias"])


def train_grads(p, utterances, num_speakers, dtype=torch.float64):
    """-> (loss, {name: gradient after do_gradient_ops}) computed in `dtype`."""
    params = {k: v.detach().to(dtype).clone().requires_grad_(True) for k, v in p.items()}
    l, _ = forward(params, utterances.detach().to(dtype), num_speakers)
    grads = dict(zip(params, torch.autograd.grad(l, list(params.values()))))
    for k in ("similarity_weight", "similarity_bias"):
        grads[k] = grads[k] * 0.01
    return l.detach(), {k: g.detach() for k, g in grads.items()}


def clipped_adam_step(p, grads, state, lr=1e-4, max_grad_norm=3.0):
    """ClipGradByGlobalNorm(max_grad_norm) over the (already 0.01-scaled) gradients, then paddle.optimizer.Adam."""
    norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads.values()))
    scale = max_grad_norm / max(norm, max_grad_norm)
    return adam_step(p, {k: g * scale for k, g in grads.items()}, state, lr=lr), norm
