"""SpeedySpeech (reference parakeet/models/speedyspeech/speedyspeech.py), eval mode, as torch-CPU restatement:
  ResidualBlock :21-39, TextEmbedding :42-73, SpeedySpeechEncoder :76-106, DurationPredictor :109-118,
  SpeedySpeechDecoder :121-138, SpeedySpeech.forward :166-184 / .inference :186-220, SpeedySpeechInference :223-232;
  expand (modules/expansion.py:19-35) is the length regulator's 0/1 matmul of oracle.fastspeech2, paddle.round is its
  paddle_round, sinusoid_position_encoding is modules/positional_encoding.py:20-39.
Paddle's padding="same" follows parakeet_b200.models.speedyspeech.paddle_same_conv (DESIGN.md §2 records the decision).
"""
import math

import torch
import torch.nn.functional as F

from oracle.fastspeech2 import length_regulator_expand, paddle_round
from parakeet_b200.models.speedyspeech import BN_EPS, paddle_same_conv

SHIPPED_CFG = dict(encoder_hidden_size=128, encoder_kernel_size=3, encoder_dilations=[1, 3, 9, 27, 1, 3, 9, 27, 1, 1],
                   duration_predictor_hidden_size=128, decoder_hidden_size=128, decoder_output_size=80, decoder_kernel_size=3,
                   decoder_dilations=[1, 3, 9, 27, 1, 3, 9, 27, 1, 3, 9, 27, 1, 3, 9, 27, 1, 1])
SMALL_CFG = dict(SHIPPED_CFG, encoder_dilations=[1, 3, 9], decoder_dilations=[1, 27])


def conv1d_same(p, name, x, dilation):
    """nn.Conv1D(padding="same", data_format="NLC") on (B, T, C)."""
    w = p[name + ".weight"]
    dil, left, right = paddle_same_conv(w.shape[-1], dilation)
    return F.conv1d(F.pad(x.transpose(1, 2), (left, right)), w, p[name + ".bias"], dilation=dil).transpose(1, 2)


def batch_norm(p, name, x):
    """nn.BatchNorm1D(data_format="NLC"), eval mode: running statistics, eps 1e-5."""
    return (x - p[name + "._mean"]) / torch.sqrt(p[name + "._variance"] + BN_EPS) * p[name + ".weight"] + p[name + ".bias"]


def residual_block(p, pre, x, dilation, n):
    h = x
    for j in range(n):
        h = batch_norm(p, f"{pre}blocks.{j}.2", torch.relu(conv1d_same(p, f"{pre}blocks.{j}.0", h, dilation)))
    return x + h


def linear(p, name, x):
    return x @ p[name + ".weight"] + p[name + ".bias"]


def embedding(table, ids):
    return torch.where((ids == 0).unsqueeze(-1), torch.zeros(()), table[ids])      # padding_idx=0 -> zeros


def encoder(p, cfg, text, tones):
    e = embedding(p["encoder.embedding.text_embedding.weight"], text)
    if tones is not None:
        e = e + embedding(p["encoder.embedding.tone_embedding.weight"], tones)
    e = torch.relu(linear(p, "encoder.prenet.0", e))
    x = e
    for i, d in enumerate(cfg["encoder_dilations"]):
        x = residual_block(p, f"encoder.res_blocks.{i}.", x, d, 2)
    x = e + linear(p, "encoder.postnet1.0", x)
    return linear(p, "encoder.postnet2.2", batch_norm(p, "encoder.postnet2.1", torch.relu(x)))


def duration_predictor(p, x):
    for i in range(3):
        x = residual_block(p, f"duration_predictor.layers.{i}.", x, 1, 1)
    return linear(p, "duration_predictor.layers.3", x).squeeze(-1)


def sinusoid_position_encoding(num_positions, feature_size):
    channel = torch.arange(0, feature_size, 2, dtype=torch.float32)
    index = torch.arange(0, num_positions, 1, dtype=torch.float32)
    angle = index.unsqueeze(-1) / (10000.0 ** (channel / float(feature_size)))
    pe = torch.zeros(num_positions, feature_size)
    pe[:, 0::2] = torch.sin(angle)
    pe[:, 1::2] = torch.cos(angle)
    return pe


def decoder(p, cfg, x):
    xx = x
    for i, d in enumerate(cfg["decoder_dilations"]):
        xx = residual_block(p, f"decoder.res_blocks.{i}.", xx, d, 2)
    x = x + linear(p, "decoder.postnet1.0", xx)
    return linear(p, "decoder.postnet2.1", residual_block(p, "decoder.postnet2.0.", x, 1, 2))


def forward(p, cfg, text, tones, durations):
    """SpeedySpeech.forward (eval): (decoded (B, L, odim), pred_durations (B, T))."""
    enc = encoder(p, cfg, text, tones)
    pred = duration_predictor(p, enc)
    x = length_regulator_expand(enc, durations.to(torch.int64))
    x = x + sinusoid_position_encoding(x.shape[1], x.shape[2])
    return decoder(p, cfg, x), pred


def inference_durations(p, cfg, text, tones=None):
    enc = encoder(p, cfg, text.unsqueeze(0), tones.unsqueeze(0) if tones is not None else None)
    return enc, paddle_round(torch.exp(duration_predictor(p, enc))).to(torch.int64)


def inference(p, cfg, text, tones=None):
    """SpeedySpeech.inference: (T,) ids -> (L, odim)."""
    enc, d = inference_durations(p, cfg, text, tones)
    if int(d.sum()) == 0:
        return torch.zeros(0, cfg["decoder_output_size"])
    x = length_regulator_expand(enc, d)
    x = x + sinusoid_position_encoding(x.shape[1], x.shape[2])
    return decoder(p, cfg, x)[0]


def inference_denorm(p, cfg, text, tones, mu, sigma):
    """SpeedySpeechInference.forward: inference then ZScore.inverse (normalizer.py:30-33)."""
    return inference(p, cfg, text, tones) * sigma + mu


def synth_params(seed, cfg, vocab_size=40, tone_size=None, log_duration=1.6):
    """Seeded Paddle-layout state dict with non-trivial BatchNorm statistics; the duration head's bias sets the typical
    log-duration (exp(1.6) ~ 5 frames per phone)."""
    g = torch.Generator().manual_seed(seed)
    C = cfg["encoder_hidden_size"]
    p = {}

    def lin(name, i, o, gain=1.0):
        p[name + ".weight"] = (torch.rand(i, o, generator=g) * 2 - 1) * gain * math.sqrt(6.0 / (i + o))
        p[name + ".bias"] = (torch.rand(o, generator=g) * 2 - 1) * 0.1

    def bn(name):
        p[name + ".weight"] = 0.5 + torch.rand(C, generator=g)
        p[name + ".bias"] = (torch.rand(C, generator=g) * 2 - 1) * 0.2
        p[name + "._mean"] = torch.rand(C, generator=g) * 0.5
        p[name + "._variance"] = 0.5 + torch.rand(C, generator=g)

    def res_block(pre, k, n):
        for j in range(n):
            q = f"{pre}blocks.{j}."
            p[q + "0.weight"] = (torch.rand(C, C, k, generator=g) * 2 - 1) / math.sqrt(C * k)
            p[q + "0.bias"] = (torch.rand(C, generator=g) * 2 - 1) * 0.1
            bn(q + "2")

    emb = torch.randn(vocab_size, C, generator=g)
    emb[0] = 0
    p["encoder.embedding.text_embedding.weight"] = emb
    if tone_size:
        tone = torch.randn(tone_size, C, generator=g)
        tone[0] = 0
        p["encoder.embedding.tone_embedding.weight"] = tone
    lin("encoder.prenet.0", C, C)
    for i in range(len(cfg["encoder_dilations"])):
        res_block(f"encoder.res_blocks.{i}.", cfg["encoder_kernel_size"], 2)
    lin("encoder.postnet1.0", C, C)
    bn("encoder.postnet2.1")
    lin("encoder.postnet2.2", C, C)
    for i, k in enumerate((4, 3, 1)):
        res_block(f"duration_predictor.layers.{i}.", k, 1)
    lin("duration_predictor.layers.3", C, 1, gain=0.05)
    p["duration_predictor.layers.3.bias"] = torch.full((1,), float(log_duration))
    for i in range(len(cfg["decoder_dilations"])):
        res_block(f"decoder.res_blocks.{i}.", cfg["decoder_kernel_size"], 2)
    lin("decoder.postnet1.0", C, C)
    res_block("decoder.postnet2.0.", cfg["decoder_kernel_size"], 2)
    lin("decoder.postnet2.1", C, cfg["decoder_output_size"])
    return p
