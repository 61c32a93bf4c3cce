"""The SpeedySpeech training step restated on the oracle (torch-CPU + autograd, any float dtype): what the CUDA step is checked
against, itself pinned to the reference's own train-mode SpeedySpeech, masked_l1_loss, weighted_mean and ssim executed on the Paddle
stand-in (scripts/make_golden_ref.py speedyspeech_train -> tests/golden/ref_executed_speedyspeech_train.npz).  SpeedySpeechUpdater.update_core (speedyspeech_updater.py:48-85) with the model in train() mode: every BatchNorm1D
takes its batch statistics over all rows and returns the new running statistics (momentum 0.9, biased variance), the duration
predictor reads encodings.detach(), loss = masked_l1 (modules/losses.py:60-100) + (1 - ssim) (modules/ssim.py:21-80) +
weighted_mean(huber) with fluid.layers.huber_loss(input, label, delta): r = label - input, 0.5 r^2 for |r| <= delta, else
delta (|r| - 0.5 delta).  The eval-mode pieces come from oracle.speedyspeech unchanged; Adam from oracle.fastspeech2.adam_step
with ClipGradByGlobalNorm in front (training/optimizer.py:29-46).  Restated Paddle primitive of this module (Paddle is not
installable here; re-verify where it is): fluid.layers.huber_loss as written above, from huber_loss_op.h."""
import math

import torch
import torch.nn.functional as F

from oracle import speedyspeech as oss
from oracle.fastspeech2 import adam_step, length_regulator_expand
from parakeet_b200.models.speedyspeech import BN_EPS

BUFFERS = ("_mean", "_variance")


def bn_train(p, name, x, new_stats):
    flat = x.reshape(-1, x.shape[-1])
    mean, var = flat.mean(0), flat.var(0, unbiased=False)
    new_stats[name + "._mean"] = (0.9 * p[name + "._mean"] + 0.1 * mean).detach()
    new_stats[name + "._variance"] = (0.9 * p[name + "._variance"] + 0.1 * var).detach()
    return (x - mean) / torch.sqrt(var + BN_EPS) * p[name + ".weight"] + p[name + ".bias"]


def residual_block(p, pre, x, n, new_stats):
    h = x
    for j in range(n):
        h = bn_train(p, f"{pre}blocks.{j}.2", torch.relu(oss.conv1d_same(p, f"{pre}blocks.{j}.0", h, 1)), new_stats)
    return x + h


def embedding(table, ids):
    return torch.where((ids == 0).unsqueeze(-1), torch.zeros((), dtype=table.dtype), table[ids])


def forward_train(p, cfg, text, tones, durations, new_stats):
    """SpeedySpeech.forward (:166-184) in train() mode -> (decoded (B, L, odim), pred_durations (B, T))."""
    e = embedding(p["encoder.embedding.text_embedding.weight"], text)
    if tones is not None:
        e = e + embedding(p["encoder.embedding.tone_embedding.weight"], tones)
    e = torch.relu(oss.linear(p, "encoder.prenet.0", e))
    x = e
    for i in range(len(cfg["encoder_dilations"])):
        x = residual_block(p, f"encoder.res_blocks.{i}.", x, 2, new_stats)
    x = e + oss.linear(p, "encoder.postnet1.0", x)
    enc = oss.linear(p, "encoder.postnet2.2", bn_train(p, "encoder.postnet2.1", torch.relu(x), new_stats))
    h = enc.detach()
    for i in range(3):
        h = residual_block(p, f"duration_predictor.layers.{i}.", h, 1, new_stats)
    pred = oss.linear(p, "duration_predictor.layers.3", h).squeeze(-1)
    x = length_regulator_expand(enc, durations.to(torch.int64))
    x = x + oss.sinusoid_position_encoding(x.shape[1], x.shape[2]).to(x.dtype)
    xx = x
    for i in range(len(cfg["decoder_dilations"])):
        xx = residual_block(p, f"decoder.res_blocks.{i}.", xx, 2, new_stats)
    x = x + oss.linear(p, "decoder.postnet1.0", xx)
    return oss.linear(p, "decoder.postnet2.1", residual_block(p, "decoder.postnet2.0.", x, 2, new_stats)), pred


def sequence_mask(lengths, maxlen, dtype):
    return (torch.arange(maxlen)[None, :] < lengths[:, None]).to(dtype)


def masked_l1(pred, target, mask):
    return ((pred - target).abs() * mask).sum() / (mask.sum() * (pred.numel() / mask.numel()))


def huber(inp, label, delta=1.0):
    r = label - inp
    return torch.where(r.abs() <= delta, 0.5 * r * r, delta * (r.abs() - 0.5 * delta))


def ssim(img1, img2, window_size=11):
    """(B, 1, H, W) images: mean of the SSIM map, the 2-D Gaussian window applied with zero padding."""
    g = torch.tensor([math.exp(-(x - window_size // 2) ** 2 / (2 * 1.5 ** 2)) for x in range(window_size)], dtype=img1.dtype)
    g = g / g.sum()
    w = (g[:, None] @ g[None, :])[None, None]
    f = lambda im: F.conv2d(im, w, padding=window_size // 2)
    mu1, mu2 = f(img1), f(img2)
    s1, s2, s12 = f(img1 * img1) - mu1 * mu1, f(img2 * img2) - mu2 * mu2, f(img1 * img2) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    return (((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 * mu1 + mu2 * mu2 + c1) * (s1 + s2 + c2))).mean()


def losses(decoded, pred, batch):
    """update_core :57-80 -> dict of the four tensors."""
    feats = batch["feats"].to(decoded.dtype)
    spec_mask = sequence_mask(batch["num_frames"], feats.shape[1], decoded.dtype).unsqueeze(-1)
    text_mask = sequence_mask(batch["num_phones"], pred.shape[1], decoded.dtype)
    l1 = masked_l1(decoded, feats, spec_mask)
    target = torch.log(torch.clamp(batch["durations"].to(decoded.dtype), min=1.0))
    dur = (huber(pred, target) * text_mask).sum() / text_mask.sum()
    ss = 1.0 - ssim((decoded * spec_mask).unsqueeze(1), (feats * spec_mask).unsqueeze(1))
    return dict(loss=l1 + ss + dur, l1_loss=l1, duration_loss=dur, ssim_loss=ss)


def train_step_grads(p, cfg, batch, dtype=torch.float64):
    """-> (losses as floats, gradient of every trainable tensor, new running statistics), evaluated in `dtype`."""
    q = {k: v.to(dtype).clone() for k, v in p.items()}
    for k, v in q.items():
        if not k.endswith(BUFFERS):
            v.requires_grad_(True)
    new_stats = {}
    decoded, pred = forward_train(q, cfg, batch["phones"], batch.get("tones"), batch["durations"], new_stats)
    ls = losses(decoded, pred, batch)
    ls["loss"].backward()
    grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in q.items() if not k.endswith(BUFFERS)}
    return {k: float(v.detach()) for k, v in ls.items()}, grads, new_stats


def eval_losses(p, cfg, batch):
    """SpeedySpeechEvaluator.evaluate_core (:110-157): eval-mode forward, same losses."""
    with torch.no_grad():
        decoded, pred = oss.forward(p, cfg, batch["phones"], batch.get("tones"), batch["durations"])
        return {k: float(v) for k, v in losses(decoded, pred, batch).items()}


def clipped_adam_step(p, grads, state, lr=2e-3, max_grad_norm=1.0):
    """ClipGradByGlobalNorm(max_grad_norm) then paddle.optimizer.Adam; returns the new parameters and the gradient norm."""
    norm = math.sqrt(sum(float((g.double() ** 2).sum()) for g in grads.values()))
    scale = max_grad_norm / max(norm, max_grad_norm)
    new = adam_step({k: p[k] for k in grads}, {k: g * scale for k, g in grads.items()}, state, lr=lr)
    return {**p, **new}, norm


def fixture_sample(t, n=1024):
    """How the reference-executed fixture stores a gradient: every stride-th element, stride = numel // n (all of it up to n)."""
    flat = t.detach().reshape(-1)
    return flat[::max(1, flat.numel() // n)]


def synth_batch(seed, lens, vocab_size=40, tone_size=None, max_dur=6):
    """Seeded batch with the keys of the reference's speedyspeech_batch_fn; the longest utterance fills feats exactly."""
    g = torch.Generator().manual_seed(seed)
    B, T = len(lens), max(lens)
    phones, durations = torch.zeros(B, T, dtype=torch.int64), torch.zeros(B, T, dtype=torch.int64)
    tones = torch.zeros(B, T, dtype=torch.int64) if tone_size else None
    for b, n in enumerate(lens):
        phones[b, :n] = torch.randint(1, vocab_size, (n,), generator=g)
        durations[b, :n] = torch.randint(0, max_dur + 1, (n,), generator=g)
        durations[b, 0] = max(int(durations[b, 0]), 1)
        if tone_size:
            tones[b, :n] = torch.randint(1, tone_size, (n,), generator=g)
    num_frames = durations.sum(1)
    feats = torch.randn(B, int(num_frames.max()), 80, generator=g)
    feats = feats * sequence_mask(num_frames, feats.shape[1], feats.dtype).unsqueeze(-1)
    batch = dict(phones=phones, num_phones=torch.tensor(lens, dtype=torch.int64), num_frames=num_frames, feats=feats, durations=durations)
    if tone_size:
        batch["tones"] = tones
    return batch
