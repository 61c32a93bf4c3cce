"""CPU tests of the SpeedySpeech training step: the oracle restatement (oracle/speedyspeech_train.py) against direct evaluations of the
formulas, the new C symbols, and the host-side validation of SpeedySpeechTrainStep."""
import math

import pytest
import torch

from oracle import speedyspeech_train as sst
from oracle import speedyspeech as oss
from parakeet_b200 import _lib


def test_ssim_restatement_against_direct_fp64_formula():
    g = torch.Generator().manual_seed(0)
    a, b = torch.rand(1, 1, 9, 7, generator=g, dtype=torch.float64), torch.rand(1, 1, 9, 7, generator=g, dtype=torch.float64)
    w1 = [math.exp(-(x - 5) ** 2 / (2 * 1.5 ** 2)) for x in range(11)]
    w1 = [v / sum(w1) for v in w1]

    def filt(img, i, j):
        s = 0.0
        for di in range(11):
            for dj in range(11):
                ii, jj = i + di - 5, j + dj - 5
                if 0 <= ii < 9 and 0 <= jj < 7:
                    s += w1[di] * w1[dj] * float(img[ii, jj])
        return s

    x, y = a[0, 0], b[0, 0]
    total = 0.0
    for i in range(9):
        for j in range(7):
            mx, my = filt(x, i, j), filt(y, i, j)
            sx, sy, sxy = filt(x * x, i, j) - mx * mx, filt(y * y, i, j) - my * my, filt(x * y, i, j) - mx * my
            total += ((2 * mx * my + 1e-4) * (2 * sxy + 9e-4)) / ((mx * mx + my * my + 1e-4) * (sx + sy + 9e-4))
    assert abs(float(sst.ssim(a, b)) - total / 63) < 1e-12
    assert abs(float(sst.ssim(a, a)) - 1.0) < 1e-12


def test_huber_below_at_and_above_delta_and_zero_durations():
    r = torch.tensor([0.25, -1.0, 1.0, 3.0, -2.5], dtype=torch.float64)
    out = sst.huber(torch.zeros(5, dtype=torch.float64), r)
    assert torch.allclose(out, torch.tensor([0.03125, 0.5, 0.5, 2.5, 2.0], dtype=torch.float64))
    batch = dict(feats=torch.zeros(1, 2, 80), num_frames=torch.tensor([2]), num_phones=torch.tensor([2]), durations=torch.tensor([[0, 2]]))
    ls = sst.losses(torch.zeros(1, 2, 80, dtype=torch.float64), torch.tensor([[0.0, math.log(2.0)]], dtype=torch.float64), batch)
    assert abs(float(ls["duration_loss"])) < 1e-15          # log(max(0, 1)) = 0: a zero duration is a target of 0, not -inf
    assert abs(float(ls["l1_loss"])) < 1e-15 and abs(float(ls["ssim_loss"])) < 1e-12


def test_train_mode_oracle_matches_eval_oracle_when_statistics_agree():
    """With the running statistics set to the batch statistics the eval-mode oracle must reproduce the train-mode forward, and
    the duration predictor must give the encoder no gradient."""
    cfg = oss.SMALL_CFG
    p = {k: v.double() for k, v in oss.synth_params(3, cfg, tone_size=5).items()}
    batch = sst.synth_batch(4, [7, 5, 2], tone_size=5)
    stats = {}
    dec, pred = sst.forward_train(p, cfg, batch["phones"], batch["tones"], batch["durations"], stats)
    q = dict(p)
    for k, v in stats.items():                              # running = 0.9 * old + 0.1 * batch -> recover the batch value
        q[k] = (v - 0.9 * p[k]) / 0.1
    dec2, pred2 = oss.forward(q, cfg, batch["phones"], batch["tones"], batch["durations"])
    assert torch.allclose(dec, dec2, atol=1e-9) and torch.allclose(pred, pred2, atol=1e-9)
    assert dec.shape[1] == batch["feats"].shape[1]
    w = {k: v.clone().requires_grad_(not k.endswith(sst.BUFFERS)) for k, v in p.items()}
    _, pred3 = sst.forward_train(w, cfg, batch["phones"], batch["tones"], batch["durations"], {})
    pred3.sum().backward()
    assert w["encoder.prenet.0.weight"].grad is None and w["duration_predictor.layers.3.weight"].grad is not None


def test_gradients_cover_every_trainable_tensor_and_padding_rows_get_none():
    cfg = oss.SMALL_CFG
    p = oss.synth_params(5, cfg, tone_size=4)
    losses, grads, stats = sst.train_step_grads(p, cfg, sst.synth_batch(6, [6, 3], tone_size=4))
    assert set(grads) == {k for k in p if not k.endswith(sst.BUFFERS)} and set(stats) == {k for k in p if k.endswith(sst.BUFFERS)}
    assert all(float(g.abs().max()) > 0 for g in grads.values())
    assert float(grads["encoder.embedding.text_embedding.weight"][0].abs().max()) == 0.0
    assert float(grads["encoder.embedding.tone_embedding.weight"][0].abs().max()) == 0.0
    assert abs(losses["loss"] - losses["l1_loss"] - losses["ssim_loss"] - losses["duration_loss"]) < 1e-12


def fixture_cases():
    import os
    import numpy as np
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_executed_speedyspeech_train.npz"))
    for tag in ("a", "b"):
        get = lambda prefix: {k[len(tag) + 1 + len(prefix):]: torch.from_numpy(z[k]) for k in z.files if k.startswith(f"{tag}/{prefix}")}
        yield tag, int(z[f"{tag}/seed"]), int(z[f"{tag}/tone_size"]), get("batch/"), {k: float(z[f"{tag}/{k}"]) for k in
                                                                                      ("loss", "l1_loss", "duration_loss", "ssim_loss")}, \
            get("grad/"), get("gradnorm/"), get("stat/")


def test_oracle_equals_the_reference_executed_training_fixture():
    """Losses, every parameter gradient and the new running statistics of the reference's own code (fp32) against the oracle."""
    for tag, seed, tone_size, batch, losses, grads, norms, stats in fixture_cases():
        cfg = oss.SMALL_CFG
        p = oss.synth_params(seed, cfg, tone_size=tone_size)
        got_l, got_g, got_s = sst.train_step_grads(p, cfg, batch)
        for k, v in losses.items():
            assert abs(got_l[k] - v) < 2e-6 * max(1.0, abs(v)), (tag, k)
        assert set(got_g) == set(grads) and set(got_s) == set(stats)
        for k, g in grads.items():
            ref, mine = g.double(), sst.fixture_sample(got_g[k])
            assert ((mine - ref).norm() / ref.norm().clamp_min(1e-30)).item() < 2e-3, (tag, k)      # fp32 reference against fp64
            assert abs(float(got_g[k].norm()) - float(norms[k])) < 2e-3 * float(norms[k]) + 1e-12, (tag, k)
        for k, v in stats.items():
            assert torch.allclose(got_s[k].float(), v, rtol=1e-5, atol=1e-6), (tag, k)


def test_clipped_adam_scales_only_above_the_threshold():
    p = {"w": torch.ones(4, dtype=torch.float64)}
    g = {"w": torch.full((4,), 2.0, dtype=torch.float64)}            # norm 4
    a, n1 = sst.clipped_adam_step(p, g, {}, lr=0.1, max_grad_norm=1.0)
    b, _ = sst.clipped_adam_step(p, {"w": g["w"] / 4}, {}, lr=0.1, max_grad_norm=1.0)
    assert n1 == 4.0 and torch.equal(a["w"], b["w"])


def test_new_symbols_are_exported_and_reject_bad_arguments():
    L = _lib.lib()
    for name in ("pk_ss_bn_train_fwd", "pk_ss_bn_relu_bwd", "pk_ss_loss"):
        assert name in _lib.exported_symbols() and hasattr(L, name)
    assert L.pk_ss_bn_train_fwd(None, 4, 128, None, None, 1e-5, 0.9, None, None, None, None, None, None, None, None, None, None) == -1
    assert L.pk_ss_bn_relu_bwd(None, None, None, None, None, 4, 128, None, None, None, None, None, None, None, None) == -1
    assert L.pk_ss_loss(None, None, None, 1, 1, 80, None, None, None, 1, None, None, None, None, None) == -1
    assert b"NULL" in L.pk_last_error()


def test_step_is_exported_and_refuses_what_it_cannot_run():
    from parakeet_b200.models import SpeedySpeech
    from parakeet_b200.training import SpeedySpeechTrainStep
    with pytest.raises(_lib.PkError):                              # hidden size != 128: the model's constructor refuses
        SpeedySpeech(vocab_size=40, **dict(oss.SMALL_CFG, encoder_hidden_size=64))
    m = SpeedySpeech(vocab_size=40, device="cpu", **oss.SMALL_CFG)
    with pytest.raises(_lib.PkError, match="CUDA"):
        SpeedySpeechTrainStep(m)
    with pytest.raises(_lib.PkError):
        SpeedySpeechTrainStep(object())
