"""GPU parity of the multi-speaker FastSpeech2 training step (aishell3 / vctk: spk_id -> spk_embedding_table -> F.normalize
-> "concat" / "add" projection) against torch autograd on the oracle (tests/_fs2ms.py), and of its speaker kernels against fp64."""
import numpy as np
import pytest
import torch

import _fs2ms

pytestmark = pytest.mark.gpu

SPK3 = [3, 0, 3]                                   # a repeated speaker and the padding id; 1, 2, 4, 5 absent
AISHELL3_SPEAKERS = 218
SPK8 = [5, 0, 17, 5, 217, 3, 17, 100]


def _lengths(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(60, 141, (n,), generator=g).tolist()          # the aishell3 per-GPU shape: 8 utterances of 60..140 phonemes


def _batch(seed, lengths, spk, **kw):
    from oracle import fastspeech2 as ofs
    b = ofs.synth_train_batch(seed, lengths, **kw)
    b["spk_id"] = torch.tensor(spk, dtype=torch.int64)
    return b


def _step(spk_type, p, cuda, num_speakers=_fs2ms.NUM_SPEAKERS, lr=1e-3, dropout=False, seed=0, use_graphs=None, rates=None):
    from parakeet_b200.training import FastSpeech2TrainStep
    m = _fs2ms.model(spk_type, p, cuda, num_speakers, **(rates or {}))
    return m, FastSpeech2TrainStep(m, learning_rate=lr, dropout=dropout, seed=seed, use_graphs=use_graphs)


def test_speaker_kernels_vs_fp64(cuda):
    """pk_spk_embed_fwd, pk_spk_time_sum, pk_spk_normalize_bwd and pk_spk_table_grad against fp64 torch: duplicate ids, the
    padding id, absent speakers (exact zeros), every Tmax row summed, and two runs bit-identical."""
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(3)
    N, D, T, A = 9, 256, 37, 384
    table = torch.randn(N, D, generator=g, dtype=torch.float64)
    ids = torch.tensor([3, 0, 3, 5, 1, 3, 8], dtype=torch.int64)
    B = ids.numel()
    x = table[ids] * (ids != 0).unsqueeze(-1)
    xr = x.clone().requires_grad_(True)
    e_ref = torch.nn.functional.normalize(xr, p=2, dim=1, eps=1e-12)
    dcat = torch.randn(B, T, A + D, generator=g, dtype=torch.float64)
    de_ref = dcat[:, :, A:].sum(1)                                       # all T rows
    e_ref.backward(de_ref)
    dtab_ref = torch.zeros(N, D, dtype=torch.float64).index_add_(0, ids, xr.grad * (ids != 0).unsqueeze(-1))
    outs = []
    for _ in range(2):
        tc, ic, dc = table.float().to(cuda), ids.to(cuda), dcat.float().to(cuda).contiguous()
        e, norms = ops.spk_embed_fwd(tc, ic, 0)
        de, dhs = ops.spk_time_sum(dc, A, D, dhs_cols=A)
        dsum_add, none = ops.spk_time_sum(dc, 0, A)
        dx = ops.spk_normalize_bwd(e, norms, de, ic, N, 0)
        dtab = torch.full((N, D), float("nan"), device=cuda)              # every row must be written
        ops.spk_table_grad(dx, ic, dtab, 0)
        torch.cuda.synchronize()
        outs.append([t.cpu() for t in (e, norms, de, dhs, dsum_add, dx, dtab)])
        assert none is None
    for a, b in zip(*outs):
        assert torch.equal(a, b)                                          # no atomics: bit-identical
    e, norms, de, dhs, dsum_add, dx, dtab = outs[0]

    def rel(a, b):
        return ((a.double() - b).abs().max() / b.abs().max()).item()
    assert rel(e, e_ref.detach()) < 1e-6 and rel(norms, x.norm(dim=1)) < 1e-6
    assert torch.equal(dhs, dcat[:, :, :A].float())
    assert rel(de, de_ref) < 1e-5 and rel(dsum_add, dcat[:, :, :A].sum(1)) < 1e-5
    assert rel(dx[ids != 0], xr.grad[ids != 0]) < 1e-5
    assert torch.equal(dx[ids == 0], torch.zeros_like(dx[ids == 0]))      # padding id: exact zeros, no NaN
    assert rel(dtab, dtab_ref) < 1e-5
    for r in (0, 2, 4, 6, 7):                                              # padding row and absent speakers
        assert torch.equal(dtab[r], torch.zeros(D)), r


def _check_grads(ts, grads_ref, strict_keys, loose):
    """Every tensor within 5e-3 relative L2 (the cfg5 criterion of test_gpu_training.py) and at most 15 % of them outside 1e-3:
    at the aishell3 shape 25 (concat) and 21 (add) of 193 tensors land between 1e-3 and 2.5e-3 on an H100, nearly all of them
    pitch predictor, pitch embedding and postnet gradients, which are off the speaker path's backward: the projection adds one
    more split-bf16 GEMM to the forward, and the L1 loss turns that forward rounding into sign flips of a few frame gradients.
    With loose=True (3 utterances, where a ReLU pre-activation within rounding of 0 moves a weight gradient by percents -
    test_gpu_training.py) 5e-2 for every tensor.  The speaker path's own tensors are held to 5e-3 in both cases."""
    errs = {}
    for k, gref in grads_ref.items():
        g, r = ts.grads[k].detach().double().cpu(), gref.double()
        if k.endswith("self_attn.linear_k.bias"):        # true gradient 0 (softmax ignores a per-row shift): rounding noise in both
            assert g.abs().max().item() < 1e-4 and r.abs().max().item() < 1e-4, k
            continue
        d = (g - r).norm().item()
        errs[k] = 0.0 if d <= 1e-7 else d / max(r.norm().item(), 1e-12)
    worst = sorted(errs.items(), key=lambda t: -t[1])
    for k in strict_keys:
        assert errs[k] < 5e-3, (k, errs[k])
    if loose:
        assert worst[0][1] < 5e-2, worst[:8]
    else:
        assert worst[0][1] < 5e-3, worst[:8]
        assert sum(e > 1e-3 for _, e in worst) <= 0.15 * len(worst), worst[:32]


SPK_KEYS = ("spk_embedding_table.weight", "spk_projection.weight", "spk_projection.bias")


@pytest.mark.parametrize("spk_type", ["concat", "add"])
@pytest.mark.parametrize("shape", ["3utt", "aishell3"])
def test_multispeaker_step_gradients_vs_oracle(cuda, spk_type, shape):
    if shape == "3utt":
        n_spk, batch = _fs2ms.NUM_SPEAKERS, _batch(13, [19, 27, 22], SPK3)
    else:
        n_spk, batch = AISHELL3_SPEAKERS, _batch(51, _lengths(8, 50), SPK8)
    p = _fs2ms.params(spk_type, num_speakers=n_spk)
    losses_ref, grads_ref, stats_ref = _fs2ms.train_step_grads(p, spk_type, batch, batch["spk_id"])
    m, ts = _step(spk_type, p, cuda, n_spk)
    got = [float(v) for v in ts.forward_backward(batch)]
    ref = [losses_ref[k] for k in ("l1_loss", "duration_loss", "pitch_loss", "energy_loss")]
    assert np.allclose(got, ref, rtol=1e-3), (got, ref)
    _check_grads(ts, grads_ref, SPK_KEYS, loose=shape == "3utt")
    tab = ts.grads["spk_embedding_table.weight"].cpu()
    present = set(batch["spk_id"].tolist()) - {0}
    for r in range(n_spk):
        if r not in present:
            assert torch.equal(tab[r], torch.zeros_like(tab[r])), r          # dense gradient: exact zeros, row 0 included
    for k, v in stats_ref.items():                                         # BatchNorm running statistics
        got, r = m.state_dict()[k].detach().double().cpu(), v.double()
        assert (got - r).abs().max().item() <= 2e-3 * r.abs().max().item() + 2e-6, k


def test_multispeaker_three_step_adam_trajectory(cuda):
    """Three steps with different speakers each step: speaker 3 is in step 1 only, so in steps 2-3 its row moves by Adam's
    momentum alone; rows of speakers never seen and row 0 stay bit-identical."""
    from oracle import fastspeech2 as ofs
    spk_type, lr = "concat", 2e-5
    p = _fs2ms.params(spk_type)
    base = _batch(52, _lengths(4, 53), [3, 0, 3, 1])
    spks = ([3, 0, 3, 1], [1, 0, 5, 5], [5, 1, 0, 0])
    p_ref, state, loss_ref = dict(p), {}, []
    for s in spks:
        losses, grads, stats = _fs2ms.train_step_grads(p_ref, spk_type, base, torch.tensor(s))
        loss_ref.append(losses["loss"])
        p_ref = {**p_ref, **ofs.adam_step({k: p_ref[k] for k in grads}, grads, state, lr=lr), **stats}
    m, ts = _step(spk_type, p, cuda, lr=lr)
    loss_got = [float(ts.step(dict(base, spk_id=torch.tensor(s))).sum()) for s in spks]
    assert np.allclose(loss_got, loss_ref, rtol=2e-3), (loss_got, loss_ref)
    tab, tab0, tab_ref = m.state_dict()["spk_embedding_table.weight"].cpu(), p["spk_embedding_table.weight"], p_ref["spk_embedding_table.weight"]
    for r in (0, 2, 4):
        assert torch.equal(tab[r], tab0[r]), r
    for r in (1, 3, 5):
        moved = (tab_ref[r] - tab0[r]).norm().item()
        assert moved > 0 and (tab[r] - tab_ref[r]).norm().item() < 5e-2 * moved, r
    sd = m.state_dict()
    for k in ("spk_projection.weight", "spk_projection.bias"):
        d = (sd[k].cpu().double() - p_ref[k].double()).norm().item() / (p_ref[k] - p[k]).double().norm().item()
        assert d < 5e-2, (k, d)


def test_multispeaker_step_with_the_shipped_dropout_rates_vs_oracle(cuda):
    from oracle import fastspeech2 as ofs
    spk_type, seed = "concat", 2024
    p = _fs2ms.params(spk_type)
    batch = _batch(61, _lengths(4, 62), [2, 0, 4, 2])
    rates = dict(ofs.YAML_DROPOUT)
    losses_ref, grads_ref, _ = _fs2ms.train_step_grads(p, spk_type, batch, batch["spk_id"], dropout=ofs.PhiloxDropout(seed, 1), rates=rates)
    m, ts = _step(spk_type, p, cuda, dropout=True, seed=seed, rates=rates)
    got = [float(v) for v in ts.forward_backward(batch)]
    ref = [losses_ref[k] for k in ("l1_loss", "duration_loss", "pitch_loss", "energy_loss")]
    assert np.allclose(got, ref, rtol=1e-3), (got, ref)
    errs = []
    for k, gref in grads_ref.items():
        if k.endswith("self_attn.linear_k.bias"):                      # true gradient 0: rounding noise in both
            continue
        g, r = ts.grads[k].detach().double().cpu(), gref.double()
        if k.endswith("embed.1.alpha") or k.endswith("embed.0.alpha"):
            # one scalar summing dx * PE over every token and channel: on this batch and these masks the encoder's sum cancels
            # to 0.016 (0.14 for the single-speaker model on the same batch and masks), so hold its ABSOLUTE error to what the
            # single-speaker step shows there (8.6e-4 on an H100; 8.8e-4 here)
            assert (g - r).abs().max().item() < 2e-3, (k, float(g), float(r))
            continue
        if (g - r).norm().item() > 1e-7:
            errs.append((k, (g - r).norm().item() / max(r.norm().item(), 1e-12)))
    errs.sort(key=lambda t: -t[1])
    assert not errs or errs[0][1] < 2e-2, errs[:8]
    assert sum(e > 5e-3 for _, e in errs) <= 0.1 * len(grads_ref), errs[:24]
    assert all(e < 5e-3 for k, e in errs if k in SPK_KEYS), [t for t in errs if t[0] in SPK_KEYS]


def test_multispeaker_graph_replay_with_new_speakers_equals_eager(cuda):
    """The captured graph reads spk_id from its input tensor: replays with other speakers (same batch size) equal eager."""
    spk_type = "add"
    p = _fs2ms.params(spk_type)
    base = _batch(71, [20, 33, 27], SPK3)
    spks = ([3, 0, 3], [1, 2, 5], [0, 4, 4], [5, 5, 1], [2, 0, 1])
    runs = []
    for graphs in (False, True):
        m, ts = _step(spk_type, p, cuda, lr=2e-5, use_graphs=graphs)
        losses = [float(ts.step(dict(base, spk_id=torch.tensor(s))).sum()) for s in spks]
        runs.append((losses, {k: v.detach().double().cpu().clone() for k, v in m.state_dict().items()}, ts))
    assert runs[1][2]._fb_graphs.replays >= 3 and runs[0][2]._fb_graphs.replays == 0
    assert np.allclose(runs[0][0], runs[1][0], rtol=2e-4), (runs[0][0], runs[1][0])
    for k, v in runs[0][1].items():
        init = p[k].double()
        if (v - init).abs().max().item() < 2e-5 or k.endswith("self_attn.linear_k.bias"):
            continue
        d = (runs[1][1][k] - v).norm().item() / max((v - init).norm().item(), 1e-12)
        assert d < 5e-2, (k, d)
    tab_e, tab_g = runs[0][1]["spk_embedding_table.weight"], runs[1][1]["spk_embedding_table.weight"]
    assert torch.equal(tab_e[0], p["spk_embedding_table.weight"][0].double()) and torch.equal(tab_g[0], tab_e[0])
    for r in range(1, _fs2ms.NUM_SPEAKERS):                               # every speaker was in some batch: all rows moved
        assert not torch.equal(tab_g[r], p["spk_embedding_table.weight"][r].double()), r


def test_multispeaker_checkpoint_round_trip_then_resume_equals_uninterrupted(cuda):
    from oracle import fastspeech2 as ofs
    spk_type = "concat"
    p = _fs2ms.params(spk_type)
    base = _batch(81, [18, 25, 21], SPK3)
    spks = ([3, 0, 3], [1, 2, 3], [4, 0, 5])
    rates = dict(ofs.YAML_DROPOUT)
    m1, ts1 = _step(spk_type, p, cuda, lr=2e-5, dropout=True, seed=9, rates=rates)
    full = [float(ts1.step(dict(base, spk_id=torch.tensor(s))).sum()) for s in spks]
    m2, ts2 = _step(spk_type, p, cuda, lr=2e-5, dropout=True, seed=9, rates=rates)
    part = [float(ts2.step(dict(base, spk_id=torch.tensor(s))).sum()) for s in spks[:2]]
    state = ts2.state_dict(epoch=1)
    assert "spk_embedding_table.weight_moment1_0" in state["main_optimizer"] and "spk_projection.weight_moment2_0" in state["main_optimizer"]
    state = {"main_params": {k: v.cpu() for k, v in state["main_params"].items()},
             "main_optimizer": {k: (v.cpu() if torch.is_tensor(v) else v) for k, v in state["main_optimizer"].items()},
             "epoch": state["epoch"], "iteration": state["iteration"]}
    m3, ts3 = _step(spk_type, _fs2ms.params(spk_type, seed=2), cuda, lr=2e-5, dropout=True, seed=9, rates=rates)
    ts3.set_state_dict(state)
    part.append(float(ts3.step(dict(base, spk_id=torch.tensor(spks[2]))).sum()))
    assert np.allclose(part, full, rtol=1e-4), (part, full)
    a, b = m1.state_dict(), m3.state_dict()
    for k, v in a.items():
        v, init = v.double().cpu(), p[k].double()
        if (v - init).abs().max().item() < 2e-5 or k.endswith("self_attn.linear_k.bias"):
            continue                                                    # zero-gradient tensors (see the graph replay test)
        assert (b[k].double().cpu() - v).norm().item() < 2e-2 * (v - init).norm().item(), k
    assert torch.equal(b["spk_embedding_table.weight"][0].cpu(), p["spk_embedding_table.weight"][0])


def test_multispeaker_training_reduces_loss(cuda):
    for spk_type in ("concat", "add"):
        m, ts = _step(spk_type, _fs2ms.params(spk_type), cuda)
        batch = _batch(6, [12, 9, 15, 10], [2, 0, 4, 2], dur_range=(1, 4))
        first = float(ts.step(batch).sum())
        for _ in range(7):
            last = float(ts.step(batch).sum())
        assert last < first, (spk_type, first, last)


def test_unsupported_conditioning_raises(cuda):
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    from oracle import fastspeech2 as ofs
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, num_tones=7, tone_embed_dim=32, device=cuda)
    with pytest.raises(NotImplementedError, match="tone"):
        FastSpeech2TrainStep(m)
    _, ts = _step("concat", _fs2ms.params("concat"), cuda)
    batch = _batch(6, [12, 9], [1, 2])
    with pytest.raises(NotImplementedError, match="spembs"):
        ts.step(dict(batch, spembs=torch.zeros(2, 256)))
    del batch["spk_id"]
    with pytest.raises(ValueError, match="spk_id"):
        ts.step(batch)
