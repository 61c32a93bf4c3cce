"""GPU parity of the TransformerTTS training step (TransformerTTSUpdater.update_core) and of its kernels against fp64 torch and
the oracle (oracle/transformer_tts_train.py: train_step_grads)."""
import math

import numpy as np
import pytest
import torch

from oracle import fastspeech2 as ofs
from oracle import transformer_tts_train as ot

pytestmark = pytest.mark.gpu

YAML_RATES = dict(transformer_enc_dropout_rate=0.1, transformer_enc_positional_dropout_rate=0.1, transformer_enc_attn_dropout_rate=0.1,
                  transformer_dec_dropout_rate=0.1, transformer_dec_positional_dropout_rate=0.1, transformer_dec_attn_dropout_rate=0.1,
                  transformer_enc_dec_attn_dropout_rate=0.1, postnet_dropout_rate=0.5)
RECIPE = dict(ot.LJSPEECH)


def _rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return (a - b).norm().item() / max(b.norm().item(), 1e-30)


# ------------------------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tq", [1, 63, 64, 65, 800])
def test_causal_masked_softmax_and_guided_softmax_bwd(cuda, tq):
    """pk_masked_softmax (causal self-attention, Tq = Tk) and pk_softmax_bwd (source attention, ragged ilens / olens,
    guided heads 0..1 of 3) against fp64 autograd of softmax -> <P, dP> + coef * sum G P."""
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(tq)
    B, H, Hg, layers, sigma, lam = 2, 3, 2, 2, 0.4, 10.0
    # causal softmax
    olens = torch.tensor([tq, max(1, tq - tq // 3)], dtype=torch.int32)
    ld = (tq + 63) // 64 * 64
    s = torch.randn(B * H, tq, ld, generator=g) * 2
    p = ops.masked_softmax(s.to(cuda), olens.to(cuda), B, H, tq, tq, causal=True).float().cpu()
    keep = ofs.make_non_pad_mask(olens, tq).unsqueeze(1) & torch.tril(torch.ones(tq, tq, dtype=torch.bool))
    keep = keep.repeat_interleave(H, 0)
    ref = torch.softmax(s[..., :tq].double().masked_fill(~keep, -1e300), -1).masked_fill(~keep, 0.0)
    # P comes back as split-bf16 planes (~2^-17 relative) from fp32 arithmetic
    assert (p[..., :tq].double() - ref).abs().max().item() < 2e-5 and (ld == tq or p[..., tq:].abs().max().item() == 0)
    # guided softmax backward: Tq query rows over Tk keys
    tk = max(2, tq // 4 + 3)
    ilens = torch.tensor([tk, max(1, tk - 2)], dtype=torch.int32)
    ldk = (tk + 63) // 64 * 64
    z = (torch.randn(B * H, tq, tk, generator=g) * 2).double().requires_grad_(True)
    km = ofs.make_non_pad_mask(ilens, tk).unsqueeze(1).repeat_interleave(H, 0)
    P = torch.softmax(z.masked_fill(~km, -1e300), -1).masked_fill(~km, 0.0)
    dp = torch.randn(B * H, tq, tk, generator=g).double()
    n = sum(int(ilens[b]) * int(olens[b]) for b in range(B))
    coef = lam / (Hg * layers * n)
    G = torch.zeros(B, H, tq, tk, dtype=torch.float64)
    for b in range(B):
        G[b, :Hg, :int(olens[b]), :int(ilens[b])] = ot.guided_mask(int(ilens[b]), int(olens[b]), sigma).double()
    G = G.reshape(B * H, tq, tk)
    scale = 1.0 / math.sqrt(64)
    ((P * dp).sum() + coef * (G * P).sum()).backward()
    Pp = torch.nn.functional.pad(P.detach().float(), (0, ldk - tk))
    dpp = torch.nn.functional.pad(dp.float(), (0, ldk - tk))
    partials = torch.full((B, Hg, tq), 7.0, device=cuda)
    guided = dict(heads=Hg, layers=layers, ilens=ilens.to(cuda), olens=olens.to(cuda), sigma=sigma, lam=lam, partials=partials)
    ds = ops.softmax_bwd(ops.Split.from_f32(Pp.to(cuda)), dpp.to(cuda), tk, scale, guided).float().cpu()
    assert _rel(ds[..., :tk], z.grad * scale) < 3e-5 and (ldk == tk or ds[..., tk:].abs().max().item() == 0)
    pref = (G * P.detach()).sum(-1).reshape(B, H, tq)[:, :Hg]
    assert _rel(partials, pref) < 1e-5
    losses = torch.zeros(5, device=cuda)
    ops.tts_guided_loss(partials, ilens.to(cuda), olens.to(cuda), tq, tk, Hg * layers, lam, losses)
    want = lam * pref.sum().item() / (Hg * layers * n)
    assert abs(losses[4].item() - want) <= 1e-5 * abs(want) and abs(losses[0].item() - want) <= 1e-5 * abs(want)


def test_tts_loss_and_gradients(cuda):
    """pk_tts_loss / pk_tts_loss_bwd against fp64 autograd of oracle.tts_loss, frames past olens masked out (with garbage)."""
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(3)
    B, L, odim = 3, 150, 80
    olens = torch.tensor([150, 97, 12], dtype=torch.int32)
    before, after, ys = (torch.randn(B, L, odim, generator=g).double().requires_grad_(i < 2) for i in range(3))
    logits = (torch.randn(B, L, generator=g) * 3).double().requires_grad_(True)
    labels = ofs.make_pad_mask(olens.long() - 1, L).double()
    labels[:, -1] = 1
    for lt in ("L1", "L2", "L1+L2"):
        for t in (before, after, logits):
            t.grad = None
        l1, l2, bce = ot.tts_loss(after, before, logits, ys, labels, olens.long(), 5.0)
        loss = {"L1": l1, "L2": l2, "L1+L2": l1 + l2}[lt] + bce
        loss.backward()
        args = [t.detach().float().contiguous().to(cuda) for t in (before, after, ys, logits, labels)] + [olens.to(cuda)]
        got = ops.tts_loss(*args, pos_weight=5.0, loss_type=lt).cpu()
        for i, v in enumerate((loss, l1, l2, bce)):
            assert abs(got[i].item() - v.item()) <= 1e-5 * abs(v.item()), (lt, i, got[i].item(), v.item())
        gb, ga, gl = ops.tts_loss_bwd(*args, pos_weight=5.0, loss_type=lt)
        assert _rel(gb, before.grad) < 1e-5 and _rel(ga, after.grad) < 1e-5 and _rel(gl, logits.grad) < 1e-5, lt


# ------------------------------------------------------------------------------------------------------------------
# the step
# ------------------------------------------------------------------------------------------------------------------
def _model(cfg, params, dev):
    from parakeet_b200.models import TransformerTTS
    m = TransformerTTS(cfg["idim"], cfg["odim"], device=dev, **{k: v for k, v in cfg.items() if k not in ("idim", "odim")})
    m.set_state_dict(params)
    return m


def _recipe_batch(seed, B=16):
    """A ragged batch of B utterances: 20..60 tokens, 60..300 frames, garbage in the padded frames."""
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(20, 61, (B,), generator=g)
    frames = torch.randint(60, 301, (B,), generator=g)
    lens[0], frames[0] = 60, 300
    return ot.golden_batch(RECIPE, seed, lens=tuple(lens.tolist()), frames=tuple(frames.tolist()))


def _on(batch, dev):
    text, tl, sp, sl = batch
    return dict(text=text.to(dev), text_lengths=tl.to(dev), speech=sp.to(dev), speech_lengths=sl.to(dev))


def _compare(ts, batch, cfg, params, lam, dropout, seed, step=1):
    text, tl, sp, sl = batch
    keep = ot.train_prenet_masks(seed, step, sp.shape[0], sp.shape[1], cfg["dprenet_units"], cfg["dprenet_layers"])
    drop = ofs.PhiloxDropout(seed, step) if dropout else None
    losses_ref, grads_ref, stats_ref = ot.train_step_grads(params, cfg, dict(text=text, text_lengths=tl, speech=sp, speech_lengths=sl),
                                                           keep, dropout=drop, rates=YAML_RATES if dropout else None, lam=lam)
    got = ts.forward_backward(_on(batch, ts.dev))
    for k, v in losses_ref.items():
        assert abs(float(got[k]) - v) <= 1e-4 * max(abs(v), 1.0), (k, float(got[k]), v)
    errs = sorted(((_rel(ts.grads[k], r), k) for k, r in grads_ref.items() if "linear_k.bias" not in k), reverse=True)
    print(f"worst gradient relative L2: {errs[0][0]:.2e} ({errs[0][1]})")
    assert errs[0][0] < 5e-3, errs[:6]
    for k in grads_ref:
        if "linear_k.bias" in k:     # the true gradient is zero (softmax shift invariance)
            assert ts.grads[k].abs().max().item() < 1e-4, k
    for k, v in stats_ref.items():
        assert _rel(ts.m._params[k], v) < 1e-4, k
    return grads_ref


@pytest.mark.parametrize("which", ["small", "recipe"])
def test_full_step_gradients_vs_oracle(cuda, which):
    """Dropout off (the prenet's always-on masks shared with the oracle): losses within 1e-4, every gradient within 5e-3 relative
    L2, the BatchNorm running statistics; at the golden's small config and at the recipe config on a ragged batch of 16."""
    from parakeet_b200.training import TransformerTTSTrainStep
    if which == "small":
        cfg, params = ot.TRAIN_SMALL, ot.synth_params(13, ot.TRAIN_SMALL)
        ref = np.load(__file__.replace("test_gpu_transformer_tts_training.py", "golden/ref_executed_transformer_tts_train.npz"))
        batch = tuple(torch.from_numpy(ref[f"batch/{k}"]) for k in ("text", "text_lengths", "speech", "speech_lengths"))
    else:
        cfg, params = RECIPE, ot.synth_params(21, RECIPE)
        batch = _recipe_batch(22)
    ts = TransformerTTSTrainStep(_model(cfg, params, cuda), guided_attn_loss_lambda=ot.TRAIN_LAMBDA, dropout=False, seed=ot.TRAIN_SEED)
    _compare(ts, batch, cfg, params, ot.TRAIN_LAMBDA, False, ot.TRAIN_SEED)
    if which == "small":           # and against the reference executed on the stand-in (the stored gradient elements)
        for k in [f[len("grad/"):] for f in ref.files if f.startswith("grad/") and "linear_k.bias" not in f]:
            gk = ts.grads[k].reshape(-1).cpu()
            got = gk[::max(1, gk.numel() // 1024)].double().numpy()
            want = ref[f"grad/{k}"].astype(np.float64)
            assert np.linalg.norm(got - want) <= 5e-3 * np.linalg.norm(want), k


def test_dropout_with_yaml_rates(cuda):
    """Every rate of the recipe yaml: the step's Philox masks restated in the oracle, losses and gradients agree."""
    from parakeet_b200.training import TransformerTTSTrainStep
    cfg, params = ot.TRAIN_SMALL, ot.synth_params(31, ot.TRAIN_SMALL)
    batch = ot.golden_batch(cfg, 32, lens=(9, 4, 6), frames=(40, 23, 31))
    ts = TransformerTTSTrainStep(_model(cfg, params, cuda), guided_attn_loss_lambda=10.0, dropout=YAML_RATES, seed=77)
    _compare(ts, batch, cfg, params, 10.0, True, 77)


def test_three_step_adam_trajectory(cuda):
    from parakeet_b200.training import TransformerTTSTrainStep
    cfg, params = ot.TRAIN_SMALL, ot.synth_params(41, ot.TRAIN_SMALL)
    batch = ot.golden_batch(cfg, 42, lens=(9, 4, 6), frames=(40, 23, 31))
    text, tl, sp, sl = batch
    lr = 2e-5
    ts = TransformerTTSTrainStep(_model(cfg, params, cuda), learning_rate=lr, guided_attn_loss_lambda=10.0, dropout=False, seed=3,
                                 use_graphs=True)
    p_ref, state, g1 = {k: v.double() for k, v in params.items()}, {}, None
    for s in range(1, 4):
        keep = ot.train_prenet_masks(3, s, sp.shape[0], sp.shape[1], cfg["dprenet_units"], cfg["dprenet_layers"])
        lref, gref, stats = ot.train_step_grads(p_ref, cfg, dict(text=text, text_lengths=tl, speech=sp, speech_lengths=sl), keep, lam=10.0)
        g1 = gref if g1 is None else g1
        p_new = ofs.adam_step({k: p_ref[k] for k in gref}, gref, state, lr=lr)
        p_ref = {**p_ref, **p_new, **stats}
        got = ts.step(_on(batch, cuda))
        assert abs(float(got["loss"]) - lref["loss"]) <= 1e-4 * abs(lref["loss"]), (s, float(got["loss"]), lref["loss"])
    # Adam's first steps move every weight by ~lr * sign(g): compare the elements whose first gradient is not lost in rounding
    # noise (|g| above 1e-3 of the tensor's largest; where the true gradient is ~0 the sign, and so the move, is arbitrary)
    worst = []
    for k, v in p_ref.items():
        if k not in g1 or "linear_k.bias" in k:
            continue
        mask = g1[k].abs() > 1e-3 * g1[k].abs().max()
        if mask.any():
            moved = (v - params[k].double()).abs().max().item()
            err = ((ts.m._params[k].double().cpu() - v).abs() * mask).max().item() / (moved + lr * 1e-2)
            worst.append((err, k))
    worst.sort(reverse=True)
    assert worst[0][0] < 1e-2, worst[:5]


def test_graph_replay_matches_eager(cuda):
    """Graphed steps (eager, capture, replays) equal eager steps to reduction-order noise, with dropout on (fresh masks every
    replay: the losses change from step to step), also after a larger batch shape and an evaluate() in between."""
    from parakeet_b200.training import TransformerTTSTrainStep
    cfg, params = ot.TRAIN_SMALL, ot.synth_params(51, ot.TRAIN_SMALL)
    small = _on(ot.golden_batch(cfg, 52, lens=(9, 4, 6), frames=(40, 23, 31)), cuda)
    large = _on(ot.golden_batch(cfg, 53, lens=(12, 5, 8, 11), frames=(60, 33, 41, 50)), cuda)
    runs = []
    for graphs in (True, False):
        ts = TransformerTTSTrainStep(_model(cfg, params, cuda), learning_rate=1e-4, guided_attn_loss_lambda=10.0, dropout=YAML_RATES,
                                     seed=9, use_graphs=graphs)
        losses = [float(ts.step(small)["loss"]) for _ in range(3)]
        losses.append(float(ts.step(large)["loss"]))
        ev = ts.evaluate(small)
        losses += [float(ts.step(small)["loss"]) for _ in range(2)]
        runs.append((losses, ts.flat.clone(), float(ev["loss"])))
    (la, fa, ea), (lb, fb, eb) = runs
    assert len(set(round(v, 6) for v in la[:3])) == 3, la          # fresh masks on every replay
    assert np.allclose(la, lb, rtol=1e-4), (la, lb)
    assert abs(ea - eb) <= 1e-4 * abs(eb)
    assert _rel(fa, fb) < 1e-4                              # parameters after 6 Adam steps of lr 1e-4


def test_checkpoint_resume_continues_trajectory(cuda, tmp_path):
    from parakeet_b200.training import TransformerTTSTrainStep
    cfg, params = ot.TRAIN_SMALL, ot.synth_params(61, ot.TRAIN_SMALL)
    batch = _on(ot.golden_batch(cfg, 62, lens=(9, 4, 6), frames=(40, 23, 31)), cuda)
    mk = lambda: TransformerTTSTrainStep(_model(cfg, params, cuda), learning_rate=1e-4, dropout=YAML_RATES, seed=5)  # noqa: E731
    a = mk()
    for _ in range(2):
        a.step(batch)
    a.save(str(tmp_path / "snap.pdz"))
    la = float(a.step(batch)["loss"])
    b = mk()
    b.load(str(tmp_path / "snap.pdz"))
    lb = float(b.step(batch)["loss"])
    assert abs(la - lb) <= 1e-5 * abs(la) and _rel(b.flat, a.flat) < 1e-6


def test_inference_after_step_uses_updated_weights(cuda):
    from parakeet_b200.training import TransformerTTSTrainStep
    cfg, params = ot.TRAIN_SMALL, ot.synth_params(71, ot.TRAIN_SMALL)
    text, tl, sp, sl = ot.golden_batch(cfg, 72, lens=(9, 4, 6), frames=(40, 23, 31))
    m = _model(cfg, params, cuda)
    before = m.forward(text.to(cuda), tl.to(cuda), sp.to(cuda), sl.to(cuda), seed=1)[0].clone()
    ts = TransformerTTSTrainStep(m, learning_rate=1e-3, dropout=False)
    ts.step(_on((text, tl, sp, sl), cuda))
    after = m.forward(text.to(cuda), tl.to(cuda), sp.to(cuda), sl.to(cuda), seed=1)[0]
    fresh = _model(cfg, {k: v.cpu() for k, v in m.state_dict().items()}, cuda)
    want = fresh.forward(text.to(cuda), tl.to(cuda), sp.to(cuda), sl.to(cuda), seed=1)[0]
    assert _rel(after, before) > 1e-4 and _rel(after, want) < 1e-6
