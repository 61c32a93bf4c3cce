"""GPU parity of the FastSpeech2 training step (forward in train mode, loss, backward, Adam) against torch autograd on the
oracle (FastSpeech2Updater.update_core, fastspeech2_updater.py:51-99)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _close(a, ref, rtol=2e-3, atol=2e-6):
    a, ref = a.detach().double().cpu(), ref.detach().double().cpu()
    return (a - ref).abs().max().item() <= rtol * ref.abs().max().item() + atol


def test_fs2_train_kernels_unit(cuda):
    """Row-wise backward kernels against torch autograd."""
    from parakeet_b200 import _lib, ops
    from parakeet_b200.ops import _ptr, _stream
    L = _lib.lib()
    g = torch.Generator().manual_seed(0)
    # LayerNorm backward
    x = torch.randn(37, 384, generator=g, requires_grad=True)
    gam, bet = torch.randn(384, generator=g, requires_grad=True), torch.randn(384, generator=g, requires_grad=True)
    dy = torch.randn(37, 384, generator=g)
    torch.nn.functional.layer_norm(x, (384,), gam, bet).backward(dy)
    dx = torch.zeros(37, 384, device=cuda)
    dg, db = torch.zeros(384, device=cuda), torch.zeros(384, device=cuda)
    xg, gg, dyg = x.detach().to(cuda), gam.detach().to(cuda), dy.to(cuda)
    ops.layer_norm_bwd(xg, gg, dyg, dx, False, dg, db)
    assert _close(dx, x.grad) and _close(dg, gam.grad) and _close(db, bet.grad)
    # softmax backward (with zero-probability padding columns)
    s = torch.randn(6, 20, 64, generator=g)
    s[:, :, 17:] = -1e30
    s.requires_grad_(True)
    p = torch.softmax(s, -1)
    dp = torch.randn(6, 20, 64, generator=g)
    (p * 0.3).backward(dp)        # scale 0.3 plays the role of 1/sqrt(dk)
    pg, dpg = ops.Split.from_f32(p.detach().to(cuda)), dp.to(cuda)
    ds = ops.softmax_bwd(pg, dpg, 17, 0.3).float()
    assert _close(ds[:, :, :17], s.grad[:, :, :17]) and ds[:, :, 17:].abs().max().item() == 0
    # transpose with shift
    a = torch.randn(3, 10, 16, generator=g)
    src = ops.Split.from_f32(a.to(cuda))
    dst = ops.Split.zeros((5, 3 * 64), cuda)
    ops.transpose_planes(src, z=3, rows=10, src_zstride=160, ld_src=16, c0=4, cols=5, shift=-1, r_out=10, dst=dst, dst_zstride=64, ld_dst=192)
    ref = torch.zeros(5, 3, 64)
    ref[:, :, 1:10] = a[:, :9, 4:9].permute(2, 0, 1)
    assert torch.allclose(dst.float().cpu().reshape(5, 3, 64), ref, atol=1e-4)
    # BatchNorm train forward / backward (+ tanh)
    xb = torch.randn(50, 24, generator=g, requires_grad=True)
    gb, bb = torch.randn(24, generator=g, requires_grad=True), torch.randn(24, generator=g, requires_grad=True)
    mean, var = xb.mean(0), xb.var(0, unbiased=False)
    yb = torch.tanh((xb - mean) / torch.sqrt(var + 1e-5) * gb + bb)
    dyb = torch.randn(50, 24, generator=g)
    yb.backward(dyb)
    rm, rv = torch.zeros(24, device=cuda), torch.ones(24, device=cuda)
    sums = torch.zeros(64, device=cuda)
    y = torch.empty(50, 24, device=cuda)
    sm, sr = torch.empty(24, device=cuda), torch.empty(24, device=cuda)
    xc, gc, bc, dyc = xb.detach().to(cuda), gb.detach().to(cuda), bb.detach().to(cuda), dyb.to(cuda)   # locals: must outlive the launches
    _lib.check(L.pk_batch_norm_train(_ptr(xc), 50, 24, _ptr(gc), _ptr(bc), 1e-5, 2, 0.9, _ptr(rm), _ptr(rv),
                                     _ptr(sums), _ptr(y), None, None, _ptr(sm), _ptr(sr), _stream()), "bn")
    assert _close(y, yb) and _close(rm, 0.1 * mean) and _close(rv, 0.9 + 0.1 * var)
    dxb = torch.empty(50, 24, device=cuda)
    _lib.check(L.pk_batch_norm_bwd(_ptr(xc), _ptr(dyc), _ptr(y), _ptr(sm), _ptr(sr), _ptr(gc), 2, 50, 24, _ptr(sums),
                                   _ptr(dxb), _stream()), "bn_bwd")
    assert _close(dxb, xb.grad) and _close(sums[:24], bb.grad) and _close(sums[24:48], gb.grad)
    # length regulator backward
    d = torch.tensor([[2, 0, 3], [1, 1, 1]])
    dyl = torch.randn(2, 5, 8, generator=g)
    dxl = torch.empty(2, 3, 8, device=cuda)
    dylc, dc = dyl.to(cuda), d.to(cuda)
    _lib.check(L.pk_length_regulate_bwd(_ptr(dylc), _ptr(dc), 2, 3, 8, 5, _ptr(dxl), _stream()), "lr_bwd")
    ref = torch.stack([torch.stack([dyl[0, 0:2].sum(0), torch.zeros(8), dyl[0, 2:5].sum(0)]), torch.stack([dyl[1, 0], dyl[1, 1], dyl[1, 2]])])
    assert _close(dxl, ref)
    # Adam, paddle semantics
    from oracle import fastspeech2 as ofs
    p0, g0 = torch.randn(1000, generator=g), torch.randn(1000, generator=g)
    st = {}
    ref1 = ofs.adam_step({"w": p0}, {"w": g0}, st, lr=1e-3)["w"]
    ref2 = ofs.adam_step({"w": ref1}, {"w": g0 * 0.5}, st, lr=1e-3)["w"]
    pc, mc, vc = p0.clone().to(cuda), torch.zeros(1000, device=cuda), torch.zeros(1000, device=cuda)
    g0c, g1c = g0.to(cuda), (g0 * 0.5).to(cuda)
    _lib.check(L.pk_adam(_ptr(pc), _ptr(g0c), _ptr(mc), _ptr(vc), 1000, 1e-3, 0.9, 0.999, 1e-8, 1, 1.0, None, 0.0, _stream()), "adam")
    assert torch.allclose(pc.cpu(), ref1, atol=1e-7)
    _lib.check(L.pk_adam(_ptr(pc), _ptr(g1c), _ptr(mc), _ptr(vc), 1000, 1e-3, 0.9, 0.999, 1e-8, 2, 1.0, None, 0.0, _stream()), "adam")
    assert torch.allclose(pc.cpu(), ref2, atol=1e-7)


def test_fs2_training_step_gradients_and_adam_update(cuda):
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    params = ofs.synth_params(1)
    batch = ofs.synth_train_batch(5, [9, 14, 11], dur_range=(1, 4))
    losses_ref, grads_ref, stats_ref = ofs.train_step_grads(params, None, batch, stop_gradient_from_pitch_predictor=True)
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=cuda)
    m.set_state_dict(params)
    ts = FastSpeech2TrainStep(m, learning_rate=1e-3, dropout=False)
    losses = ts.forward_backward(batch)
    got = [float(v) for v in losses]
    ref = [losses_ref[k] for k in ("l1_loss", "duration_loss", "pitch_loss", "energy_loss")]
    assert np.allclose(got, ref, rtol=1e-3), (got, ref)
    # Gradients of all 198 trainable tensors.  ReLU is not differentiable at 0: a pre-activation within ~1e-5 of zero can
    # get a different mask on the GPU (whose forward differs from the oracle by ~1e-5) and that single element changes the
    # gradients of its layer's weights by a percent or two on a 34-token batch (the oracle shows exactly which layers have
    # such elements: scripts/gpu_check_train.py).  So: every tensor within 5e-2 in relative L2, and >= 85 % of them within
    # the strict 2e-3 max-norm bound.
    strict, loose_bad = 0, []
    for k, gref in grads_ref.items():
        g = ts.grads[k].detach().double().cpu()
        r = gref.double()
        strict += _close(g, r)
        if (g - r).norm().item() > 5e-2 * r.norm().item() + 1e-5:
            loose_bad.append((k, (g - r).norm().item(), r.norm().item()))
    assert not loose_bad, loose_bad[:8]
    assert strict >= 0.85 * len(grads_ref), (strict, len(grads_ref))
    for k, v in stats_ref.items():                       # BatchNorm running statistics (momentum 0.9)
        assert _close(m.state_dict()[k], v), k
    # one optimiser step (paddle Adam) moves every parameter like the oracle
    ts2_ref = ofs.adam_step({k: params[k] for k in grads_ref}, grads_ref, {}, lr=1e-3)
    ts.gflat  # gradients are in place from forward_backward
    from parakeet_b200 import _lib
    from parakeet_b200.ops import _ptr, _stream
    _lib.check(_lib.lib().pk_adam(_ptr(ts.flat), _ptr(ts.gflat), _ptr(ts.adam_m), _ptr(ts.adam_v), ts.flat.numel(), 1e-3, 0.9, 0.999, 1e-8, 1,
                                  1.0, None, 0.0, _stream()), "pk_adam")
    # Adam's first step moves every weight by ~lr * sign(g): compare where the gradient is not numerically zero (|g| > 1e-5;
    # elements whose true gradient is ~0, e.g. the key biases of the attention, take an arbitrary sign) and not kink-affected
    worst = 0.0
    for k, v in ts2_ref.items():
        mask = (grads_ref[k].abs() > 1e-5) & ((ts.grads[k].cpu() - grads_ref[k]).abs() < 0.1 * grads_ref[k].abs())
        if mask.any():
            worst = max(worst, ((m.state_dict()[k].cpu() - v).abs() * mask).max().item())
    assert worst < 1e-4, worst


def test_fs2_training_reduces_loss(cuda):
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=cuda)
    m.set_state_dict(ofs.synth_params(1))
    batch = ofs.synth_train_batch(6, [12, 9, 15, 10], dur_range=(1, 4))
    ts = FastSpeech2TrainStep(m, learning_rate=1e-3, dropout=False)
    first = float(ts.step(batch).sum())
    for _ in range(7):
        last = float(ts.step(batch).sum())
    assert last < first, (first, last)


def _cfg5_lengths(n=8, seed=50):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(60, 141, (n,), generator=g).tolist()          # cfg 5: 8 utterances per GPU, T ~ U{60..140}


def test_fs2_training_step_cfg5_shape_vs_oracle(cuda):
    """BASELINE cfg 5 per-GPU shape (8 utterances of 60..140 phonemes, durations U{2..12} -> ~5 600 mel frames): losses,
    every gradient tensor and the BatchNorm statistics against torch autograd on the oracle.  On a batch this size a single
    ReLU kink no longer moves a weight gradient by percents: every tensor within 5e-3 in relative L2 (the
    worst are gradients such as encoder.embed.1.alpha and pitch_embed.0.weight - sums over all ~700 tokens of fp32-rounded
    terms behind 14 FFT blocks), at least 90 % of the tensors inside the 1e-3 forward contract."""
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    params = ofs.synth_params(1)
    batch = ofs.synth_train_batch(51, _cfg5_lengths())
    assert batch["speech"].shape[0] == 8 and batch["speech"].shape[1] > 500
    losses_ref, grads_ref, stats_ref = ofs.train_step_grads(params, None, batch, stop_gradient_from_pitch_predictor=True)
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=cuda)
    m.set_state_dict(params)
    ts = FastSpeech2TrainStep(m, learning_rate=1e-3, dropout=False)
    got = [float(v) for v in ts.forward_backward(batch)]
    ref = [losses_ref[k] for k in ("l1_loss", "duration_loss", "pitch_loss", "energy_loss")]
    assert np.allclose(got, ref, rtol=1e-3), (got, ref)
    bad = []
    for k, gref in grads_ref.items():
        g, r = ts.grads[k].detach().double().cpu(), gref.double()
        e = (g - r).norm().item() / max(r.norm().item(), 1e-12)
        if (g - r).norm().item() > 1e-7:
            bad.append((k, e))
    worst = sorted(bad, key=lambda t: -t[1])
    assert not worst or worst[0][1] < 5e-3, worst[:8]
    assert sum(e > 1e-3 for _, e in worst) <= 0.1 * len(grads_ref), worst[:24]
    for k, v in stats_ref.items():
        assert _close(m.state_dict()[k], v), k


def test_fs2_three_steps_follow_the_oracle_adam_trajectory(cuda):
    """Three consecutive FastSpeech2TrainStep.step() calls (forward, backward, paddle-Adam) against three oracle steps
    (train_step_grads + adam_step) on the same batch: the PARAMETERS after step 3 within 1e-3 (relative to the largest
    parameter change of that tensor, plus the fp32 noise floor lr * 1e-2 of Adam's sign-like first steps)."""
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    params = ofs.synth_params(1)
    batch = ofs.synth_train_batch(52, _cfg5_lengths(4, seed=53))
    lr = 2e-5        # Adam moves every weight by ~lr per step whatever the gradient scale: 1e-3 on this randomly initialised model
                     # is a chaotic regime (loss 7 -> 135 -> 61) in which rounding noise is amplified, not a parity test
    p_ref, state, loss_ref = dict(params), {}, []
    for _ in range(3):
        losses, grads, stats = ofs.train_step_grads(p_ref, None, batch, stop_gradient_from_pitch_predictor=True)
        loss_ref.append(losses["loss"])
        new = ofs.adam_step({k: p_ref[k] for k in grads}, grads, state, lr=lr)
        p_ref = {**p_ref, **new, **stats}
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=cuda)
    m.set_state_dict(params)
    ts = FastSpeech2TrainStep(m, learning_rate=lr, dropout=False)
    loss_got = [float(ts.step(batch).sum()) for _ in range(3)]
    assert np.allclose(loss_got, loss_ref, rtol=2e-3), (loss_got, loss_ref)
    sd = m.state_dict()
    bad = []
    for k, v in p_ref.items():
        got, ref, init = sd[k].detach().double().cpu(), v.double(), params[k].double()
        moved = (ref - init).abs().max().item()
        # elements whose gradient is numerically zero take an arbitrary sign in Adam's first steps (m / sqrt(v) of noise):
        # compare in relative L2 over the tensor, where those few elements do not dominate
        e = (got - ref).norm().item() / max((ref - init).norm().item(), 1e-12)
        if moved < lr:
            # tensors whose true gradient is (numerically) zero - the key biases of every attention (softmax is invariant to
            # them), a few dead channels: Adam divides rounding noise by its own magnitude, the direction is arbitrary in BOTH
            # implementations; only the size of the step is meaningful (<= lr per step)
            assert (got - init).abs().max().item() <= 3.5 * lr, k
            continue
        bad.append((k, e, moved))
    # Adam turns a gradient into a step of ~lr * g / |g|: elements whose gradient is small against the fp32 / split-bf16
    # rounding noise of a 5 600-frame reduction move in a slightly different direction (scripts/gpu_calib_traj.py prints
    # the per-tensor distances): most tensors stay within 5e-2 of the oracle's parameter DELTA in relative L2.
    worst = sorted(bad, key=lambda t: -t[1])
    assert worst[0][1] < 0.2, worst[:8]
    assert sum(e > 5e-2 for _, e, _ in worst) <= 0.08 * len(worst), worst[:24]
    # and the loss went down along the way
    assert loss_got[2] < loss_got[0]


def test_dropout_kernel_matches_the_numpy_philox_restatement_and_its_statistics(cuda):
    """pk_dropout against oracle.PhiloxDropout (numpy Philox4x32-10, itself pinned to the Random123 known answers in
    tests/test_oracle_cpu.py): identical masks, upscale_in_train scaling, split-plane input / output, and keep-rate statistics."""
    from oracle import fastspeech2 as ofs
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(7)
    x = torch.randn(3, 37, 101, generator=g)                             # 11 211 elements: not a multiple of 4
    for p, site, step, seed in ((0.2, 1021, 3, 12345), (0.5, 5046, 1, (1 << 40) + 17), (0.1, 0, 7, 0)):
        ref = ofs.PhiloxDropout(seed, step)(site, x, p)
        y, ys = ops.dropout(x.to(cuda), p, seed, site, step, out_f32=True, out_split=True)
        assert torch.equal((y == 0).cpu(), ref == 0)
        assert torch.allclose(y.cpu(), ref, rtol=1e-6, atol=0)
        assert torch.allclose(ys.float().cpu(), ref, rtol=2e-5, atol=1e-6)
        y2, _ = ops.dropout(ops.Split.from_f32(x.to(cuda)), p, seed, site, step)          # split input
        assert torch.allclose(y2.cpu(), ref, rtol=2e-5, atol=1e-6)
    big = torch.ones(1 << 22, device=cuda)
    for p in (0.1, 0.2, 0.5):
        y, _ = ops.dropout(big, p, 99, 4, 1)
        keep = float((y != 0).float().mean())
        assert abs(keep - (1 - p)) < 4 * (p * (1 - p) / big.numel()) ** 0.5 + 1e-4, (p, keep)    # 4 sigma
        assert abs(float(y.mean()) - 1.0) < 5e-3                                                  # upscale_in_train keeps the mean
    a, _ = ops.dropout(big, 0.5, 99, 4, 1)
    b, _ = ops.dropout(big, 0.5, 99, 5, 1)                                # another site: an independent mask
    c, _ = ops.dropout(big, 0.5, 99, 4, 2)                                # another step: an independent mask
    assert 0.45 < float(((a != 0) == (b != 0)).float().mean()) < 0.55 and 0.45 < float(((a != 0) == (c != 0)).float().mean()) < 0.55


def test_fs2_training_step_with_the_shipped_dropout_rates_vs_oracle(cuda):
    """The reference's recipe (conf/default.yaml:56-74: 0.2 on the six transformer rates, 0.5 in the pitch / energy predictors
    and the postnet, 0.1 in the duration predictor): forward losses, gradients and BatchNorm statistics of one step against the
    oracle applying the SAME Philox masks at the reference's dropout sites, and the masks change from step to step."""
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    params = ofs.synth_params(1)
    batch = ofs.synth_train_batch(61, _cfg5_lengths(4, seed=62))
    rates = dict(ofs.YAML_DROPOUT, pitch_embed_dropout=0.3)             # + one of the embedding dropouts the yaml leaves at 0
    seed = 2024
    losses_ref, grads_ref, stats_ref = ofs.train_step_grads(params, None, batch, stop_gradient_from_pitch_predictor=True,
                                                             dropout=ofs.PhiloxDropout(seed, 1), rates=rates)
    losses_nodrop, _, _ = ofs.train_step_grads(params, None, batch, stop_gradient_from_pitch_predictor=True)
    assert abs(losses_ref["loss"] - losses_nodrop["loss"]) > 1e-2                      # the masks do something
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=cuda, **rates)
    m.set_state_dict(params)
    ts = FastSpeech2TrainStep(m, learning_rate=1e-3, dropout=True, seed=seed)
    got = [float(v) for v in ts.forward_backward(batch)]
    ref = [losses_ref[k] for k in ("l1_loss", "duration_loss", "pitch_loss", "energy_loss")]
    assert np.allclose(got, ref, rtol=1e-3), (got, ref)
    errs = []
    for k, gref in grads_ref.items():
        g, r = ts.grads[k].detach().double().cpu(), gref.double()
        if k.endswith("self_attn.linear_k.bias"):        # true gradient 0 (softmax ignores a per-row shift): rounding noise in both
            assert g.abs().max().item() < 1e-4 and r.abs().max().item() < 1e-4, k
            continue
        if (g - r).norm().item() > 1e-7:
            errs.append((k, (g - r).norm().item() / max(r.norm().item(), 1e-12)))
    errs.sort(key=lambda t: -t[1])
    assert not errs or errs[0][1] < 2e-2, errs[:8]
    assert sum(e > 5e-3 for _, e in errs) <= 0.1 * len(grads_ref), errs[:24]
    for k, v in stats_ref.items():
        assert _close(m.state_dict()[k], v), k
    first = float(ts.step(batch).sum())                                    # step 1 (same masks as above), then step 2: new masks
    second_fb = [float(v) for v in ts.forward_backward(batch)]
    assert np.allclose(first, sum(ref), rtol=1e-3) and abs(sum(second_fb) - first) > 1e-3


def test_fs2_training_graph_replay_matches_eager(cuda):
    """forward + backward replayed as a CUDA graph (third step on) against the eager step, with dropout on: the device-side
    step counter must give every replay fresh masks (same as eager), losses and parameters agree to reduction-order noise."""
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    from parakeet_b200.training import FastSpeech2TrainStep
    params = ofs.synth_params(1)
    batch = ofs.synth_train_batch(71, [20, 33, 27])
    rates = dict(ofs.YAML_DROPOUT)
    runs = []
    for graphs in (False, True):
        m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, stop_gradient_from_pitch_predictor=True, device=cuda, **rates)
        m.set_state_dict(params)
        ts = FastSpeech2TrainStep(m, learning_rate=2e-5, dropout=True, seed=5, use_graphs=graphs)
        losses = [float(ts.step(batch).sum()) for _ in range(5)]
        runs.append((losses, {k: v.detach().double().cpu().clone() for k, v in m.state_dict().items()}, ts))
    assert runs[1][2]._fb_graphs.replays >= 3 and runs[0][2]._fb_graphs.replays == 0
    assert np.allclose(runs[0][0], runs[1][0], rtol=2e-4), (runs[0][0], runs[1][0])
    assert len(set(round(v, 4) for v in runs[1][0])) == 5                  # five different mask sets -> five different losses
    for k, v in runs[0][1].items():
        init = params[k].double()
        if (v - init).abs().max().item() < 2e-5 or k.endswith("self_attn.linear_k.bias"):
            continue                                                        # zero-gradient tensors (see the trajectory test)
        d = (runs[1][1][k] - v).norm().item() / max((v - init).norm().item(), 1e-12)
        assert d < 5e-2, (k, d)
