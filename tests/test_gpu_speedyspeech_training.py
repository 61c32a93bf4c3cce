"""H100 tests of the SpeedySpeech training step: the new kernels alone against fp64 torch, then SpeedySpeechTrainStep against the
oracle restatement of SpeedySpeechUpdater.update_core (oracle/speedyspeech_train.py, fp64 autograd)."""
import pytest
import torch

from oracle import speedyspeech_train as sst
from oracle import speedyspeech as oss
from parakeet_b200 import _lib, ops
from parakeet_b200.models import SpeedySpeech
from parakeet_b200.training import SpeedySpeechTrainStep

pytestmark = pytest.mark.gpu


def rel_l2(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def to_dev(batch, dev):
    return {k: v.to(dev) for k, v in batch.items()}


def make(cfg, p, dev, tone_size=None, **kw):
    m = SpeedySpeech(vocab_size=40, tone_size=tone_size, device=dev, **cfg)
    m.set_state_dict(p)
    return m, SpeedySpeechTrainStep(m, **kw)


# --------------------------------------------------------------------------------------------------------------------
# kernels alone
# --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,residual", [(1000, False), (333, True), (128, True), (7, False)])
def test_bn_train_fwd_against_fp64(cuda, rows, residual):
    g = torch.Generator().manual_seed(rows)
    r = torch.relu(torch.randn(rows, 128, generator=g) + 0.3)
    gamma, beta = 0.5 + torch.rand(128, generator=g), torch.randn(128, generator=g) * 0.2
    rm, rv = torch.rand(128, generator=g), 0.5 + torch.rand(128, generator=g)
    res = torch.randn(rows, 128, generator=g) if residual else None
    rm_d, rv_d = rm.to(cuda), rv.to(cuda)
    sc = torch.empty(ops.ss_scratch_elems(rows), device=cuda)
    y, ys, mean, rstd = ops.ss_bn_train_fwd(r.to(cuda), gamma.to(cuda), beta.to(cuda), rm_d, rv_d, sc, residual=res.to(cuda) if residual else None)
    rd = r.double()
    mu, var = rd.mean(0), rd.var(0, unbiased=False)
    ref = (rd - mu) / torch.sqrt(var + 1e-5) * gamma.double() + beta.double() + (res.double() if residual else 0)
    assert rel_l2(y, ref) < 1e-6 and rel_l2(ys.float(), ref) < 1e-5
    assert rel_l2(mean, mu) < 1e-6 and rel_l2(rstd, 1 / torch.sqrt(var + 1e-5)) < 1e-6
    assert rel_l2(rm_d, 0.9 * rm.double() + 0.1 * mu) < 1e-6 and rel_l2(rv_d, 0.9 * rv.double() + 0.1 * var) < 1e-6


@pytest.mark.parametrize("rows", [1000, 333, 5])
def test_bn_relu_bwd_against_fp64_autograd(cuda, rows):
    g = torch.Generator().manual_seed(rows + 1)
    pre = (torch.randn(rows, 128, generator=g) + 0.2).double().requires_grad_(True)
    gamma = (0.5 + torch.rand(128, generator=g)).double().requires_grad_(True)
    beta = torch.zeros(128, dtype=torch.float64, requires_grad=True)
    dy = torch.randn(rows, 128, generator=g)
    r = torch.relu(pre)
    mu, var = r.mean(0), r.var(0, unbiased=False)
    ((r - mu) / torch.sqrt(var + 1e-5) * gamma + beta).backward(dy.double())
    sc = torch.empty(ops.ss_scratch_elems(rows), device=cuda)
    dgamma, dbeta, dbias = (torch.empty(128, device=cuda) for _ in range(3))
    dr, drs = ops.ss_bn_relu_bwd(dy.to(cuda), r.detach().float().to(cuda), mu.detach().float().to(cuda),
                                 (1 / torch.sqrt(var + 1e-5)).detach().float().to(cuda), gamma.detach().float().to(cuda), sc, dgamma, dbeta,
                                 dbias=dbias, want_f32=True)
    assert rel_l2(dr, pre.grad) < 1e-5 and rel_l2(drs.float(), pre.grad) < 1e-5
    assert rel_l2(dgamma, gamma.grad) < 1e-5 and rel_l2(dbeta, beta.grad) < 1e-5 and rel_l2(dbias, pre.grad.sum(0)) < 1e-4
    dr2, _ = ops.ss_bn_relu_bwd(dy.to(cuda), r.detach().float().to(cuda), mu.detach().float().to(cuda),
                                (1 / torch.sqrt(var + 1e-5)).detach().float().to(cuda), gamma.detach().float().to(cuda), sc, dgamma, dbeta,
                                dbias=dbias, want_f32=True)
    assert torch.equal(dr, dr2)                      # fixed summation order: identical bits


@pytest.mark.parametrize("lens,frames", [([9, 4], None), ([12, 12, 3], [40, 17, 0]), ([5], None)])
def test_loss_kernel_against_fp64_autograd(cuda, lens, frames):
    """Fully masked utterance tails, an utterance with no frames at all, a frame count that is not a multiple of the tile."""
    batch = sst.synth_batch(3, lens)
    g = torch.Generator().manual_seed(5)
    if frames is not None:
        batch["num_frames"] = torch.tensor(frames)
    B, L = batch["feats"].shape[:2]
    decoded = torch.randn(B, L, 80, generator=g)
    pred = torch.randn(B, max(lens), generator=g) * 2 + 1      # |r| on both sides of delta
    dd, pp = decoded.double().requires_grad_(True), pred.double().requires_grad_(True)
    ref = sst.losses(dd, pp, batch)
    ref["loss"].backward()
    sc = torch.empty(ops.ss_scratch_elems(0, B, L, 80), device=cuda)
    out, g_dec, g_dur = ops.ss_loss(decoded.to(cuda), batch["feats"].to(cuda), batch["num_frames"].to(cuda, torch.int32), pred.to(cuda),
                                    batch["durations"].to(cuda), batch["num_phones"].to(cuda, torch.int32), sc)
    for i, k in enumerate(("loss", "l1_loss", "duration_loss", "ssim_loss")):
        v = float(ref[k].detach())
        assert abs(out[i].item() - v) < 1e-5 * max(1.0, abs(v)), k
    assert rel_l2(g_dec, dd.grad) < 1e-4 and rel_l2(g_dur, pp.grad) < 1e-5
    only, none1, none2 = ops.ss_loss(decoded.to(cuda), batch["feats"].to(cuda), batch["num_frames"].to(cuda, torch.int32), pred.to(cuda),
                                     batch["durations"].to(cuda), batch["num_phones"].to(cuda, torch.int32), sc, want_grads=False)
    assert torch.equal(only, out) and none1 is None and none2 is None


# --------------------------------------------------------------------------------------------------------------------
# the step against the oracle
# --------------------------------------------------------------------------------------------------------------------
def relu_mask_flips(step, batch, p, cfg, dev):
    """forward_backward with every ReLU output the GPU fed to a BatchNorm compared with the oracle's pre-activation at the same
    place -> (losses, number of elements whose ReLU mask differs, number of elements compared)."""
    pre, rs = [], []
    real_relu, real_bn = torch.relu, ops.ss_bn_train_fwd
    sst.torch.relu = lambda x: (pre.append(x.detach()), real_relu(x))[1]
    try:
        sst.forward_train({k: v.double() for k, v in p.items()}, cfg, batch["phones"], batch.get("tones"), batch["durations"], {})
    finally:
        sst.torch.relu = real_relu
    ops.ss_bn_train_fwd = lambda r, *a, **k: (rs.append(r), real_bn(r, *a, **k))[1]
    try:
        out = step.forward_backward(to_dev(batch, dev))
    finally:
        ops.ss_bn_train_fwd = real_bn
    assert len(pre) == len(rs) + 1                       # the oracle's first ReLU is the prenet's, which no BatchNorm follows
    flips = sum(int(((a.reshape(r.shape) > 0) != (r.cpu() > 0)).sum()) for a, r in zip(pre[1:], rs))
    return out, flips, sum(r.numel() for r in rs)


def check_forward_backward(cuda, cfg, lens, tone_size, seed):
    """ReLU is not differentiable at 0: the GPU forward differs from the fp64 oracle by ~1e-5 (split-bf16 GEMMs), so a
    pre-activation that close to zero can get the other mask, and behind a train-mode BatchNorm that one element moves the
    gradients of its layer and of everything upstream by a percent or two.  The flips are COUNTED here, by comparing masks with the
    oracle: with none, every tensor must be within 5e-3 in relative L2; with some (at most 1e-4 of the elements), the
    duration predictor's tensors, which the flipped decoder / encoder elements cannot reach, still must, and 5e-2 caps the rest."""
    p = oss.synth_params(seed, cfg, tone_size=tone_size)
    batch = sst.synth_batch(seed + 1, lens, tone_size=tone_size)
    ref_losses, ref_grads, ref_stats = sst.train_step_grads(p, cfg, batch)
    m, step = make(cfg, p, cuda, tone_size)
    out, flips, compared = relu_mask_flips(step, batch, p, cfg, cuda)
    for k, v in ref_losses.items():
        assert abs(out[k].item() - v) < 1e-4 * abs(v), (k, out[k].item(), v)
    errs = sorted(((rel_l2(step.grads[k], g), k, float(g.norm())) for k, g in ref_grads.items()), reverse=True)
    loose = [e for e in errs if e[0] >= 5e-3]
    print(f"{flips} ReLU mask flips of {compared}; {len(loose)} of {len(errs)} gradient tensors beyond 5e-3, worst {errs[0][:2]}")
    assert flips <= 1e-4 * compared, (flips, compared)
    if flips == 0:
        assert not loose, loose[:8]
    assert errs[0][0] < 5e-2, errs[:8]
    assert not [e for e in loose if e[1].startswith("duration_predictor.")], loose[:8]
    for k, v in ref_stats.items():
        assert rel_l2(m.state_dict()[k], v) < 1e-4, k
    assert step.grads["encoder.embedding.text_embedding.weight"][0].abs().max().item() == 0.0     # padding_idx row
    return step


@pytest.mark.parametrize("k,n,pre", [(4, 1, "duration_predictor.layers.0."), (3, 1, "duration_predictor.layers.1."),
                                     (1, 1, "duration_predictor.layers.2."), (3, 2, "decoder.postnet2.0.")])
def test_residual_block_forward_and_backward_alone_against_fp64(cuda, k, n, pre):
    """One train-mode ResidualBlock (conv GEMM + the new BatchNorm kernels + data and weight gradients) for 1, 3 and 4 taps - the
    even kernel pads one more row on the right -, one and two units, 3 x 37 rows (not a multiple of any tile)."""
    cfg = oss.SMALL_CFG
    p = oss.synth_params(11, cfg)
    m, step = make(cfg, p, cuda)
    g = torch.Generator().manual_seed(k * 10 + n)
    x, dy = torch.randn(3, 37, 128, generator=g), torch.randn(3, 37, 128, generator=g)
    q = {kk: v.double().requires_grad_(kk.startswith(pre) and not kk.endswith(sst.BUFFERS)) for kk, v in p.items()}
    xd = x.double().requires_grad_(True)
    stats = {}
    y_ref = sst.residual_block(q, pre, xd, n, stats)
    y_ref.backward(dy.double())
    step.conv.reset()
    step._ws = step.workspace(3 * 37)
    step._zp.begin(("block", k, n))
    xg = x.to(cuda)
    y, ys, ctx = step.block_fwd(xg, ops.Split.from_f32(xg), pre, k, n)
    dx = step.block_bwd(dy.to(cuda), ctx)
    assert rel_l2(y, y_ref) < 1e-5 and rel_l2(ys.float(), y_ref) < 2e-5 and rel_l2(dx, xd.grad) < 1e-4
    for kk, v in q.items():
        if v.requires_grad:
            assert rel_l2(step.grads[kk], v.grad) < 2e-4, kk
    for kk, v in stats.items():
        assert rel_l2(m.state_dict()[kk], v) < 1e-5, kk


def test_reference_executed_fixture_against_the_cuda_step(cuda):
    """The reference's own train-mode SpeedySpeech and losses (tests/golden/ref_executed_speedyspeech_train.npz) directly against
    SpeedySpeechTrainStep.forward_backward."""
    from test_speedyspeech_training_cpu import fixture_cases
    for tag, seed, tone_size, batch, losses, grads, norms, stats in fixture_cases():
        cfg = oss.SMALL_CFG
        m, step = make(cfg, oss.synth_params(seed, cfg, tone_size=tone_size), cuda, tone_size)
        p = oss.synth_params(seed, cfg, tone_size=tone_size)
        out, flips, compared = relu_mask_flips(step, batch, p, cfg, cuda)
        for kk, v in losses.items():
            assert abs(out[kk].item() - v) < 1e-4 * abs(v), (tag, kk)
        errs = sorted(((rel_l2(sst.fixture_sample(step.grads[kk]), g), kk) for kk, g in grads.items()), reverse=True)
        loose = [e for e in errs if e[0] >= 5e-3]
        print(f"fixture {tag}: {flips} ReLU mask flips of {compared}; {len(loose)} of {len(errs)} gradient tensors beyond 5e-3, worst {errs[0]}")
        # the accounting of check_forward_backward, without its duration-predictor clause: here a flip may sit in the predictor
        assert flips <= 1e-4 * compared and (flips > 0 or not loose), (tag, flips, loose[:8])
        assert errs[0][0] < 5e-2, (tag, errs[:8])
        for kk, v in stats.items():
            assert rel_l2(m.state_dict()[kk], v) < 1e-4, (tag, kk)


@pytest.mark.parametrize("tone_size", [None, 7])
def test_forward_backward_small_config(cuda, tone_size):
    """Kernel sizes 1, 3 and 4 (the duration predictor's), padded tokens and frames live, an all-padding token column."""
    check_forward_backward(cuda, oss.SMALL_CFG, [11, 7, 11, 3], tone_size, 20)


def test_forward_backward_shipped_config_recipe_shaped_batch(cuda):
    g = torch.Generator().manual_seed(0)
    lens = [int(v) for v in torch.randint(60, 141, (16,), generator=g)]
    check_forward_backward(cuda, oss.SHIPPED_CFG, lens, None, 30)


@pytest.mark.parametrize("clip", [1.0, 1e4])
def test_three_steps_follow_the_clipped_adam_trajectory(cuda, clip):
    """lr 2e-5 as in the FastSpeech2 trajectory test: Adam moves every weight by ~lr per step whatever its gradient, and at the
    recipe's 2e-3 a randomly initialised model is a chaotic regime that amplifies rounding, not a parity test."""
    cfg, lr = oss.SMALL_CFG, 2e-5
    p = oss.synth_params(40, cfg)
    m, step = make(cfg, p, cuda, max_grad_norm=clip, learning_rate=lr)
    state = {}
    q = {k: v.double() for k, v in p.items()}
    for i in range(3):
        batch = sst.synth_batch(50 + i, [9, 6, 8])
        losses, grads, stats = sst.train_step_grads(q, cfg, batch)
        q, norm = sst.clipped_adam_step({**q, **stats}, grads, state, lr=lr, max_grad_norm=clip)
        assert (norm > clip) == (clip == 1.0)               # one run clips, the other does not
        out = step.step(to_dev(batch, cuda))
        assert abs(out["loss"].item() - losses["loss"]) < 1e-4 * abs(losses["loss"]), i
    got = m.state_dict()
    for k, v in q.items():
        if k.endswith(sst.BUFFERS):
            assert rel_l2(got[k], v) < 1e-4, k
    names = [k for k in q if not k.endswith(sst.BUFFERS)]
    delta = torch.cat([(got[k].detach().double().cpu() - p[k].double()).reshape(-1) for k in names])
    ref = torch.cat([(q[k] - p[k].double()).reshape(-1) for k in names])
    assert 2.5 * lr < ref.abs().max().item() <= 3.02 * lr                    # three sign-like steps
    assert ((delta - ref).norm() / ref.norm()).item() < 0.1


def test_graph_replay_equals_eager_and_a_second_shape_gets_its_own_graph(cuda):
    cfg = oss.SMALL_CFG
    p = oss.synth_params(60, cfg)
    batches = [sst.synth_batch(61, [8, 5]), sst.synth_batch(62, [10, 4, 6])]
    m1, graphed = make(cfg, p, cuda)
    m2, eager = make(cfg, p, cuda)
    eager._graphs.enabled = False
    for rnd in range(3):                     # eager, capture, replay - for both shapes, interleaved
        for b in batches:
            a, e = graphed.step(to_dev(b, cuda)), eager.step(to_dev(b, cuda))
            assert a["loss"].item() == e["loss"].item(), rnd
    assert graphed._graphs.replays >= 2 and len(graphed._graphs._graphs) == 2
    for k, v in m1.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k


def test_a_captured_graph_survives_larger_shapes_and_evaluate(cuda):
    """The kernels' workspace address is baked into a captured graph: capture and replay a small shape, then run a larger shape
    and an evaluate on a larger batch (both need a larger workspace), then replay the small one - bit for bit an eager twin."""
    cfg = oss.SMALL_CFG
    p = oss.synth_params(65, cfg)
    small, large, larger = (to_dev(sst.synth_batch(66 + i, lens), cuda) for i, lens in enumerate(([5, 4], [12, 9, 11], [14, 14, 13, 12])))
    m1, graphed = make(cfg, p, cuda)
    m2, eager = make(cfg, p, cuda)
    eager._graphs.enabled = False
    for b in (small, small, small, large, small, large, large):
        a, e = graphed.step(b), eager.step(b)
        assert a["loss"].item() == e["loss"].item()
    assert graphed.evaluate(larger)["loss"].item() == eager.evaluate(larger)["loss"].item()
    mel = m1.eval().inference(small["phones"][0, :5])                     # new allocations between replays
    for b in (small, large, small):
        a, e = graphed.step(b), eager.step(b)
        assert a["loss"].item() == e["loss"].item()
    assert graphed._graphs.replays >= 5 and mel.shape[1] == 80
    for k, v in m1.state_dict().items():
        assert torch.equal(v, m2.state_dict()[k]), k


def test_evaluate_equals_oracle_eval_and_changes_nothing(cuda):
    cfg = oss.SMALL_CFG
    p = oss.synth_params(70, cfg, tone_size=5)
    batch = sst.synth_batch(71, [9, 9, 2], tone_size=5)
    m, step = make(cfg, p, cuda, tone_size=5)
    flag = m.training
    before = {k: v.clone() for k, v in m.state_dict().items()}
    out = step.evaluate(to_dev(batch, cuda))
    ref = sst.eval_losses(p, cfg, batch)
    for k, v in ref.items():
        assert abs(out[k].item() - v) < 1e-4 * abs(v), k
    assert m.training == flag and all(torch.equal(v, before[k]) for k, v in m.state_dict().items())


def test_checkpoint_resume_equals_uninterrupted_run(cuda, tmp_path):
    cfg = oss.SMALL_CFG
    p = oss.synth_params(80, cfg)
    batches = [to_dev(sst.synth_batch(81 + i, [7, 5]), cuda) for i in range(3)]
    m1, s1 = make(cfg, p, cuda)
    for b in batches:
        s1.step(b)
    m2, s2 = make(cfg, p, cuda)
    s2.step(batches[0])
    s2.step(batches[1])
    s2.save(str(tmp_path / "snapshot_iter_2.pdz"))
    m3, s3 = make(cfg, oss.synth_params(99, cfg), cuda)
    s3.load(str(tmp_path / "snapshot_iter_2.pdz"))
    assert s3.step_count == 2
    s3.step(batches[2])
    for k, v in m1.state_dict().items():
        assert torch.equal(v, m3.state_dict()[k]), k
    assert set(s1.state_dict()) == {"main_params", "main_optimizer", "epoch", "iteration"}


def test_inference_after_two_steps_uses_updated_weights_and_statistics(cuda):
    cfg = oss.SMALL_CFG
    p = oss.synth_params(90, cfg)
    m, step = make(cfg, p, cuda)
    m.eval()
    text = torch.randint(1, 40, (13,), generator=torch.Generator().manual_seed(1))
    first = m.inference(text.to(cuda))
    for i in range(2):
        step.step(to_dev(sst.synth_batch(91 + i, [9, 6]), cuda))
    assert not m.training                                      # the step neither needs nor sets train() mode
    mel = m.inference(text.to(cuda))
    now = {k: v.detach().cpu() for k, v in m.state_dict().items()}
    assert not torch.equal(now["decoder.postnet2.0.blocks.0.2._mean"], p["decoder.postnet2.0.blocks.0.2._mean"])
    with torch.no_grad():
        ref = oss.inference(now, cfg, text)
    assert mel.shape == ref.shape and rel_l2(mel, ref) < 1e-3
    assert first.shape != mel.shape or rel_l2(first, ref) > 1e-3


def test_bad_batches_raise_and_do_not_fault(cuda):
    cfg = oss.SMALL_CFG
    m, step = make(cfg, oss.synth_params(1, cfg), cuda)
    good = to_dev(sst.synth_batch(2, [6, 4]), cuda)
    with pytest.raises(_lib.PkError, match="frames"):
        step.step({**good, "feats": good["feats"][:, :-1]})
    with pytest.raises(_lib.PkError, match="tone_size"):
        step.step({**good, "tones": good["phones"]})
    with pytest.raises(_lib.PkError, match="shape"):
        step.step({**good, "num_frames": good["num_frames"][:1]})
    with pytest.raises(_lib.PkError, match="CUDA"):
        step.step({**good, "feats": good["feats"].cpu()})
    L = _lib.lib()
    x = torch.zeros(4, 64, device=cuda)
    assert L.pk_ss_bn_train_fwd(x.data_ptr(), 4, 64, x.data_ptr(), x.data_ptr(), 1e-5, 0.9, None, None, None, x.data_ptr(), x.data_ptr(),
                                None, None, x.data_ptr(), x.data_ptr(), None) == -3
