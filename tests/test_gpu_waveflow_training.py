"""WaveFlowTrainStep on the GPU: loss and every parameter gradient against fp64 autograd on the oracle, the reference's zero
output_proj initialisation, Adam against the oracle's Paddle restatement, and bit-for-bit reproducibility (two steps from one
state, eager vs captured vs replayed)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

GRAD_TOL = 5e-3


def _setup(cuda, channels, seed, n_group=16, n_flows=2, n_layers=3, batch=3, frames=28, samples=None, zero_output_proj=False):
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    p = owf.synth_params(seed, upsample_factors=(16, 16), n_flows=n_flows, n_layers=n_layers, n_group=n_group, channels=channels, n_mels=80)
    if zero_output_proj:                                   # the reference's initialisation (Constant(0.))
        p = {k: (torch.zeros_like(v) if "output_proj" in k else v) for k, v in p.items()}
    m = ConditionalWaveFlow([16, 16], n_flows, n_layers, n_group, channels, 80, (3, 3), device=cuda)
    m.set_state_dict(p)
    g = torch.Generator().manual_seed(seed + 7)
    mel = torch.randn(batch, 80, frames, generator=g) * 0.5 - 3
    audio = (torch.rand(batch, samples or frames * 256 - 7, generator=g) * 2 - 1) * 0.5
    return m, p, audio, mel, dict(n_flows=n_flows, n_layers=n_layers, n_group=n_group)


def _rel_l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / max(float(b.norm()), 1e-300))


def _noise_only(k):
    """input_proj.weight_v: weight norm over ONE input element makes w = g * sign(v); its gradient is 0 up to rounding."""
    return k.endswith("input_proj.weight_v")


def _check_grads(step, p, ref, loss, ref_loss, tol=GRAD_TOL):
    assert abs(float(loss) - float(ref_loss)) <= 1e-5 * abs(float(ref_loss)), (float(loss), float(ref_loss))
    errs = {}
    for k in p:
        got = step.grads[k]
        if _noise_only(k):
            scale = float(ref[k[:-1] + "g"].norm())
            assert float(got.double().norm()) <= 1e-5 * scale, k
            continue
        errs[k] = _rel_l2(got, ref[k])
    worst = max(errs, key=errs.get)
    print(f"worst gradient {worst}: {errs[worst]:.2e}; median {sorted(errs.values())[len(errs) // 2]:.2e}")
    bad = {k: v for k, v in errs.items() if v > tol}
    assert not bad, bad


@pytest.mark.parametrize("channels,n_group,frames", [(64, 16, 28), (128, 16, 28), (64, 8, 28)])
def test_loss_and_every_gradient_vs_fp64_oracle(cuda, channels, n_group, frames):
    """B = 3, 28 frames, 28 * 256 - 7 samples (W = 447 at n_group 16: every width dilation reaches live columns, the last
    128-column tile is partial)."""
    from oracle import waveflow_train as owt
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    m, p, audio, mel, cfg = _setup(cuda, channels, 11 + channels + n_group, n_group=n_group, frames=frames)
    step = WaveFlowTrainStep(m)
    loss = step.forward_backward_graphed(audio.to(cuda), mel.to(cuda))
    ref_loss, ref = owt.train_grads(p, audio, mel, **cfg)
    _check_grads(step, p, ref, loss, ref_loss)


def test_recipe_clip_length_128_channels(cuda):
    """The recipe's clip length (65 frames = 16 640 samples, W = 1040) at 128 channels and 8 layers (width dilations up to 128)."""
    from oracle import waveflow_train as owt
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    m, p, audio, mel, cfg = _setup(cuda, 128, 3, n_layers=8, batch=2, frames=65, samples=16640)
    step = WaveFlowTrainStep(m)
    loss = step.forward_backward_graphed(audio.to(cuda), mel.to(cuda))
    ref_loss, ref = owt.train_grads(p, audio, mel, **cfg)
    _check_grads(step, p, ref, loss, ref_loss)


def test_zero_output_proj_initialisation(cuda):
    from oracle import waveflow_train as owt
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    m, p, audio, mel, cfg = _setup(cuda, 64, 5, frames=12, zero_output_proj=True)
    step = WaveFlowTrainStep(m)
    step.forward_backward_graphed(audio.to(cuda), mel.to(cuda))
    _, ref = owt.train_grads(p, audio, mel, **cfg)
    for k in p:
        if "output_proj" in k:
            assert _rel_l2(step.grads[k], ref[k]) < GRAD_TOL, k
        else:
            assert float(step.grads[k].abs().max()) == 0.0, k


def test_adam_matches_oracle_and_three_steps_follow_its_trajectory(cuda):
    from oracle import waveflow_train as owt
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    m, p, audio, mel, cfg = _setup(cuda, 64, 9, frames=12)
    step = WaveFlowTrainStep(m, learning_rate=2e-4)
    a, me = audio.to(cuda), mel.to(cuda)
    p0 = {k: v.detach().cpu().clone() for k, v in m.state_dict().items()}
    loss = step.step((me, a))
    assert tuple(loss.shape) == (1,) and loss.is_cuda
    grads = {k: v.detach().cpu().clone() for k, v in step.grads.items()}
    want = owt.adam_step(p0, grads, {}, lr=2e-4)
    for k, v in m.state_dict().items():
        assert float((v.cpu() - want[k]).abs().max()) <= 1e-6, k
    # two more steps; the oracle runs the same three steps in fp64
    step.step((me, a))
    step.step((me, a))
    q, st = {k: v.double() for k, v in p.items()}, {}
    for _ in range(3):
        _, g = owt.train_grads(q, audio, mel, **cfg)
        q = owt.adam_step(q, g, st, lr=2e-4)
    for k, v in m.state_dict().items():
        if _noise_only(k):          # Adam turns a rounding-noise gradient into steps of up to ~1e-2 lr: only bounded
            assert float((v.cpu().double() - p[k].double()).abs().max()) <= 2e-5, k
            continue
        assert _rel_l2(v.cpu().double() - p[k].double(), q[k] - p[k].double()) < 2e-2, k


def test_steps_are_bit_reproducible_and_replay_equals_eager(cuda):
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    outs = []
    for _ in range(2):
        m, p, audio, mel, _ = _setup(cuda, 64, 21, frames=10)
        step = WaveFlowTrainStep(m)
        a, me = audio.to(cuda), mel.to(cuda)
        losses = [step.forward_backward_graphed(a, me).clone() for _ in range(3)]   # eager, captured, replayed
        grads = step.gflat.clone()
        for _ in range(3):
            step.forward_backward_graphed(a, me)
            assert torch.equal(step.gflat, grads)
        assert step._graphs.replays >= 3
        assert all(torch.equal(x, losses[0]) for x in losses)
        step.step((me, a))
        step.step((me, a))
        outs.append((losses[0], grads, step.flat.clone()))
    assert torch.equal(outs[0][0], outs[1][0]) and torch.equal(outs[0][1], outs[1][1]) and torch.equal(outs[0][2], outs[1][2])


def test_state_dict_round_trip_and_cuda_only(cuda, tmp_path):
    from parakeet_b200._lib import PkError
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    m, p, audio, mel, _ = _setup(cuda, 64, 2, frames=8)
    step = WaveFlowTrainStep(m)
    with pytest.raises(PkError):
        step.step((mel, audio))
    a, me = audio.to(cuda), mel.to(cuda)
    step.step((me, a))
    base = step.save(str(tmp_path))
    assert base.endswith("step-1")
    step.step((me, a))
    after_two = step.flat.clone()
    m2, *_ = _setup(cuda, 64, 2, frames=8)
    step2 = WaveFlowTrainStep(m2)
    assert step2.load(str(tmp_path)) == 1 and step2.step_count == 1
    step2.step((me, a))
    assert torch.equal(step2.flat, after_two)
    # the model's tensors are views of the flat buffer: state_dict shows the updated weights
    assert torch.equal(m2.state_dict()["decoder.0.resnet.0.conv.weight_v"].reshape(-1),
                       step2.flat[step2.off["decoder.0.resnet.0.conv.weight_v"]:][:m2.state_dict()["decoder.0.resnet.0.conv.weight_v"].numel()])


def test_gradients_vs_executed_reference(cuda):
    """The gradients the reference's own ConditionalWaveFlow.forward + WaveFlowLoss produced (2 flows x 8 layers, 64 channels)."""
    from test_waveflow_training_cpu import _sampled, golden_setup
    from parakeet_b200.models import ConditionalWaveFlow
    from parakeet_b200.training.waveflow_step import WaveFlowTrainStep
    g, p, audio, mel, cfg = golden_setup()
    m = ConditionalWaveFlow([16, 16], 2, 8, 16, 64, 80, (3, 3), device=cuda)
    m.set_state_dict(p)
    step = WaveFlowTrainStep(m)
    loss = step.forward_backward_graphed(audio.to(cuda), mel.to(cuda))
    assert abs(float(loss) - float(g["loss"][0])) <= 1e-5 * abs(float(g["loss"][0]))
    for k in p:
        if _noise_only(k):
            continue
        assert _rel_l2(_sampled(step.grads[k]), torch.from_numpy(g["grad/" + k])) < GRAD_TOL, k
        assert abs(float(step.grads[k].double().norm()) - float(g["gradnorm/" + k])) <= GRAD_TOL * float(g["gradnorm/" + k]), k


# ------------------------------------------------------------------------------------------------ single kernels vs fp64 autograd
def test_upsample_bwd_kernel_alone(cuda):
    """pk_waveflow_upsample_bwd: leaky_relu(0.4) o Conv2DTranspose(1 -> 1, (3, 2f), stride (1, f), pad (1, f/2)), untrimmed."""
    import torch.nn.functional as F
    from parakeet_b200 import _lib
    from parakeet_b200.ops import _ptr, _stream
    L = _lib.lib()
    g = torch.Generator().manual_seed(3)
    for B, M, t_in, f in ((2, 80, 9, 16), (3, 72, 37, 8)):
        x = torch.randn(B, M, t_in, generator=g, dtype=torch.float64)
        w = torch.randn(3, 2 * f, generator=g, dtype=torch.float64) * 0.3
        b = torch.randn(1, generator=g, dtype=torch.float64) * 0.1
        dy = torch.randn(B, M, t_in * f, generator=g, dtype=torch.float64)
        xr, wr, br = (t.clone().requires_grad_(True) for t in (x, w, b))
        y = F.leaky_relu(F.conv_transpose2d(xr[:, None], wr[None, None], br, stride=(1, f), padding=(1, f // 2)), 0.4)[:, 0]
        dx_ref, dw_ref, db_ref = torch.autograd.grad(y, (xr, wr, br), dy)
        xc, wc, bc, dyc = (t.float().to(cuda).contiguous() for t in (x, w, b, dy))
        yc = torch.empty(B, M, t_in * f, device=cuda)
        _lib.check(L.pk_waveflow_upsample(_ptr(xc), _ptr(wc), _ptr(bc), B, M, t_in, f, 0, 0.4, _ptr(yc), _stream()))
        assert _rel_l2(yc, y.detach()) < 1e-6
        dpre, dx, dw, db = torch.empty_like(yc), torch.empty_like(xc), torch.empty_like(wc), torch.empty(1, device=cuda)
        scratch = torch.empty(1 << 16, device=cuda)
        _lib.check(L.pk_waveflow_upsample_bwd(_ptr(xc), _ptr(yc), _ptr(dyc), _ptr(wc), B, M, t_in, f, 0.4, _ptr(dpre), _ptr(dx), _ptr(scratch),
                                              scratch.numel(), _ptr(dw), _ptr(db), _stream()))
        assert _rel_l2(dx, dx_ref) < 1e-5 and _rel_l2(dw, dw_ref) < 1e-5 and _rel_l2(db, db_ref) < 1e-5


def test_forward_tail_bwd_kernel_alone(cuda):
    """pk_waveflow_forward_tail_bwd against autograd of z = x exp(logs) + b, (logs, b) = output_proj(skip), the permutation and
    the loss terms sum(z'^2) / (2 n) - sum(logs) / n (the last flow) or <dy, x_next> (any other)."""
    from parakeet_b200 import _lib
    from parakeet_b200.ops import Split, _ptr, _stream
    L = _lib.lib()
    gen = torch.Generator().manual_seed(5)
    B, G, W, C = 2, 16, 45, 64
    perm = list(reversed(range(G // 2))) + list(reversed(range(G // 2, G)))
    inv = [perm.index(h) for h in range(G)]
    skip = torch.randn(B, G + 1, W, C, generator=gen, dtype=torch.float64) * 0.3
    skip[:, G - 1:] = 0
    out_w = torch.randn(2, C, generator=gen, dtype=torch.float64) * 0.05
    out_b = torch.randn(2, generator=gen, dtype=torch.float64) * 0.05
    x = torch.randn(B, G, W, generator=gen, dtype=torch.float64)
    dy = torch.randn(B, G, W, generator=gen, dtype=torch.float64)
    n = B * G * W
    sc, wr, br = (t.clone().requires_grad_(True) for t in (skip, out_w, out_b))
    par = torch.einsum("bjwc,kc->bjwk", sc[:, :G - 1], wr) + br
    z = torch.cat([x[:, :1], x[:, 1:] * torch.exp(par[..., 0]) + par[..., 1]], 1)
    xn = z[:, perm]
    skip_c, w_c, b_c, x_c, dy_c = (t.float().to(cuda).contiguous() for t in (skip, out_w, out_b, x, dy))   # named: must outlive the launches
    inv_c = torch.tensor(inv, dtype=torch.int32, device=cuda)
    xn_c, logs_c = torch.empty(B, G, W, device=cuda), torch.empty(B, G - 1, W, device=cuda)
    _lib.check(L.pk_waveflow_train_tail_fwd(_ptr(skip_c), _ptr(w_c), _ptr(b_c), _ptr(x_c), _ptr(inv_c), B, G, W, C, _ptr(xn_c), _ptr(logs_c),
                                            _stream()))
    assert _rel_l2(xn_c, xn.detach()) < 1e-6
    for last in (False, True):
        obj = ((xn ** 2).sum() / (2 * n) - par[..., 0].sum() / n) if last else (xn * dy).sum()
        d_skip, d_w, d_b = torch.autograd.grad(obj, (sc, wr, br), retain_graph=True)
        xr = x.clone().requires_grad_(True)
        z2 = torch.cat([xr[:, :1], xr[:, 1:] * torch.exp(par.detach()[..., 0]) + par.detach()[..., 1]], 1)[:, perm]
        dx_ref = torch.autograd.grad(((z2 ** 2).sum() / (2 * n)) if last else (z2 * dy).sum(), xr)[0]
        dx, dparams = torch.empty(B, G, W, device=cuda), torch.zeros(B, G + 1, W, 2, device=cuda)
        dskip, ds = torch.zeros(B, G + 1, W, C, device=cuda), Split.zeros((B * (G + 1) * W, 2 * C), cuda)
        _lib.check(L.pk_waveflow_forward_tail_bwd(_ptr(skip_c), _ptr(w_c), _ptr(b_c), _ptr(x_c), _ptr(inv_c),
                                                  _ptr(None if last else dy_c), _ptr(xn_c if last else None), 1.0 / n, -1.0 / n if last else 0.0,
                                                  B, G, W, C, _ptr(dx), _ptr(dparams), _ptr(dskip), _ptr(ds.hi), _ptr(ds.lo), 2 * C, C, _stream()))
        assert _rel_l2(dx, dx_ref) < 1e-5 and _rel_l2(dskip, d_skip) < 1e-5, last
        assert _rel_l2(ds.float()[:, C:].reshape(B, G + 1, W, C), d_skip) < 1e-5
        assert _rel_l2(torch.einsum("bjwk,bjwc->kc", dparams.double().cpu(), skip), d_w) < 1e-5
        assert _rel_l2(dparams.double().cpu().sum((0, 1, 2)), d_b) < 1e-5


def _planes(v, cuda):
    from parakeet_b200.ops import Split
    v = v.float()
    hi = v.to(torch.bfloat16)
    lo = (v - hi.float()).to(torch.bfloat16)
    s = Split.empty(tuple(v.shape), cuda)
    s.hi.copy_(hi)
    s.lo.copy_(lo)
    return s


@pytest.mark.parametrize("channels", [64, 128])
def test_backward_layer_kernel_alone(cuda, channels):
    """pk_waveflow_backward_layer at W = 447 (dilation 128 reaches live columns on both sides, the last 128-column tile is
    partial), n_group 16, both GEMMs, against fp64 autograd of conv2d (causal height padding [2, 0], width 'same') and the gate."""
    import ctypes as C_
    import torch.nn.functional as F
    from parakeet_b200 import _lib
    from parakeet_b200.ops import _stream
    L = _lib.lib()
    C, B, G, W, d, NL = channels, 2, 16, 447, 128, 2
    Q = B * (G + 1)
    gen = torch.Generator().manual_seed(channels)
    r = lambda *s, k=1.0: torch.randn(*s, generator=gen, dtype=torch.float64) * k
    w1, w2 = r(2 * C, C, 3, 3, k=(1 / (9 * C)) ** 0.5), r(2 * C, C, k=C ** -0.5)
    dh_in, dx_old, dskip, h = r(B, G - 1, W, 2 * C), r(B, G - 1, W, C), r(B, G - 1, W, C), r(B, G - 1, W, 2 * C)
    net = lambda t: torch.cat([t, torch.zeros(B, 2, *t.shape[2:], dtype=t.dtype)], 1).reshape(Q, W, t.shape[-1])
    # operands as the step holds them; the fp64 reference uses exactly the split values the kernel reads
    dh_all = torch.zeros(Q + 2, W, NL * 2 * C, dtype=torch.float64)
    dh_all[:Q, :, 2 * C:] = net(dh_in)
    dh_s = _planes(dh_all, cuda)
    dh_in = dh_s.float().double().cpu()[:Q, :, 2 * C:].reshape(B, G + 1, W, 2 * C)[:, :G - 1]
    a2 = torch.zeros(Q, W, 2 * C, dtype=torch.float64)
    a2[:, :, C:] = net(dskip)
    a2_s = _planes(a2, cuda)
    dskip = a2_s.float().double().cpu()[:, :, C:].reshape(B, G + 1, W, C)[:, :G - 1]
    w1b = torch.cat([w1[:, :, 2 - s, :].flip(-1).permute(1, 2, 0).reshape(C, 6 * C) for s in range(3)], 1)
    w1b_s, w2b_s = _planes(w1b, cuda), _planes(w2.t().contiguous(), cuda)
    w1q = torch.zeros_like(w1)                               # the weights as the kernel sees them (hi + lo)
    w1bq = w1b_s.float().double().cpu().reshape(C, 3, 3, 2 * C)
    for s in range(3):
        w1q[:, :, 2 - s, :] = w1bq[:, s].permute(2, 0, 1).flip(-1)
    w2q = w2b_s.float().double().cpu().t()
    dx = net(dx_old).float().to(cuda).contiguous()
    h_c = net(h).float().to(cuda).contiguous()
    a = _lib.WaveflowBackwardLayerArgs()
    a.batch, a.width, a.channels, a.n_group, a.dilation, a.has_gemm1, a.has_gemm2, a.dh_ld = B, W, C, G, d, 1, 1, NL * 2 * C
    a.dh_in_hi, a.dh_in_lo = dh_s.hi[:, :, 2 * C:].data_ptr(), dh_s.lo[:, :, 2 * C:].data_ptr()
    a.w1_hi, a.w1_lo, a.w2_hi, a.w2_lo = w1b_s.hi.data_ptr(), w1b_s.lo.data_ptr(), w2b_s.hi.data_ptr(), w2b_s.lo.data_ptr()
    a.dx, a.a2_hi, a.a2_lo, a.h = dx.data_ptr(), a2_s.hi.data_ptr(), a2_s.lo.data_ptr(), h_c.data_ptr()
    a.dh_out_hi, a.dh_out_lo = dh_s.hi.data_ptr(), dh_s.lo.data_ptr()
    _lib.check(L.pk_waveflow_backward_layer(C_.byref(a), _stream()))
    # reference: dx = dx_old + conv^T(dh_in); dz = [dx | dskip] W2; gate backward with h
    x = torch.zeros(B, C, G - 1, W, dtype=torch.float64, requires_grad=True)
    y = F.conv2d(F.pad(x, (d, d, 2, 0)), w1q, dilation=(1, d))
    dx_ref = dx_old + torch.autograd.grad(y, x, dh_in.permute(0, 3, 1, 2))[0].permute(0, 2, 3, 1)
    dz = torch.cat([dx_ref, dskip], -1) @ w2q
    t, sg = torch.tanh(h[..., :C]), torch.sigmoid(h[..., C:])
    dh_ref = torch.cat([dz * sg * (1 - t * t), dz * t * sg * (1 - sg)], -1)
    unnet = lambda t_: t_.reshape(B, G + 1, W, -1)[:, :G - 1].double().cpu()
    assert _rel_l2(unnet(dx), dx_ref) < 2e-5
    assert _rel_l2(unnet(a2_s.float()[:, :, :C]), dx_ref) < 2e-5
    out = dh_s.float()[:Q, :, :2 * C]
    assert _rel_l2(unnet(out), dh_ref) < 5e-5
    assert float(out.reshape(B, G + 1, W, 2 * C)[:, G - 1:].abs().max()) == 0.0     # pad rows untouched


def test_small_training_kernels_alone(cuda):
    """pk_waveflow_train_outer_sum, _loss, _cond_gather / _cond_scatter (adjoint pair), _input_fwd / _input_bwd and _update, each
    against fp64 torch on the same inputs; the reductions are run twice and must agree bit for bit."""
    import math
    from parakeet_b200 import _lib
    from parakeet_b200.ops import Split, _ptr, _stream
    L, st = _lib.lib(), _stream()
    gen = torch.Generator().manual_seed(13)
    r = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    f = lambda t: t.float().to(cuda).contiguous()
    # outer_sum: out[i, j] = sum_r a[r, i] b[r, j], and the column sum (b = NULL)
    a, b = r(5000, 96), r(5000, 2)
    a_c, b_c, scratch, out = f(a), f(b), torch.empty(1 << 18, device=cuda), torch.empty(96, 2, device=cuda)
    _lib.check(L.pk_waveflow_train_outer_sum(_ptr(a_c), 96, 96, _ptr(b_c), 2, 2, 5000, _ptr(scratch), scratch.numel(), _ptr(out), 2, 1, 0, st))
    assert _rel_l2(out, a.t() @ b) < 1e-6
    first = out.clone()
    _lib.check(L.pk_waveflow_train_outer_sum(_ptr(a_c), 96, 96, _ptr(b_c), 2, 2, 5000, _ptr(scratch), scratch.numel(), _ptr(out), 2, 1, 0, st))
    assert torch.equal(out, first)
    col = torch.empty(96, device=cuda)
    _lib.check(L.pk_waveflow_train_outer_sum(_ptr(a_c), 96, 96, None, 1, 1, 5000, _ptr(scratch), scratch.numel(), _ptr(col), 1, 0, 0, st))
    assert _rel_l2(col, a.sum(0)) < 1e-6
    # loss
    z, logs = r(3, 4000), r(7000) * 0.1
    z_c, logs_c, loss = f(z), f(logs), torch.empty(1, device=cuda)
    _lib.check(L.pk_waveflow_train_loss(_ptr(z_c), z.numel(), _ptr(logs_c), logs.numel(), 0.7, _ptr(loss), st))
    want = ((z.float().double() ** 2).sum() / (2 * 0.49) - logs.float().double().sum()) / z.numel() + 0.5 * math.log(2 * math.pi) + math.log(0.7)
    assert abs(float(loss) - float(want)) <= 1e-6 * abs(float(want))
    # cond gather / scatter: <gather(c), y> == <c, scatter(y)>
    B, G, W, M = 2, 8, 37, 80
    Q, tc = B * (G + 1), W * G + 5
    rows = torch.tensor([3, 1, 7, 0, 2, 6, 4, 5], dtype=torch.int32, device=cuda)
    c, y = r(B, M, tc), r(Q, W, M)
    c_c, y_c, g = f(c), f(y), Split.empty((Q, W, M), cuda)
    _lib.check(L.pk_waveflow_train_cond_gather(_ptr(c_c), _ptr(rows), B, G, W, M, tc, _ptr(g.hi), _ptr(g.lo), st))
    dc = torch.zeros(B, M, tc, device=cuda)
    _lib.check(L.pk_waveflow_train_cond_scatter(_ptr(y_c), _ptr(rows), B, G, W, M, tc, _ptr(dc), st))
    rr = rows.cpu().long()
    ref = torch.zeros(B, G + 1, W, M, dtype=torch.float64)
    for j in range(G - 1):
        ref[:, j] = c.float().double()[:, :, rr[j + 1]::G][:, :, :W].permute(0, 2, 1)
    assert _rel_l2(g.float(), ref.reshape(Q, W, M)) < 1e-5
    lhs = float((g.float().double().cpu() * y.float().double()).sum())
    rhs = float((dc.double().cpu() * c.float().double()).sum())
    assert abs(lhs - rhs) <= 1e-4 * abs(lhs) + 1e-3
    # input_proj forward / backward and the residual update
    C = 64
    x, w, bias, dh = r(B, G, W), r(C), r(C), r(Q, W, C)
    x_c, w_c, bias_c, dh_c = f(x), f(w), f(bias), f(dh)
    h32, xin = torch.empty(Q, W, C, device=cuda), Split.zeros((Q + 2, W, C), cuda)
    _lib.check(L.pk_waveflow_train_input_fwd(_ptr(x_c), _ptr(w_c), _ptr(bias_c), B, G, W, C, _ptr(h32), _ptr(xin.hi), _ptr(xin.lo), st))
    href = torch.zeros(B, G + 1, W, C, dtype=torch.float64)
    href[:, :G - 1] = x.float().double()[:, :G - 1, :, None] * w.float().double() + bias.float().double()
    assert _rel_l2(h32, href.reshape(Q, W, C)) < 1e-6
    assert _rel_l2(xin.float()[2:], href.reshape(Q, W, C)) < 1e-5
    dx, xcol = torch.zeros(B, G, W, device=cuda), torch.zeros(Q, W, device=cuda)
    _lib.check(L.pk_waveflow_train_input_bwd(_ptr(dh_c), _ptr(x_c), _ptr(w_c), B, G, W, C, _ptr(dx), _ptr(xcol), st))
    dhn = dh.float().double().reshape(B, G + 1, W, C)[:, :G - 1]
    assert _rel_l2(dx[:, :G - 1], dhn @ w.float().double()) < 1e-5 and float(dx[:, G - 1].abs().max()) == 0.0
    out, skip = r(Q, W, 2 * C), torch.zeros(Q, W, C, device=cuda)
    out_c, nxt = f(out), Split.zeros((Q + 2, W, C), cuda)
    _lib.check(L.pk_waveflow_train_update(_ptr(out_c), B, G, W, C, _ptr(h32), _ptr(skip), 1, _ptr(nxt.hi), _ptr(nxt.lo), st))
    h_new = href.reshape(Q, W, C) + out.float().double()[..., :C]
    assert _rel_l2(h32, h_new) < 1e-6 and _rel_l2(skip, out.float().double()[..., C:]) < 1e-6
    live = torch.tensor(([1.0] * (G - 1) + [0.0, 0.0]) * B, dtype=torch.float64)[:, None, None]
    assert _rel_l2(nxt.float()[2:], h_new * live) < 1e-5
