"""GPU parity of the Parallel WaveGAN training step (PWGUpdater.update_core, parallel_wavegan_updater.py:76-153) against torch
autograd on the oracle (oracle/pwg.py: generator, discriminator - pinned to the executed reference -, oracle/stft.py: MR-STFT loss)."""
import math

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu


def _rl2(a, b):
    a, b = a.detach().double().cpu().reshape(-1), b.detach().double().cpu().reshape(-1)
    return ((a - b).norm() / b.norm().clamp_min(1e-30)).item()


def _disc_wn_params(seed=12):
    from oracle import pwg as opwg
    p = opwg.synth_discriminator_params(seed)
    g = torch.Generator().manual_seed(seed + 1)
    out = {}
    for k, v in p.items():
        if k.endswith(".weight"):
            out[k + "_g"] = v.reshape(v.shape[0], -1).norm(dim=1) * (0.7 + 0.6 * torch.rand(v.shape[0], generator=g))
            out[k + "_v"] = v
        else:
            out[k] = v
    return out


def _leaf(params):
    return {k: v.clone().requires_grad_(True) for k, v in params.items()}


def test_gan_kernels_and_clipped_adam_unit(cuda):
    from oracle import pwg as opwg
    from oracle import stft as ostft
    from parakeet_b200 import _lib, ops
    from parakeet_b200.ops import _ptr, _stream
    from parakeet_b200.training.pwg_step import PWGTrainStep
    L = _lib.lib()
    g = torch.Generator().manual_seed(0)
    # gate forward / backward
    h = torch.randn(50, 128, generator=g, requires_grad=True)
    z = torch.tanh(h[:, :64]) * torch.sigmoid(h[:, 64:])
    dz = torch.randn(50, 64, generator=g)
    z.backward(dz)
    hc, dzc = h.detach().to(cuda), dz.to(cuda)
    zc, dhc = torch.empty(50, 64, device=cuda), torch.empty(50, 128, device=cuda)
    _lib.check(L.pk_gate_fwd(_ptr(hc), 50, 64, _ptr(zc), None, None, _stream()), "gate")
    _lib.check(L.pk_gate_bwd(_ptr(hc), _ptr(dzc), 50, 64, _ptr(dhc), _stream()), "gate_bwd")
    assert rel_err(zc, z) < 1e-5 and rel_err(dhc, h.grad) < 1e-5
    # weight norm forward / backward
    v = torch.randn(7, 30, generator=g, requires_grad=True)
    gg = (torch.rand(7, generator=g) + 0.5).requires_grad_(True)
    w = v * (gg / v.norm(dim=1))[:, None]
    dw = torch.randn(7, 30, generator=g)
    w.backward(dw)
    vc, gc, dwc = v.detach().to(cuda), gg.detach().to(cuda), dw.to(cuda)
    wc, dgc, dvc = torch.empty(7, 30, device=cuda), torch.empty(7, device=cuda), torch.empty(7, 30, device=cuda)
    _lib.check(L.pk_weight_norm_fwd(_ptr(vc), _ptr(gc), 7, 30, _ptr(wc), None, _stream()), "wn")
    _lib.check(L.pk_weight_norm_bwd(_ptr(vc), _ptr(gc), _ptr(dwc), 7, 30, _ptr(dgc), _ptr(dvc), _stream()), "wn_bwd")
    assert rel_err(wc, w) < 1e-5 and rel_err(dgc, gg.grad) < 1e-4 and rel_err(dvc, v.grad) < 1e-4
    # one upsampling stage forward / backward against the oracle's stretch + FIR
    x = torch.randn(6, 11, generator=g, requires_grad=True)
    fir = torch.randn(1, 1, 1, 11, generator=g, requires_grad=True)                  # scale 5: 2 s + 1 taps
    y = opwg.upsample_net({"p.up_layers.1.weight": fir}, x.unsqueeze(0), [5], prefix="p.")[0]
    dy = torch.randn(6, 55, generator=g)
    y.backward(dy)
    xc, fc, dyc = x.detach().to(cuda), fir.detach().reshape(-1).to(cuda), dy.to(cuda)
    yc, dxc, dfc = torch.empty(6, 55, device=cuda), torch.empty(6, 11, device=cuda), torch.zeros(11, dtype=torch.float64, device=cuda)
    _lib.check(L.pk_up_stage_fwd(_ptr(xc), _ptr(fc), 6, 11, 5, _ptr(yc), _stream()), "up")
    _lib.check(L.pk_up_stage_bwd(_ptr(xc), _ptr(dyc), _ptr(fc), 6, 11, 5, _ptr(dxc), _ptr(dfc), _stream()), "up_bwd")
    assert rel_err(yc, y) < 1e-5 and rel_err(dxc, x.grad) < 1e-5 and rel_err(dfc, fir.grad.reshape(-1)) < 1e-5
    # Adam with the global-norm clip (ClipGradByGlobalNorm + paddle Adam, epsilon 1e-6)
    from oracle import fastspeech2 as ofs
    p0, g0 = torch.randn(1000, generator=g), torch.randn(1000, generator=g) * 3
    clip = 10.0
    sc = clip / max(float(g0.norm()), clip)
    ref = ofs.adam_step({"w": p0}, {"w": g0 * sc}, {}, lr=1e-4, eps=1e-6)["w"]
    pc, gc2, mc, vc2 = p0.clone().to(cuda), g0.to(cuda), torch.zeros(1000, device=cuda), torch.zeros(1000, device=cuda)
    sq = torch.zeros(1, dtype=torch.float64, device=cuda)
    _lib.check(L.pk_sq_sum(_ptr(gc2), 1000, _ptr(sq), _stream()), "sq")
    _lib.check(L.pk_adam(_ptr(pc), _ptr(gc2), _ptr(mc), _ptr(vc2), 1000, 1e-4, 0.9, 0.999, 1e-6, 1, 1.0, _ptr(sq), clip, _stream()), "adam")
    assert abs(float(sq) - float(g0.double().pow(2).sum())) < 1e-3 * float(sq) and torch.allclose(pc.cpu(), ref, atol=1e-8)


def test_mr_stft_loss_value_and_gradient(cuda):
    from oracle import stft as ostft
    from parakeet_b200.models import PWGDiscriminator, PWGGenerator
    from oracle import pwg as opwg
    from parakeet_b200.training import PWGTrainStep
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(2, 7500, generator=g) * 0.3).requires_grad_(True)
    y = torch.randn(2, 7500, generator=g) * 0.3
    sc, mag = ostft.multi_resolution_stft_loss(x, y)
    (sc + mag).backward()
    gen = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device=cuda)
    ts = PWGTrainStep(gen, PWGDiscriminator(device=cuda))
    sc_c, mag_c, dx = ts.stft_loss(x.detach().to(cuda), y.to(cuda))
    assert abs(float(sc_c) - float(sc)) < 1e-4 * float(sc) and abs(float(mag_c) - float(mag)) < 1e-4 * float(mag)
    assert _rl2(dx, x.grad) < 2e-3, _rl2(dx, x.grad)


def _setup(cuda, frames=25, batch=2):
    from oracle import pwg as opwg
    from parakeet_b200.models import PWGDiscriminator, PWGGenerator
    gp = opwg.synth_params(2, weight_norm=True)
    dp = _disc_wn_params()
    gen = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device=cuda)
    gen.set_state_dict(gp)
    dis = PWGDiscriminator(device=cuda)
    assert sorted(dis.state_dict()) == sorted(dp)
    dis.set_state_dict(dp)
    noise, mel = opwg.synth_inputs(7, batch=batch, mel_frames=frames)
    wav = torch.randn(batch, 1, frames * 300, generator=torch.Generator().manual_seed(8)) * 0.3
    return gp, dp, gen, dis, noise, mel, wav


def test_discriminator_forward_and_step_gradients(cuda):
    from oracle import pwg as opwg
    from parakeet_b200.training import PWGTrainStep
    gp, dp, gen, dis, noise, mel, wav = _setup(cuda)
    with torch.no_grad():
        ref = opwg.discriminator_forward(opwg.fold_weight_norm(dp), wav)
    assert rel_err(dis(wav.to(cuda)), ref) < 1e-3
    ts = PWGTrainStep(gen, dis, discriminator_train_start_steps=0)
    ts.iteration = 1
    got = ts.discriminator_losses_and_grads(noise.to(cuda), mel.to(cuda), wav[:, 0].to(cuda))
    q = _leaf(dp)
    with torch.no_grad():
        wav_ = opwg.generator_forward(opwg.fold_weight_norm(gp), noise, mel)
    fd = opwg.fold_weight_norm(q)
    p, pf = opwg.discriminator_forward(fd, wav), opwg.discriminator_forward(fd, wav_)
    real, fake = torch.nn.functional.mse_loss(p, torch.ones_like(p)), torch.nn.functional.mse_loss(pf, torch.zeros_like(pf))
    (real + fake).backward()
    assert abs(float(got["real_loss"]) - float(real)) < 1e-3 * abs(float(real)) and abs(float(got["fake_loss"]) - float(fake)) < 1e-3 * abs(float(fake))
    errs = sorted(((k, _rl2(ts.d.grads[k], q[k].grad)) for k in q), key=lambda t: -t[1])
    assert errs[0][1] < 5e-3, errs[:6]


def test_generator_step_gradients_stft_only_and_adversarial(cuda):
    from oracle import pwg as opwg
    from parakeet_b200.training import PWGTrainStep
    gp, dp, gen, dis, noise, mel, wav = _setup(cuda)
    for adversarial in (False, True):
        ts = PWGTrainStep(gen, dis, discriminator_train_start_steps=0)
        ts.iteration = 1 if adversarial else 0
        got = ts.generator_losses_and_grads(noise.to(cuda), mel.to(cuda), wav[:, 0].to(cuda))
        q = _leaf(gp)
        out = opwg.gan_step_losses(opwg.fold_weight_norm(q), opwg.fold_weight_norm(dp), noise, mel, wav, adversarial=adversarial)
        out["generator_loss"].backward()
        for k in ("spectral_convergence_loss", "log_stft_magnitude_loss", "generator_loss") + (("adversarial_loss",) if adversarial else ()):
            assert abs(float(got[k]) - float(out[k])) < 2e-3 * abs(float(out[k])), (k, float(got[k]), float(out[k]))
        assert rel_err(ts._wav_fake, out["wav_"][:, 0]) < 1e-3
        errs = []
        for k in q:
            if q[k].grad is None:
                continue
            if float(q[k].grad.norm()) < 1e-6:
                # first_conv.weight_v: a weight-normed (64, 1, 1) kernel has rows of length 1, w = g * sign(v), d w / d v = 0 exactly
                assert float(ts.g.grads[k].norm()) < 1e-4, k
                continue
            errs.append((k, _rl2(ts.g.grads[k], q[k].grad)))
        errs.sort(key=lambda t: -t[1])
        assert errs[0][1] < 3e-2, (adversarial, errs[:8])
        assert sum(e > 1.5e-2 for _, e in errs) <= 0.1 * len(errs), (adversarial, errs[:24])


def test_update_core_matches_oracle_update(cuda):
    """One whole update_core past discriminator_train_start_steps: losses and BOTH parameter updates (clip + Adam eps 1e-6) against
    autograd + the oracle's Adam on the same noise."""
    from oracle import fastspeech2 as ofs
    from oracle import pwg as opwg
    from parakeet_b200.training import PWGTrainStep
    gp, dp, gen, dis, noise, mel, wav = _setup(cuda)
    ts = PWGTrainStep(gen, dis, discriminator_train_start_steps=0, use_graphs=False)
    ts.iteration = 1
    got = ts.update_core((wav, mel), noise=noise.to(cuda))

    def step(params, loss_fn, lr, clip):
        q = _leaf(params)
        loss = loss_fn(q)
        loss.backward()
        grads = {k: (v.grad if v.grad is not None else torch.zeros_like(v)) for k, v in q.items()}
        gn = math.sqrt(sum(float(g.double().pow(2).sum()) for g in grads.values()))
        sc = clip / max(gn, clip)
        return ofs.adam_step(params, {k: g * sc for k, g in grads.items()}, {}, lr=lr, eps=1e-6), float(loss)
    gp2, gl = step(gp, lambda q: opwg.gan_step_losses(opwg.fold_weight_norm(q), opwg.fold_weight_norm(dp), noise, mel, wav)["generator_loss"], 1e-4, 10.0)

    def dloss(q):
        with torch.no_grad():
            wav_ = opwg.generator_forward(opwg.fold_weight_norm(gp2), noise, mel)
        fd = opwg.fold_weight_norm(q)
        p, pf = opwg.discriminator_forward(fd, wav), opwg.discriminator_forward(fd, wav_)
        return torch.nn.functional.mse_loss(p, torch.ones_like(p)) + torch.nn.functional.mse_loss(pf, torch.zeros_like(pf))
    dp2, dl = step(dp, dloss, 5e-5, 1.0)
    assert abs(float(got["generator_loss"]) - gl) < 2e-3 * abs(gl) and abs(float(got["discriminator_loss"]) - dl) < 2e-3 * abs(dl)
    for name, new, old, model in (("G", gp2, gp, gen), ("D", dp2, dp, dis)):
        sd = model.state_dict()
        # Adam's first step moves every element by ~lr * g / (|g| + eps): elements whose gradient is small against the rounding
        # noise of the backward pass (the gradients themselves are checked above) take the other sign, so the comparison is on
        # the parameter DELTA in relative L2 per tensor - median tight, a small tail loose; first_conv.weight_v has zero gradient
        es = []
        for k, v in new.items():
            moved = (v - old[k]).double().norm().item()
            if moved < 1e-9 or k == "first_conv.weight_v":
                continue
            es.append((k, (sd[k].detach().double().cpu() - v.double()).norm().item() / moved))
        es.sort(key=lambda t: -t[1])
        assert es[len(es) // 2][1] < 0.05, (name, es[len(es) // 2])
        assert es[0][1] < 0.6 and sum(e > 0.35 for _, e in es) <= 0.03 * len(es), (name, es[:8])
    assert ts.iteration == 2 and ts.g.steps == 1 and ts.d.steps == 1


def test_update_core_graph_replay_matches_eager(cuda):
    """update_core with its two forward + backward halves replayed as CUDA graphs (third call on) against the eager step: the same
    losses and parameters after four steps, for fresh noise at every step."""
    from parakeet_b200.training import PWGTrainStep
    runs = []
    for graphs in (False, True):
        gp, dp, gen, dis, noise, mel, wav = _setup(cuda, frames=20)
        ts = PWGTrainStep(gen, dis, discriminator_train_start_steps=0, use_graphs=graphs)
        ts.iteration = 1
        g = torch.Generator().manual_seed(99)
        losses = []
        for _ in range(4):
            nz = torch.randn(noise.shape, generator=g).to(cuda)
            out = ts.update_core((wav, mel), noise=nz)
            losses.append([float(out["generator_loss"]), float(out["discriminator_loss"])])
        runs.append((losses, {k: v.detach().double().cpu().clone() for k, v in gen.state_dict().items()}, ts))
    assert runs[1][2]._graphs.replays >= 4 and runs[0][2]._graphs.replays == 0
    assert np.allclose(runs[0][0], runs[1][0], rtol=2e-3), (runs[0][0], runs[1][0])
    gp0 = _setup(cuda, frames=20)[0]
    k = "conv_layers.7.conv.weight_v"                                      # compare the parameter DELTAS (Adam sign noise, see above)
    d_e, d_g = runs[0][1][k] - gp0[k].double(), runs[1][1][k] - gp0[k].double()
    assert ((d_g - d_e).norm() / d_e.norm()).item() < 0.3
