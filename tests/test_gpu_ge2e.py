"""GE2E speaker encoder on the H100: the persistent LSTM kernels against fp64, the model against the oracle, the training step's
gradients, clipped-Adam trajectory, graph replay and checkpoint resume."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _cell_ref(g_in, b_hh, w_hh, h0, c0):
    """fp64 recurrence of one layer, time-major g_in (T, B, 4H) -> (h (T+1, B, H), c (T+1, B, H), gates (T, B, 4H))."""
    T = g_in.shape[0]
    h, c = [h0], [c0]
    gs = []
    for t in range(T):
        z = g_in[t] + b_hh + h[-1] @ w_hh.t()
        i, f, g, o = z.chunk(4, 1)
        i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
        c.append(f * c[-1] + i * g)
        h.append(o * torch.tanh(c[-1]))
        gs.append(torch.cat([i, f, g, o], 1))
    return torch.stack(h), torch.stack(c), torch.stack(gs)


@pytest.mark.parametrize("rows,T,H,init", [(1, 160, 256, False), (63, 7, 256, True), (64, 1, 256, False), (65, 12, 256, True),
                                           (640, 160, 256, False), (64 * 40, 3, 256, True), (65, 20, 64, True)])
def test_lstm_fwd_against_fp64(rows, T, H, init):
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(rows + T)
    g_in = torch.randn(T, rows, 4 * H, generator=g) * 0.5
    w_hh = (torch.rand(4 * H, H, generator=g) * 2 - 1) / H ** 0.5
    b_hh = torch.randn(4 * H, generator=g) * 0.1
    h0 = torch.randn(rows, H, generator=g) * 0.3 if init else torch.zeros(rows, H)
    c0 = torch.randn(rows, H, generator=g) * 0.3 if init else torch.zeros(rows, H)
    h_ref, c_ref, g_ref = _cell_ref(g_in.double(), b_hh.double(), w_hh.double(), h0.double(), c0.double())
    from parakeet_b200.models.lstm_speaker_encoder import start_states
    wp = ops.lstm_pack_fwd(w_hh.to(DEV), ops.lstm_gate_perm(H, DEV))
    h_all, h_split, c = start_states(T, rows, H, DEV, h0.to(DEV), c0.to(DEV))
    ops.lstm_fwd(g_in.to(DEV), b_hh.to(DEV), wp, h_all, h_split, c)
    assert _rel(h_all, h_ref) < 1e-3 and _rel(c, c_ref[-1]) < 1e-3
    assert torch.equal(h_split.hi.float() + h_split.lo.float(), ops.Split.from_f32(h_all).float())
    h2, h2_split, c_all = start_states(T, rows, H, DEV, h0.to(DEV), c0.to(DEV), keep_c=True)
    gates = torch.empty(T, rows, 4 * H, device=DEV)
    ops.lstm_fwd(g_in.to(DEV), b_hh.to(DEV), wp, h2, h2_split, c_all, gates)
    assert torch.equal(h2, h_all) and _rel(c_all, c_ref) < 1e-3 and _rel(gates, g_ref) < 1e-3


@pytest.mark.parametrize("rows,T,H", [(65, 9, 256), (640, 20, 256), (3, 5, 64)])
def test_lstm_bwd_against_fp64_autograd(rows, T, H):
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(7 * rows + T)
    g_in = (torch.randn(T, rows, 4 * H, generator=g) * 0.5).double().requires_grad_(True)
    w_hh = ((torch.rand(4 * H, H, generator=g) * 2 - 1) / H ** 0.5).double()
    b_hh = (torch.randn(4 * H, generator=g) * 0.1).double()
    dh_in = torch.randn(T, rows, H, generator=g).double()
    dh_last = torch.randn(rows, H, generator=g).double()
    h, c, gates = _cell_ref(g_in, b_hh, w_hh, torch.zeros(rows, H, dtype=torch.float64), torch.zeros(rows, H, dtype=torch.float64))
    ((h[1:] * dh_in).sum() + (h[-1] * dh_last).sum()).backward()
    from parakeet_b200.models.lstm_speaker_encoder import start_states
    h_all, h_split, c_all = start_states(T, rows, H, DEV, keep_c=True)
    gd = torch.empty(T, rows, 4 * H, device=DEV)
    w32 = w_hh.float().to(DEV)
    ops.lstm_fwd(g_in.detach().float().to(DEV), b_hh.float().to(DEV), ops.lstm_pack_fwd(w32, ops.lstm_gate_perm(H, DEV)), h_all, h_split,
                 c_all, gd)
    dg = torch.empty(T, rows, 4 * H, device=DEV)
    split = ops.Split.empty((T, rows, 4 * H), DEV)
    ops.lstm_bwd(ops.lstm_pack_bwd(w32), gd, c_all, dh_in.float().to(DEV), dh_last.float().to(DEV), dg, split)
    assert _l2(dg, g_in.grad) < 5e-3
    assert torch.equal(split.hi.float() + split.lo.float(), ops.Split.from_f32(dg).float())


def _model(tag):
    from oracle import ge2e as og
    from parakeet_b200.models import LSTMSpeakerEncoder
    cfg, shape, seed = og.GOLDEN_CONFIGS[tag]
    p = og.synth_params(seed, *cfg)
    m = LSTMSpeakerEncoder(*cfg, device=DEV)
    m.set_state_dict(p)
    return m, p, cfg, shape, seed


@pytest.mark.parametrize("tag", ["small", "shipped"])
def test_embeddings_loss_and_similarity_against_oracle(tag):
    from oracle import ge2e as og
    m, p, cfg, (N, M, T), seed = _model(tag)
    x = og.synth_utterances(seed + 100, N * M, T, cfg[0])
    h0, c0 = og.synth_states(seed + 200, cfg[1], N * M, cfg[2])
    with torch.no_grad():
        assert _rel(m.embed_sequences(x.to(DEV)), og.embed_sequences(p, x)) < 1e-3
        assert _rel(m.embed_utterance(x.to(DEV)), og.embed_utterance(p, x)) < 1e-3
        assert _rel(m.embed_sequences(x.to(DEV), (h0.to(DEV), c0.to(DEV))), og.embed_sequences(p, x, (h0, c0))) < 1e-3
        loss_ref, sim_ref = og.forward(p, x, N)
        e = m.embed_sequences(x.to(DEV))
        assert _rel(m.similarity_matrix(e.reshape(N, -1, N)), sim_ref) < 1e-3
        loss, eer = m(x.to(DEV), N)
        assert abs(float(loss) - float(loss_ref)) < 1e-3 * abs(float(loss_ref))
        assert 0.0 <= eer <= 1.0
        pl, ps = og.loss(og.embed_sequences(p, x).reshape(N, M, -1), p["similarity_weight"], p["similarity_bias"])
        assert _rel(m.similarity_matrix(e.reshape(N, M, -1)), ps) < 1e-3


def test_embed_utterances_equals_per_utterance_calls():
    from oracle import ge2e as og
    m, p, cfg, _, seed = _model("shipped")
    counts = [3, 1, 7, 2, 5]
    parts = [og.synth_utterances(seed + i, n, 160, cfg[0]) for i, n in enumerate(counts)]
    batched = m.embed_utterances(parts)
    single = torch.stack([m.embed_utterance(q.to(DEV)) for q in parts])
    assert batched.shape == (len(counts), cfg[3])
    assert _rel(batched, single) < 1e-5


def test_recipe_shape_gradients_against_fp64_oracle():
    """Every parameter gradient of one step at the recipe shape (64 x 10 x 160 x 40, 3 x 256): the loss runs on (64, 40, 64)."""
    from oracle import ge2e as og
    from parakeet_b200.models import LSTMSpeakerEncoder
    from parakeet_b200.training import GE2ETrainStep
    p = og.synth_params(9, 40, 3, 256, 256)
    x = og.synth_utterances(10, 640, 160, 40)
    m = LSTMSpeakerEncoder(40, 3, 256, 256, device=DEV)
    m.set_state_dict(p)
    step = GE2ETrainStep(m, num_speakers=64)
    loss, _ = step.forward_backward(x.to(DEV))
    loss_ref, grads = og.train_grads(p, x, 64)
    assert abs(float(loss) - float(loss_ref)) < 1e-3 * abs(float(loss_ref))
    for k, gk in grads.items():
        if k == "similarity_bias":      # zero up to rounding (softmax rows sum to one)
            assert abs(float(step.grads[k])) < 1e-6
            continue
        assert _l2(step.grads[k], gk) < 5e-3, (k, _l2(step.grads[k], gk))


@pytest.mark.parametrize("clip", [3.0, 1e-3])
def test_three_step_clipped_adam_trajectory(clip):
    from oracle import ge2e as og
    from parakeet_b200.models import LSTMSpeakerEncoder
    from parakeet_b200.training import GE2ETrainStep
    cfg = (40, 3, 256, 256)
    p = og.synth_params(11, *cfg)
    m = LSTMSpeakerEncoder(*cfg, device=DEV)
    m.set_state_dict(p)
    step = GE2ETrainStep(m, learning_rate=1e-3, max_grad_norm=clip, num_speakers=4)
    ref, state, norms = {k: v.double() for k, v in p.items()}, {}, []
    for i in range(3):
        x = og.synth_utterances(20 + i, 20, 40, 40)
        step.step(x.to(DEV))
        _, grads = og.train_grads(ref, x, 4)
        ref, norm = og.clipped_adam_step(ref, grads, state, lr=1e-3, max_grad_norm=clip)
        norms.append(norm)
    if clip < 1:
        assert min(norms) > clip                       # the clip is active at every step
    for k, v in ref.items():
        got = m.state_dict()[k]
        assert _l2(got, v) < 1e-4, k                   # the parameters themselves, at the parity of the step's gradients
        delta = got - p[k].to(DEV)
        if k == "similarity_bias":
            # its gradient is zero up to rounding (each softmax row sums to one), so Adam's sign-like step has no defined direction
            # in either computation: only its size, three steps of at most lr, is pinned
            assert float(delta.abs().max()) <= 3.02e-3
            continue
        # Adam moves every weight by ~lr per step whatever the size of its gradient, so a weight whose gradient is within the
        # 5e-3 parity of zero may step either way: the update itself is compared at 5e-2 (the other steps' trajectory tests
        # allow 2e-2 to 0.1 for the same reason)
        assert _l2(delta, v - p[k].double()) < 5e-2, k


def test_graph_replay_equals_eager_and_steps_are_reproducible(monkeypatch, tmp_path):
    from oracle import ge2e as og
    from parakeet_b200.models import LSTMSpeakerEncoder
    from parakeet_b200.training import GE2ETrainStep
    cfg = (40, 3, 256, 256)
    p = og.synth_params(13, *cfg)
    xs = [og.synth_utterances(30 + i, 20, 50, 40).to(DEV) for i in range(4)]
    other = og.synth_utterances(40, 20, 31, 40).to(DEV)

    def run(graphs, n_steps, interleave=False):
        monkeypatch.setenv("PK_TRAIN_GRAPH", "1" if graphs else "0")
        m = LSTMSpeakerEncoder(*cfg, device=DEV)
        m.set_state_dict(p)
        # clip inactive: the global norm comes from FlatAdam's shared pk_sq_sum (per-block atomics in double), whose last bit
        # may differ between runs; everything the step itself computes is free of atomics
        st = GE2ETrainStep(m, max_grad_norm=1e9, num_speakers=4)
        losses = []
        for i in range(n_steps):
            losses.append(st.step(xs[i]))
            if interleave and i == 1:
                st.forward_backward_graphed(other)          # a different shape between two replays
        return m, st, torch.cat(losses)

    m_e, _, l_e = run(False, 4)
    m_g, _, l_g = run(True, 4, interleave=True)
    assert torch.equal(l_e, l_g)
    for k in p:
        assert torch.equal(m_e.state_dict()[k], m_g.state_dict()[k]), k
    m_e2, _, l_e2 = run(False, 4)
    assert torch.equal(l_e, l_e2)
    # checkpoint after two steps, resume in a fresh step, continue: equals the uninterrupted run
    m_a, st_a, _ = run(False, 2)
    st_a.save(str(tmp_path))
    m_b = LSTMSpeakerEncoder(*cfg, device=DEV)
    st_b = GE2ETrainStep(m_b, max_grad_norm=1e9, num_speakers=4)
    assert st_b.load(str(tmp_path)) == 2 and st_b.step_count == 2
    for i in (2, 3):
        st_b.step(xs[i])
    for k in p:
        assert torch.equal(m_b.state_dict()[k], m_e.state_dict()[k]), k


def test_unsupported_hidden_size_and_bad_grouping_raise_before_launch():
    from parakeet_b200.models import LSTMSpeakerEncoder
    with pytest.raises(ValueError):
        LSTMSpeakerEncoder(40, 3, 128, 256, device=DEV)
    m = LSTMSpeakerEncoder(40, 1, 64, 64, device=DEV)
    with pytest.raises(ValueError):
        m(torch.zeros(10, 5, 40, device=DEV), 3)
