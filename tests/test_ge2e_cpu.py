"""GE2E speaker encoder on the CPU: the oracle against vectors written by executing the reference's own LSTMSpeakerEncoder
(scripts/make_golden_ref.py ge2e), the oracle LSTM against torch.nn.LSTM, the forward's grouping hazard, state-dict keys, the
EER, the C ABI's argument checks, ptxas pins of the recurrence kernels and the persistent launch's scheduling argument."""
import os

import numpy as np
import pytest
import torch

import _ptxas

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_executed_ge2e.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


def _rel(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


@pytest.mark.parametrize("tag", ["small", "shipped"])
def test_oracle_equals_executed_reference(g, tag):
    from oracle import ge2e as og
    cfg, (N, M, T), seed = og.GOLDEN_CONFIGS[tag]
    p = og.synth_params(seed, *cfg)
    assert sorted(p) == sorted(g[f"{tag}/keys"].tolist())
    x = og.synth_utterances(seed + 100, N * M, T, cfg[0])
    assert np.array_equal(x.reshape(-1)[::97].numpy(), g[f"{tag}/x_sample"])
    with torch.no_grad():
        assert _rel(og.embed_sequences(p, x), g[f"{tag}/embeds"]) < 1e-5
        assert _rel(og.embed_utterance(p, x), g[f"{tag}/embed_reduce"]) < 1e-5
        h0, c0 = og.synth_states(seed + 200, cfg[1], N * M, cfg[2])
        assert _rel(og.embed_sequences(p, x, (h0, c0)), g[f"{tag}/embeds_init"]) < 1e-5
        loss, sim = og.forward(p, x, N)
        assert _rel(sim, g[f"{tag}/sim"]) < 1e-5
        assert abs(float(loss) - float(g[f"{tag}/loss"])) < 1e-5 * max(1.0, abs(float(g[f"{tag}/loss"])))
        pl, ps = og.loss(og.embed_sequences(p, x).reshape(N, M, -1), p["similarity_weight"], p["similarity_bias"])
        assert _rel(ps, g[f"{tag}/plain_sim"]) < 1e-5
        assert abs(float(pl) - float(g[f"{tag}/plain_loss"])) < 1e-5
    _, grads = og.train_grads(p, x, N)
    for k, gk in grads.items():
        flat = gk.reshape(-1)
        ref = g[f"{tag}/grad/{k}"]
        # similarity_bias' gradient is zero up to rounding (each softmax row sums to one): an absolute floor of 1e-8
        assert np.abs(flat[::max(1, flat.numel() // 1024)].numpy() - ref).max() <= 1e-4 * np.abs(ref).max() + 1e-8, k
        assert abs(float(flat.norm()) - float(g[f"{tag}/gradnorm/{k}"])) <= 1e-4 * float(g[f"{tag}/gradnorm/{k}"]) + 1e-8, k


def test_reference_eer_equals_numpy_eer(g):
    """The EER the reference computed with sklearn equals the package's numpy + scipy restatement on the same matrix."""
    from parakeet_b200.models.lstm_speaker_encoder import equal_error_rate
    for tag in ("small", "shipped"):
        sim = g[f"{tag}/sim"]
        N = sim.shape[1]
        assert abs(equal_error_rate(sim, N, sim.shape[0] // N) - float(g[f"{tag}/eer"])) < 1e-6


def test_numpy_roc_equals_sklearn():
    sk = pytest.importorskip("sklearn.metrics")
    from parakeet_b200.models.lstm_speaker_encoder import roc_curve
    rng = np.random.RandomState(3)
    for n in (30, 640, 4096):
        y = (rng.rand(n) < 0.1).astype(np.float32)
        s = np.round(rng.randn(n), 1).astype(np.float32)
        a, b = sk.roc_curve(y, s)[:2], roc_curve(y, s)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])


def test_oracle_lstm_equals_torch_lstm_fp64():
    from oracle import ge2e as og
    p = {k: v.double() for k, v in og.synth_params(5, 12, 2, 16, 8).items()}
    ref = torch.nn.LSTM(12, 16, 2, batch_first=True).double()
    with torch.no_grad():
        for l in range(2):
            for part in og.LSTM_PARTS:
                getattr(ref, f"{part}_l{l}").copy_(p[og.lstm_key(l, part)])
    x = torch.randn(3, 9, 12, dtype=torch.float64)
    h0, c0 = torch.randn(2, 3, 16, dtype=torch.float64), torch.randn(2, 3, 16, dtype=torch.float64)
    with torch.no_grad():
        out, (h, c) = og.lstm(p, x, h0, c0)
        out_r, (h_r, c_r) = ref(x, (h0, c0))
    for a, b in ((out, out_r), (h, h_r), (c, c_r)):
        assert torch.allclose(a, b, rtol=0, atol=1e-12)


def test_forward_grouping_differs_from_plain_and_oracle_follows_reference(g):
    """forward reshapes to [N, -1, N], not [N, M, C]: at the small config (4, 48, 4) vs (4, 3, 64) - different losses."""
    from oracle import ge2e as og
    assert abs(float(g["small/loss"]) - float(g["small/plain_loss"])) > 1e-3
    cfg, (N, M, T), seed = og.GOLDEN_CONFIGS["small"]
    assert g["small/sim"].shape == (N * (N * M * cfg[3] // (N * N)), N)
    assert g["small/plain_sim"].shape == (N * M, N)


def test_grouping_is_checked_before_any_launch():
    from parakeet_b200.models.lstm_speaker_encoder import LSTMSpeakerEncoder
    assert LSTMSpeakerEncoder.grouping(640, 256, 64) == 40                   # the recipe: (64, 40, 64)
    with pytest.raises(ValueError):
        LSTMSpeakerEncoder.grouping(10, 3, 4)                                # 30 not divisible by 16
    with pytest.raises(ValueError):
        LSTMSpeakerEncoder.grouping(4, 4, 4)                                 # M' = 1
    with pytest.raises(ValueError):
        LSTMSpeakerEncoder(40, 3, 128, 256, device="cpu")                    # no kernel for hidden 128


def test_loss_and_similarity_refuse_cpu_tensors_before_any_launch():
    from oracle import ge2e as og
    from parakeet_b200 import _lib
    from parakeet_b200.models.lstm_speaker_encoder import LSTMSpeakerEncoder
    m = LSTMSpeakerEncoder(40, 1, 64, 64, device="cpu")
    m.set_state_dict(og.synth_params(2, 40, 1, 64, 64))
    e = torch.randn(4, 3, 64)
    for fn in (m.loss, m.similarity_matrix):
        with pytest.raises(_lib.PkError):
            fn(e)
    with pytest.raises(_lib.PkError):
        m.embed_sequences(torch.randn(2, 5, 40))


def test_gate_permutation_puts_four_gates_of_a_unit_in_one_thread_fragment():
    """pk_lstm_fwd's accumulator fragment: thread lane holds columns 8 j + 2 (lane % 4) + {0, 1}; the packed row order puts gates
    i, f (j = 2p) and g, o (j = 2p + 1) of unit 4p + lane % 4 there, and is a permutation of W_hh's rows."""
    from parakeet_b200.ops import lstm_gate_perm
    for H in (64, 256):
        perm = lstm_gate_perm(H, "cpu")
        assert sorted(perm.tolist()) == list(range(4 * H))
        for s in range(H // 32):
            for q in range(4):
                cols = [8 * j + 2 * q + e for j in range(16) for e in range(2)]
                rows = [int(perm[128 * s + c]) for c in cols]
                units = {(r % H) for r in rows}
                assert len(units) == 8 and all(sorted(r // H for r in rows if r % H == u) == [0, 1, 2, 3] for u in units)


def test_both_key_forms_load_and_linear_layout_round_trips():
    from oracle import ge2e as og
    from parakeet_b200.models.lstm_speaker_encoder import LSTMSpeakerEncoder
    p = og.synth_params(1, 40, 2, 64, 32)
    m = LSTMSpeakerEncoder(40, 2, 64, 32, device="cpu")
    m.set_state_dict(p)
    for k, v in p.items():
        assert torch.equal(m.state_dict()[k], v), k
    assert tuple(m.state_dict()["linear.weight"].shape) == (64, 32)         # Paddle Linear [in, out]
    flat = {(f"lstm.{k.split('.')[3]}_l{k.split('.')[1]}" if k.startswith("lstm.") else k): v * 2 for k, v in p.items()}
    assert "lstm.weight_ih_l1" in flat
    m.set_state_dict(flat)
    for k, v in p.items():
        assert torch.equal(m.state_dict()[k], v * 2), k


def test_new_symbols_declared_and_rejected_arguments():
    from parakeet_b200 import _lib
    syms = _lib.exported_symbols()
    for s in ("pk_lstm_fwd", "pk_lstm_bwd", "pk_ge2e_loss", "pk_ge2e_loss_scratch", "pk_ge2e_embed_bwd", "pk_segment_mean_normalize"):
        assert s in syms
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    L = _lib.lib()
    assert L.pk_lstm_fwd(None, None, None, None, 64, 10, 256, None, None, None, None, 0, None, None, 0, None) == -1   # NULL pointers
    assert L.pk_lstm_fwd(None, None, None, None, 0, 10, 256, None, None, None, None, 0, None, None, 0, None) == -1    # no rows
    assert L.pk_lstm_fwd(None, None, 8, 8, 64, 10, 256, 8, 8, 8, 8, 0, None, 8, 640, None) == -1       # TMA operands misaligned
    assert L.pk_lstm_bwd(None, None, None, None, None, None, 64, 0, 256, None, None, None, None, None, 0, None) == -1
    assert L.pk_ge2e_loss(None, 4, 1, 8, None, None, None, 0, None, None, None, None, None, None) == -1      # M < 2
    assert L.pk_ge2e_loss_scratch(64, 40, 64) > 64 * 40 * 64 * 4


@pytest.mark.parametrize("rows,hidden,max_ctas", [(1, 256, 132), (640, 256, 132), (6000, 256, 132), (65, 64, 132), (640, 256, 7),
                                                  (640, 256, 8), (64 * 17, 256, 132)])
def test_scheduling_argument(rows, hidden, max_ctas):
    """Restated from csrc/lstm.cu: every (tile, slice) of a step is served by exactly one CTA, the grid never exceeds what the
    occupancy query says is co-resident, and CTAs only wait on counters of the previous step - which every CTA finishes before
    starting its own next step, so (by induction over steps) no wait can be on a CTA that has not started."""
    from parakeet_b200.ops import lstm_schedule
    slices, tiles, groups, grid = lstm_schedule(rows, hidden, max_ctas)
    if max_ctas < slices:
        assert grid == 0                     # refused with an error code rather than launched
        return
    assert 0 < grid <= max_ctas and grid == groups * slices
    served = {}
    for b in range(grid):
        s, grp = b % slices, b // slices
        for m in range(grp, tiles, groups):
            served[(m, s)] = served.get((m, s), 0) + 1
    assert served == {(m, s): 1 for m in range(tiles) for s in range(slices)}


@_ptxas.needs_nvcc
@pytest.mark.parametrize("kernel", ["lstm_fwd_kernelILi256E", "lstm_bwd_kernelILi256E", "lstm_fwd_kernelILi64E", "lstm_bwd_kernelILi64E",
                                    "ge2e_loss_kernel"])
def test_recurrence_kernels_do_not_spill(kernel):
    rep = _ptxas.report("lstm.cu")
    e = _ptxas.entry(rep, kernel)
    assert (e["spill_stores"], e["spill_loads"]) == (0, 0), e
    assert not any(x["codes"] & _ptxas.SERIALIZED for x in rep["entries"]), rep["entries"]
