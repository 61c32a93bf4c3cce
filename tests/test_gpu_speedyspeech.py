"""SpeedySpeech on the GPU: the fused residual-block kernel (pk_ss_residual_block) against the oracle, the model against the
vectors the reference's own code produced and against the oracle at the shipped config, batch independence, graph replay, the
chain into Parallel WaveGAN, and the all-zero-durations corner."""
import os

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL = 1e-3
GOLD = os.path.join(os.path.dirname(__file__), "golden", "ref_executed_speedyspeech.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLD)


def _model(cuda, cfg, seed, tone_size=None, **kw):
    from oracle import speedyspeech as oss
    from parakeet_b200.models import SpeedySpeech
    params = oss.synth_params(seed, cfg, tone_size=tone_size, **kw)
    m = SpeedySpeech(40, tone_size=tone_size, device=cuda, **cfg)
    m.set_state_dict(params)
    return m.eval(), params


# ------------------------------------------------------------------------------------------------ the kernel alone
def _block_params(seed, k, n, C=128):
    gen = torch.Generator().manual_seed(seed)
    p = {}
    for j in range(n):
        q = f"blk.blocks.{j}."
        p[q + "0.weight"] = (torch.rand(C, C, k, generator=gen) * 2 - 1) / (C * k) ** 0.5
        p[q + "0.bias"] = (torch.rand(C, generator=gen) * 2 - 1) * 0.1
        p[q + "2.weight"] = 0.5 + torch.rand(C, generator=gen)
        p[q + "2.bias"] = (torch.rand(C, generator=gen) * 2 - 1) * 0.2
        p[q + "2._mean"] = torch.rand(C, generator=gen) * 0.5
        p[q + "2._variance"] = 0.5 + torch.rand(C, generator=gen)
    return p


@pytest.mark.parametrize("n,k", [(1, 1), (1, 3), (1, 4), (2, 3)])
@pytest.mark.parametrize("lengths,use_lens", [([1], False), ([2], False), ([300], False), ([1], True), ([2], True), ([300], True),
                                              ([300, 131, 7], True)])
def test_residual_block_kernel_vs_oracle(cuda, n, k, lengths, use_lens):
    """T = 1, 2 and 300 (not a multiple of the 126- or 128-row tile); batch 3 with ragged lengths."""
    from oracle import speedyspeech as oss
    from parakeet_b200 import ops
    from parakeet_b200.models.speedyspeech import BN_EPS, paddle_same_conv
    p = _block_params(10 * n + k, k, n)
    B, T = len(lengths), max(lengths)
    x = torch.randn(B, T, 128, generator=torch.Generator().manual_seed(T))
    for b, L in enumerate(lengths):
        x[b, L:] = 0                                       # the kernel's precondition under lens
    convs = []
    for j in range(n):
        q = f"blk.blocks.{j}."
        s = p[q + "2.weight"] / torch.sqrt(p[q + "2._variance"] + BN_EPS)
        convs.append(dict(w=ops.pack_weight(p[q + "0.weight"], cuda), b=p[q + "0.bias"].to(cuda),
                          s=s.to(cuda), t=(p[q + "2.bias"] - p[q + "2._mean"] * s).to(cuda)))
    xd = x.to(cuda)
    lens = torch.tensor(lengths, dtype=torch.int32, device=cuda) if use_lens else None
    y, ys = ops.ss_residual_block(xd, ops.Split.from_f32(xd), convs, k, paddle_same_conv(k, 1)[1], lens)
    with torch.no_grad():
        want = torch.zeros_like(x)
        for b, L in enumerate(lengths):
            want[b, :L] = oss.residual_block(p, "blk.", x[b:b + 1, :L], 1, n)[0]
    assert rel_err(y, want) < TOL
    assert rel_err(ys.float(), want) < TOL
    for b, L in enumerate(lengths):
        if use_lens:
            assert y[b, L:].abs().sum() == 0 and ys.hi[b, L:].float().abs().sum() == 0      # zero rows past each length


# ------------------------------------------------------------------------------------------------ the model
def test_model_vs_executed_reference(cuda, g):
    from oracle import speedyspeech as oss
    from parakeet_b200.models import SpeedySpeechInference
    from parakeet_b200.modules.normalizer import ZScore
    m, _ = _model(cuda, oss.SMALL_CFG, 6, tone_size=7)
    text, tones = torch.from_numpy(g["small_inf_text"]).to(cuda), torch.from_numpy(g["small_inf_tones"]).to(cuda)
    mel = m.inference(text)
    assert mel.shape == g["small_inf_mel"].shape and rel_err(mel, torch.from_numpy(g["small_inf_mel"])) < TOL
    mel = m.inference(text, tones)
    assert mel.shape == g["small_inf_tone_mel"].shape and rel_err(mel, torch.from_numpy(g["small_inf_tone_mel"])) < TOL
    norm = ZScore(torch.from_numpy(g["small_wr_mu"]), torch.from_numpy(g["small_wr_sigma"]), device=cuda)
    logmel = SpeedySpeechInference(norm, m)(text, tones)
    assert logmel.shape == g["small_wr_logmel"].shape and rel_err(logmel, torch.from_numpy(g["small_wr_logmel"])) < TOL
    dec, pred = m(torch.from_numpy(g["small_fwd_text"]).to(cuda), torch.from_numpy(g["small_fwd_tones"]).to(cuda),
                  torch.from_numpy(g["small_fwd_durations"]).to(cuda))
    assert dec.shape == g["small_fwd_decoded"].shape and rel_err(dec, torch.from_numpy(g["small_fwd_decoded"])) < TOL
    assert rel_err(pred, torch.from_numpy(g["small_fwd_pred_durations"])) < TOL
    m2, _ = _model(cuda, oss.SHIPPED_CFG, 7)
    mel = m2.inference(torch.from_numpy(g["shipped_inf_text"]).to(cuda))
    assert mel.shape == g["shipped_inf_mel"].shape and rel_err(mel, torch.from_numpy(g["shipped_inf_mel"])) < TOL


def test_shipped_config_vs_oracle_long_utterance(cuda):
    """The baker yaml (10 + 18 blocks) at 140 phonemes, about 1 000 frames: durations exact, mel to tolerance."""
    from oracle import speedyspeech as oss
    m, params = _model(cuda, oss.SHIPPED_CFG, 11, tone_size=5, log_duration=1.95)
    gen = torch.Generator().manual_seed(140)
    text, tones = torch.randint(1, 40, (140,), generator=gen), torch.randint(1, 5, (140,), generator=gen)
    with torch.no_grad():
        _, d_ref = oss.inference_durations(params, oss.SHIPPED_CFG, text, tones)
        want = oss.inference(params, oss.SHIPPED_CFG, text, tones)
    assert 800 <= want.shape[0] <= 1200, want.shape
    mel, frames, d = m.batch_inference(text[None].to(cuda), torch.tensor([140]).to(cuda), tones[None].to(cuda))
    assert torch.equal(d.cpu(), d_ref) and int(frames[0]) == want.shape[0]
    assert rel_err(mel[0], want) < TOL


def test_batch_inference_equals_per_utterance_inference(cuda):
    from oracle import speedyspeech as oss
    m, _ = _model(cuda, oss.SMALL_CFG, 9, tone_size=7)
    gen = torch.Generator().manual_seed(3)
    lengths = [31, 7, 60, 1]
    text = torch.zeros(4, 60, dtype=torch.int64)
    tones = torch.zeros(4, 60, dtype=torch.int64)
    for i, n in enumerate(lengths):
        text[i, :n] = torch.randint(1, 40, (n,), generator=gen)
        tones[i, :n] = torch.randint(1, 7, (n,), generator=gen)
    mel, frames, d = m.batch_inference(text.to(cuda), torch.tensor(lengths).to(cuda), tones.to(cuda))
    assert mel.shape[0] == 4 and mel.shape[1] == int(frames.max())
    for i, n in enumerate(lengths):
        one = m.inference(text[i, :n].to(cuda), tones[i, :n].to(cuda))
        L = int(frames[i])
        assert one.shape[0] == L
        assert torch.equal(mel[i, :L], one), i                   # bit for bit
        assert mel[i, L:].abs().sum() == 0
        assert int(d[i, n:].abs().sum()) == 0


def test_graph_replay_equals_eager(cuda):
    from oracle import speedyspeech as oss
    m, _ = _model(cuda, oss.SMALL_CFG, 11)
    text = torch.randint(1, 40, (50,), generator=torch.Generator().manual_seed(5)).to(cuda)
    first = m.inference(text)                # eager
    second = m.inference(text)               # captured
    third = m.inference(text)                # replayed
    assert m._graphs.replays >= 2
    assert torch.equal(first, second) and torch.equal(first, third)


def test_speedyspeech_to_pwg_end_to_end_vs_oracle_chain(cuda):
    from oracle import pwg as opwg
    from oracle import speedyspeech as oss
    from parakeet_b200.models import PWGGenerator, PWGInference, SpeedySpeechInference
    from parakeet_b200.modules.normalizer import ZScore
    m, params = _model(cuda, oss.SMALL_CFG, 12, tone_size=7, log_duration=0.5)
    gp = opwg.synth_params(2, weight_norm=True)
    gen = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device=cuda)
    gen.set_state_dict(gp)
    rg = torch.Generator().manual_seed(13)
    mu_s, sig_s = torch.randn(80, generator=rg) * 0.2, torch.rand(80, generator=rg) + 0.5
    mu_p, sig_p = torch.randn(80, generator=rg) * 0.2, torch.rand(80, generator=rg) + 0.5
    text, tones = torch.randint(1, 40, (9,), generator=rg), torch.randint(1, 7, (9,), generator=rg)
    logmel = SpeedySpeechInference(ZScore(mu_s, sig_s, device=cuda), m)(text.to(cuda), tones.to(cuda))
    noise = torch.randn(1, 1, logmel.shape[0] * 300, generator=rg)
    wav = PWGInference(ZScore(mu_p, sig_p, device=cuda), gen)(logmel, x=noise.to(cuda))
    with torch.no_grad():
        want_mel = oss.inference_denorm(params, oss.SMALL_CFG, text, tones, mu_s, sig_s)
        want = opwg.pwg_inference(opwg.fold_weight_norm(gp), want_mel, mu_p, sig_p, noise)
    assert logmel.shape == want_mel.shape and rel_err(logmel, want_mel) < TOL
    assert wav.shape == want.shape and rel_err(wav, want) < TOL


def test_all_zero_durations_give_empty_output(cuda):
    from oracle import speedyspeech as oss
    m, _ = _model(cuda, oss.SMALL_CFG, 14, log_duration=-10.0)
    text = torch.randint(1, 40, (2, 12), generator=torch.Generator().manual_seed(1)).to(cuda)
    mel, frames, d = m.batch_inference(text, torch.tensor([12, 5]).to(cuda))
    assert tuple(mel.shape) == (2, 0, 80) and int(frames.abs().sum()) == 0 and int(d.abs().sum()) == 0
    assert tuple(m.inference(text[0]).shape) == (0, 80)
    dec, pred = m(text, None, torch.zeros(2, 12, dtype=torch.int64))
    assert tuple(dec.shape) == (2, 0, 80) and tuple(pred.shape) == (2, 12)
