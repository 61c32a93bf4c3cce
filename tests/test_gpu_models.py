"""GPU parity tests of the model-level path (FastSpeech2, Parallel WaveGAN) against the oracle and golden vectors."""
import math
import os

import numpy as np
import pytest
import torch

from conftest import rel_err

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
TOL = 1e-3   # north_star: "within 1e-3 rel fp32" (max-abs error / max-abs reference per tensor)


@pytest.fixture(scope="module")
def pwg(cuda):
    from oracle import pwg as opwg
    from parakeet_b200.models import PWGGenerator
    params = opwg.synth_params(2, weight_norm=True)
    gen = PWGGenerator(**opwg.DEFAULT_GENERATOR_PARAMS, device=cuda)
    gen.set_state_dict(params)
    return gen, opwg.fold_weight_norm(params)


@pytest.fixture(scope="module")
def fs2(cuda):
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2
    params = ofs.synth_params(1)
    m = FastSpeech2(80, 80, **ofs.LJSPEECH_MODEL_CFG, device=cuda)
    m.set_state_dict(params)
    return m, params


def test_pwg_golden(cuda, pwg):
    gen, _ = pwg
    g = np.load(os.path.join(GOLD, "pwg_small.npz"))
    y = gen(torch.from_numpy(g["x"]).to(cuda), torch.from_numpy(g["c"]).to(cuda))
    assert rel_err(y, torch.from_numpy(g["y"])) < TOL


def test_pwg_upsample_and_generator_vs_oracle(cuda, pwg):
    from oracle import pwg as opwg
    gen, folded = pwg
    x, c = opwg.synth_inputs(5, batch=2, mel_frames=40)
    with torch.no_grad():
        y_ref, inter = opwg.generator_forward(folded, x, c, return_intermediates=True)
    assert rel_err(gen.upsample(c.to(cuda)), inter["c_up"]) < 1e-5
    y = gen(x.to(cuda), c.to(cuda))
    assert rel_err(gen._last_x.float().transpose(1, 2), inter["x_layers"][-1]) < TOL
    assert rel_err(y, y_ref) < TOL
    # reference API: inference(c) with caller-supplied noise (RNG streams cannot match, SURVEY.md 7)
    mel, noise = torch.randn(30, 80), torch.randn(1, 1, 30 * 300)
    with torch.no_grad():
        r = opwg.generator_inference(folded, mel, noise)
    assert rel_err(gen.inference(mel.to(cuda), x=noise.to(cuda)), r) < TOL


def test_pwg_ragged_batch_equals_single_utterances(cuda, pwg):
    from oracle import pwg as opwg
    gen, folded = pwg
    frames, hop = [40, 25, 33], 300
    xs = torch.zeros(3, 1, max(frames) * hop)
    cs = torch.zeros(3, 80, max(frames) + 4)
    refs = []
    for i, f in enumerate(frames):
        xi, ci = opwg.synth_inputs(10 + i, batch=1, mel_frames=f)
        xs[i, :, :f * hop], cs[i, :, :f + 4] = xi[0], ci[0]
        with torch.no_grad():
            refs.append(opwg.generator_forward(folded, xi, ci)[0])
    lens = torch.tensor([f * hop for f in frames], dtype=torch.int32, device=cuda)
    y = gen(xs.to(cuda), cs.to(cuda), lens=lens)
    for i, f in enumerate(frames):
        assert rel_err(y[i, :, :f * hop], refs[i]) < TOL


def test_pwg_ragged_batch_graph_replay_and_empty_utterance(cuda, pwg):
    """A ragged batch holding an EMPTY utterance, run three times (eager, CUDA-graph capture, replay): every call reproduces the
    single-utterance oracle results, the empty row stays zero, and a different set of lengths of the same padded shape (another
    graph key, other band-table end blocks) is not confused with the first."""
    from oracle import pwg as opwg
    gen, folded = pwg
    hop = 300

    def make(frames, seed):
        xs = torch.zeros(len(frames), 1, 40 * hop)
        cs = torch.zeros(len(frames), 80, 44)
        refs = []
        for i, f in enumerate(frames):
            if f == 0:
                refs.append(None)
                continue
            xi, ci = opwg.synth_inputs(seed + i, batch=1, mel_frames=f)
            xs[i, :, :f * hop], cs[i, :, :f + 4] = xi[0], ci[0]
            with torch.no_grad():
                refs.append(opwg.generator_forward(folded, xi, ci)[0])
        return xs.to(cuda), cs.to(cuda), torch.tensor([f * hop for f in frames], dtype=torch.int32, device=cuda), refs
    for frames, seed in (([40, 0, 33], 30), ([21, 40, 1], 40)):
        xs, cs, lens, refs = make(frames, seed)
        replays0 = gen._graphs.replays
        for call in range(3):
            y = gen(xs, cs, lens=lens)
            for i, f in enumerate(frames):
                if f == 0:
                    assert y[i].abs().max().item() == 0
                else:
                    assert rel_err(y[i, :, :f * hop], refs[i]) < TOL, (frames, call, i)
                    assert y[i, :, f * hop:].abs().max().item() == 0 if f < 40 else True
        assert gen._graphs.replays > replays0


def test_pwg_full_size_properties(cuda, pwg):
    """cfg2 (B=32, 400 frames -> 3.84 M samples): batch independence + determinism + one utterance vs the oracle."""
    from oracle import pwg as opwg
    gen, folded = pwg
    x, c = opwg.synth_inputs(2, batch=32, mel_frames=400)
    x, c = x.to(cuda), c.to(cuda)
    y = gen(x, c).clone()
    assert torch.isfinite(y).all()
    assert torch.equal(gen(x, c), y)                               # deterministic
    y1 = gen(x[7:8].contiguous(), c[7:8].contiguous())             # utterance 7 alone == inside the batch, bit for bit
    assert torch.equal(y1[0], y[7])
    with torch.no_grad():
        r = opwg.generator_forward(folded, x[:1, :, :24000].cpu().contiguous(), c[:1, :, :84].cpu().contiguous())
    # the first 80 frames minus the receptive field (3069 samples + upsampling halo) are independent of the truncation
    n = 24000 - 3069 - 600
    assert rel_err(y[0, :, :n], r[0, :, :n]) < TOL


def test_fs2_golden(cuda, fs2):
    m, _ = fs2
    g = np.load(os.path.join(GOLD, "fs2_infer_small.npz"))
    out = m.inference(torch.from_numpy(g["text"])[0].to(cuda))
    assert out.shape[0] == int(g["durations"].sum())               # integer durations: exact
    assert rel_err(out, torch.from_numpy(g["after"][0])) < TOL
    g = np.load(os.path.join(GOLD, "fs2_forward_small.npz"))
    b = {k: torch.from_numpy(g[k]).to(cuda) for k in ("text", "text_lengths", "speech", "speech_lengths", "durations", "pitch", "energy")}
    o = m(b["text"], b["text_lengths"], b["speech"], b["speech_lengths"], b["durations"], b["pitch"], b["energy"])
    for name, t in zip(("before", "after", "d_outs", "p_outs", "e_outs"), o[:5]):
        assert rel_err(t, torch.from_numpy(g[name])) < TOL, name


def test_fs2_cfg1_and_batched_inference_vs_oracle(cuda, fs2):
    from oracle import fastspeech2 as ofs
    m, params = fs2
    xs, il = ofs.synth_text(1, [100])                              # cfg1: single utterance, 100 phonemes
    with torch.no_grad():
        _, a_ref, d_ref, p_ref, e_ref = ofs.fs2_forward(params, None, xs, il, is_inference=True)
    before, after, d, p, e, olens = m._forward(xs.to(cuda), il.to(cuda), is_inference=True)
    assert torch.equal(d.cpu(), d_ref)                             # bit-exact integer durations
    assert int(olens[0]) == a_ref.shape[1]
    assert rel_err(after, a_ref) < TOL and rel_err(p, p_ref) < TOL and rel_err(e, e_ref) < TOL
    # speed control (alpha != 1): durations re-rounded half away from zero
    with torch.no_grad():
        _, a2, d2, _, _ = ofs.fs2_forward(params, None, xs, il, is_inference=True, alpha=1.3)
    out = m.inference(xs[0].to(cuda), alpha=1.3)
    assert out.shape[0] == a2.shape[1] and rel_err(out, a2[0]) < TOL
    # ragged batch: every utterance identical to decoding it alone
    lengths = [60, 100, 83, 140]
    xs, il = ofs.synth_text(7, lengths)
    mel, olens, _ = m.batch_inference(xs.to(cuda), il.to(cuda))
    for i, n in enumerate(lengths):
        with torch.no_grad():
            r = ofs.fs2_inference(params, None, xs[i, :n])
        L = int(olens[i])
        assert L == r.shape[0]
        assert rel_err(mel[i, :L], r) < TOL
        assert L == mel.shape[1] or mel[i, L:].abs().max().item() == 0


def test_fs2_full_batch_properties(cuda, fs2):
    """cfg3-sized FS2 (32 utterances, T ~ U{60..140}): batch independence without the oracle."""
    from oracle import fastspeech2 as ofs
    m, _ = fs2
    g = torch.Generator().manual_seed(3)
    lengths = torch.randint(60, 141, (32,), generator=g).tolist()
    xs, il = ofs.synth_text(3, lengths)
    mel, olens, d = m.batch_inference(xs.to(cuda), il.to(cuda))
    assert torch.isfinite(mel).all() and (d >= 0).all()
    assert olens.cpu().tolist() == d.sum(1).to(torch.int64).cpu().tolist()
    for i in (0, 13, 31):
        single = m.inference(xs[i, :lengths[i]].to(cuda))
        assert single.shape[0] == int(olens[i])
        assert rel_err(mel[i, :single.shape[0]], single) < 1e-5


def test_zscore_and_inference_wrappers(cuda, fs2, pwg):
    from parakeet_b200.models import FastSpeech2Inference, PWGInference
    from parakeet_b200.modules.normalizer import ZScore
    m, _ = fs2
    gen, _ = pwg
    mu, sigma = torch.randn(80), torch.rand(80) + 0.5
    norm = ZScore(mu, sigma, device=cuda)
    text = torch.randint(1, 79, (20,)).to(cuda)
    mel_n = m.inference(text)
    logmel = FastSpeech2Inference(norm, m)(text)
    assert rel_err(logmel, mel_n.cpu() * sigma + mu) < 1e-6
    noise = torch.randn(1, 1, logmel.shape[0] * 300, device=cuda)
    wav = PWGInference(norm, gen)(logmel, x=noise)
    assert list(wav.shape) == [logmel.shape[0] * 300, 1] and torch.isfinite(wav).all()
    assert rel_err(wav, gen.inference(mel_n, x=noise)) < 1e-4


def test_waveflow_inference_vs_oracle(cuda):
    """cfg4 architecture (64 channels, 8 flows x 8 layers, n_group 16, upsample 16x16) at a small size, caller-supplied z."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(4)
    m = ConditionalWaveFlow([16, 16], 8, 8, 16, 64, 80, (3, 3), device=cuda)
    m.set_state_dict(params)
    folded = owf.fold_weight_norm(params)
    g = torch.Generator().manual_seed(4)
    mel = torch.randn(2, 80, 9, generator=g) * 0.5 - 3
    cond_ref = owf.encoder(folded, mel, 2)
    assert list(cond_ref.shape) == [2, 80, 256 * 9 - 272]
    assert rel_err(m.encode(mel.to(cuda)), cond_ref) < 1e-5
    z = torch.randn(2, cond_ref.shape[-1], generator=g)
    with torch.no_grad():
        ref = owf.infer(folded, mel, z)
    out = m.infer(mel.to(cuda), z=z.to(cuda))
    assert list(out.shape) == list(ref.shape)
    assert rel_err(out, ref) < TOL


def test_waveflow_wide_rows_vs_oracle(cuda):
    """W = 431 columns (28 mel frames): every width dilation up to 128 reaches live columns on both sides; odd batch."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(4)
    m = ConditionalWaveFlow([16, 16], 8, 8, 16, 64, 80, (3, 3), device=cuda)
    m.set_state_dict(params)
    folded = owf.fold_weight_norm(params)
    g = torch.Generator().manual_seed(41)
    mel = torch.randn(3, 80, 28, generator=g) * 0.5 - 3
    z = torch.randn(3, 256 * 28 - 272, generator=g)
    with torch.no_grad():
        ref = owf.infer(folded, mel, z)
    out = m.infer(mel.to(cuda), z=z.to(cuda))
    assert list(out.shape) == list(ref.shape) and rel_err(out, ref) < TOL


@pytest.mark.parametrize("channels", [64, 128])
def test_waveflow_two_gemm_path_vs_oracle(cuda, channels):
    """n_mels = 64 is outside the fused kernels' range, so inverse runs the two-GEMM row loop (pk_conv_gemm_ex with the gate and
    wf_update epilogues, N = 2C gate channels, K = 3C per tap); W = 431 columns so that every width dilation reaches live
    columns; odd batch."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(6, channels=channels, n_mels=64)
    folded = owf.fold_weight_norm(params)
    m = ConditionalWaveFlow([16, 16], 8, 8, 16, channels, 64, (3, 3), device=cuda)
    m.set_state_dict(params)
    assert not m._eligible()
    g = torch.Generator().manual_seed(43)
    mel = torch.randn(3, 64, 28, generator=g) * 0.5 - 3
    z = torch.randn(3, 256 * 28 - 272, generator=g)
    with torch.no_grad():
        ref = owf.infer(folded, mel, z)
    out = m.infer(mel.to(cuda), z=z.to(cuda))
    assert list(out.shape) == list(ref.shape) and rel_err(out, ref) < TOL


def test_waveflow_shipped_config_128_channels(cuda):
    """examples/waveflow/config.py ships channels = 128 (BASELINE cfg 4 is the 64-channel variant): the flow kernel runs the
    channels as two blocks of 64 (N = 256 MMAs); W = 431 columns so that every width dilation reaches live columns."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(5, channels=128)
    folded = owf.fold_weight_norm(params)
    g = torch.Generator().manual_seed(55)
    mel = torch.randn(3, 80, 28, generator=g) * 0.5 - 3
    z = torch.randn(3, 256 * 28 - 272, generator=g)
    with torch.no_grad():
        ref = owf.infer(folded, mel, z)
    m = ConditionalWaveFlow([16, 16], 8, 8, 16, 128, 80, (3, 3), device=cuda)
    m.set_state_dict(params)
    assert m._eligible()
    out = m.infer(mel.to(cuda), z=z.to(cuda))
    assert list(out.shape) == list(ref.shape) and rel_err(out, ref) < TOL


@pytest.mark.parametrize("channels", [64, 128])
def test_waveflow_flow_kernel_single_utterance_and_edges(cuda, channels):
    """pk_waveflow_flow scheduling corners: one utterance with a single tile per step (every tile depends on the pair's own
    previous tile: unpipelined issue order), two tiles per step, and a width just past a tile boundary (271 columns)."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(4, channels=channels)
    folded = owf.fold_weight_norm(params)
    m = ConditionalWaveFlow([16, 16], 8, 8, 16, channels, 80, (3, 3), device=cuda)
    m.set_state_dict(params)
    assert m._eligible()
    for batch, frames, seed in ((1, 9, 51), (1, 18, 52), (2, 18, 53)):     # W = 127, 271, 271
        g = torch.Generator().manual_seed(seed)
        mel = torch.randn(batch, 80, frames, generator=g) * 0.5 - 3
        z = torch.randn(batch, 256 * frames - 272, generator=g)
        with torch.no_grad():
            ref = owf.infer(folded, mel, z)
        out = m.infer(mel.to(cuda), z=z.to(cuda))
        assert rel_err(out, ref) < TOL, (batch, frames)


def test_waveflow_cfg4_full_size_properties(cuda):
    """cfg4 (B=16, 400 mel frames -> 16 x 102 128 samples, W = 6383): batch independence bit for bit, determinism / graph
    replay == eager, and one whole utterance against the oracle (mirror of test_pwg_full_size_properties)."""
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    params = owf.synth_params(4)
    m = ConditionalWaveFlow([16, 16], 8, 8, 16, 64, 80, (3, 3), device=cuda)
    m.set_state_dict(params)
    folded = owf.fold_weight_norm(params)
    g = torch.Generator().manual_seed(42)
    mel = (torch.randn(16, 80, 400, generator=g) * 0.5 - 3).to(cuda)
    t_c = 256 * 400 - 272
    z = torch.randn(16, t_c, generator=g).to(cuda)
    y0 = m.infer(mel, z=z).clone()                                  # eager
    assert list(y0.shape) == [16, t_c // 16 * 16] and torch.isfinite(y0).all()
    y1 = m.infer(mel, z=z).clone()                                  # capture
    y2 = m.infer(mel, z=z).clone()                                  # replay
    assert m._graphs.replays >= 1
    assert torch.equal(y0, y1) and torch.equal(y0, y2)
    one = m.infer(mel[5:6].contiguous(), z=z[5:6].contiguous())     # utterance 5 alone == inside the batch
    assert torch.equal(one[0], y0[5])
    # one whole utterance against the oracle (the row recurrence spreads every input over the full width, so a truncated
    # oracle run is not comparable; the full-width run costs ~1 TFLOP on the host)
    with torch.no_grad():
        ref = owf.infer(folded, mel[:1].cpu(), z[:1].cpu())
    assert rel_err(y0[0], ref[0]) < TOL


def test_fs2_loss_vs_oracle(cuda, fs2):
    """FastSpeech2Loss (use_masking=True) on the teacher-forced forward of the golden batch."""
    from oracle import fastspeech2 as ofs
    from parakeet_b200.models import FastSpeech2Loss
    m, params = fs2
    g = np.load(os.path.join(GOLD, "fs2_forward_small.npz"))
    b = {k: torch.from_numpy(g[k]).to(cuda) for k in ("text", "text_lengths", "speech", "speech_lengths", "durations", "pitch", "energy")}
    before, after, d_outs, p_outs, e_outs, ys, olens = m(b["text"], b["text_lengths"], b["speech"], b["speech_lengths"],
                                                          b["durations"], b["pitch"], b["energy"])
    losses = FastSpeech2Loss(device=cuda)(after, before, d_outs, p_outs, e_outs, ys, b["durations"], b["pitch"], b["energy"],
                                          b["text_lengths"], olens)
    got = [float(v) for v in losses]
    assert np.allclose(got, g["losses"], rtol=1e-3), (got, g["losses"])


def test_cuda_graph_replay_matches_eager(cuda, fs2):
    """The launch-bound inference paths replay as CUDA graphs from their third call on (parakeet_b200/graph.py): the
    replays must reproduce the eager result bit for bit, for new inputs of the same shape, and a weight update must drop
    the captured graphs."""
    from oracle import fastspeech2 as ofs
    from oracle import waveflow as owf
    from parakeet_b200.models import ConditionalWaveFlow
    m, params = fs2
    lengths = [50, 77, 64]
    outs = []
    for seed in (11, 12, 13, 11):                                   # eager, capture, replay, replay with the first inputs
        xs, il = ofs.synth_text(seed, lengths)
        mel, olens, d = m.batch_inference(xs.to(cuda), il.to(cuda))
        outs.append((mel.clone(), olens.clone(), d.clone()))
    assert m._graphs.replays >= 2
    assert torch.equal(outs[0][0], outs[3][0]) and torch.equal(outs[0][1], outs[3][1]) and torch.equal(outs[0][2], outs[3][2])
    xs, il = ofs.synth_text(13, lengths)
    for i, n in enumerate(lengths):                                 # a replayed result against the oracle
        with torch.no_grad():
            r = ofs.fs2_inference(params, None, xs[i, :n])
        L = int(outs[2][1][i])
        assert L == r.shape[0] and rel_err(outs[2][0][i, :L], r) < TOL
    n_graphs = len(m._graphs._graphs)
    assert n_graphs >= 1
    m.set_state_dict(m.state_dict())                                # invalidates the packed weights -> graphs dropped
    assert len(m._graphs._graphs) == 0

    wf = ConditionalWaveFlow([16, 16], 8, 8, 16, 64, 80, (3, 3), device=cuda)
    wp = owf.synth_params(4)
    wf.set_state_dict(wp)
    g = torch.Generator().manual_seed(5)
    res = []
    for it in range(3):
        mel = torch.randn(2, 80, 6, generator=g) * 0.5 - 3
        z = torch.randn(2, 256 * 6 - 272, generator=g)
        res.append((mel, z, wf.infer(mel.to(cuda), z=z.to(cuda))))
    assert wf._graphs.replays >= 1
    with torch.no_grad():
        ref = owf.infer(owf.fold_weight_norm(wp), res[2][0], res[2][1])
    assert rel_err(res[2][2], ref) < TOL
