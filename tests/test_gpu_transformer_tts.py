"""TransformerTTS on the GPU: inference, teacher-forced inference and the eval forward against the reference's own code executed
on the Paddle stand-in (tests/golden/ref_executed_transformer_tts.npz); the persistent decoder against the fp64 oracle at every step
over encoder lengths, reduction factors and a run past 1000 steps; the stop step at a threshold placed from the fp64 trajectory;
forward fed inference's own frames; CUDA-graph replay; the seed contract.

Error budget of pk_tts_decode against the fp64 oracle (bound 2e-4 of the tensor's max |value|):
  * inputs of the decoder come from split-bf16 GEMMs (the encoder, the source K / V): 3 bf16 passes drop only lo x lo, so each
    product is exact to ~2^-16 x 2^-16 relative, and the fp32 accumulation over K <= 1024 terms adds <= 1024 x 2^-24 ~ 6e-5
    relative to the sum of |terms| (a worst case; a random-sign sum is ~sqrt(K) x 2^-24 ~ 2e-6);
  * the decoder's fp32 dot products (K <= 1024) add the same ~2e-6 typical, 6e-5 worst, per matrix-vector product;
  * a step chains 2 prenet + 1 input + 8 per layer (LayerNorm renormalises the row) products: with LayerNorm before every
    sub-layer, the per-layer errors add, ~ (2 + 1 + 8 L) x 2e-6 ~ 1e-4 typical at L = 6, 5e-5 at L = 3;
  * the feedback of frame t into step t + 1 goes through the prenet ReLU / dropout and a 1 / sqrt(fan_in)-scaled Linear, so a
    frame error enters the next step at the same relative size; the bound is checked at every step, so growth would show.
So 2e-4 sits at about 2 x the typical accumulated rounding; an index, mask, cache-row or tap error gives errors of order 1e-1.
The whole-model comparison with the reference's fp32 output uses the 1e-3 relative bound of the other models (the reference's
own fp32 rounding is of the same order as ours)."""
import numpy as np
import pytest
import torch

import oracle.transformer_tts as ot
from parakeet_b200 import ops
from parakeet_b200.models import TransformerTTS, TransformerTTSInference
from parakeet_b200.modules.normalizer import ZScore

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
GOLD = "tests/golden/ref_executed_transformer_tts.npz"


def build(cfg, seed, **over):
    cfg = dict(cfg, **over)
    kw = {k: v for k, v in cfg.items() if k not in ("idim", "odim")}
    m = TransformerTTS(cfg["idim"], cfg["odim"], device=DEV, **kw)
    p = ot.synth_params(seed, cfg)
    m.set_state_dict(p)
    return m, p, cfg


def rel(a, b):
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("case", ["maxlen", "stop", "minlen"])
@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_inference_matches_the_reference_executed_fixture(tag, case):
    g = np.load(GOLD)
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    m, _, _ = build(cfg, seed)
    kw = {k: float(g[f"{tag}/{case}/{k}"]) for k in ("threshold", "maxlenratio", "minlenratio") if f"{tag}/{case}/{k}" in g.files}
    outs, probs, att = m.inference(torch.from_numpy(g[f"{tag}/text"]).to(DEV), seed=seed, **kw)
    ref = {k: torch.from_numpy(g[f"{tag}/{case}/{k}"]) for k in ("outs", "probs", "att_ws")}
    # the stop step: the fixture's thresholds sit >= 1.8e-3 from the nearest step's probability, far outside its ~1e-5 error
    assert tuple(outs.shape) == tuple(ref["outs"].shape) and tuple(att.shape) == tuple(ref["att_ws"].shape)
    for name, ours in (("outs", outs), ("probs", probs), ("att_ws", att)):
        assert rel(ours, ref[name]) < 1e-3, (name, rel(ours, ref[name]))


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_forward_matches_the_reference_executed_fixture(tag):
    g = np.load(GOLD)
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    m, _, _ = build(cfg, seed)
    x = {k: torch.from_numpy(g[f"{tag}/fwd/in/{k}"]).to(DEV) for k in ("text", "text_lengths", "speech", "speech_lengths")}
    out = m(x["text"], x["text_lengths"], x["speech"], x["speech_lengths"], seed=seed)
    names = ("after_outs", "before_outs", "logits", "ys", "labels", "olens", "ilens")
    for name, ours in zip(names, out[:7]):                                  # whole tensors, padded rows included
        ref = torch.from_numpy(g[f"{tag}/fwd/{name}"])
        assert tuple(ours.shape) == tuple(ref.shape), name
        if name in ("ys", "labels", "olens", "ilens"):
            assert torch.equal(ours.cpu().to(ref.dtype), ref), name
        else:
            assert rel(ours, ref) < 1e-3, (name, rel(ours, ref))
    assert sorted(out[7]) == sorted(str(k) for k in g[f"{tag}/fwd/need_dict"])


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_teacher_forced_inference_matches_the_fixture(tag):
    g = np.load(GOLD)
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    m, _, _ = build(cfg, seed)
    outs, probs, att = m.inference(torch.from_numpy(g[f"{tag}/text"]).to(DEV), speech=torch.from_numpy(g[f"{tag}/tf/speech"]).to(DEV),
                                   use_teacher_forcing=True, seed=seed)
    assert probs is None
    assert rel(outs, g[f"{tag}/tf/outs"]) < 1e-3 and rel(att, g[f"{tag}/tf/att_ws"]) < 1e-3
    assert (att.double().sum(-1) - 1).abs().max().item() < 1e-4


@pytest.mark.parametrize("n_text,r,adim", [pytest.param(n, r, 128, id=f"{n}-{r}") for n, r in [(0, 1), (1, 2), (150, 3), (512, 1), (150, 1)]]
                         + [pytest.param(150, 2, adim, id=f"150-2-dk{adim // 2}") for adim in (256, 384)])
def test_decoder_matches_the_fp64_oracle_at_every_step(n_text, r, adim):
    """ot.SMALL's two heads at widths 64, 128 and 192."""
    cfg = dict(ot.SMALL, reduction_factor=r, dlayers=3, adim=adim)
    m, p, cfg = build(cfg, 20 + r + adim - 128)
    text = ot.golden_text(cfg, 30 + n_text, n_text)
    T = n_text + 1
    steps = 24
    mlr = (steps + 0.5) * r / T
    outs, probs, att = m.inference(text.to(DEV), threshold=2.0, maxlenratio=mlr, seed=5)
    a64, p64, att64, _ = ot.inference(p, cfg, text, threshold=2.0, maxlenratio=mlr, seed=5)
    assert outs.shape == a64.shape and probs.numel() == steps * r and att.shape == (3, cfg["aheads"], steps, T)
    for name, ours, ref in (("outs", outs, a64), ("probs", probs, p64), ("att_ws", att, att64)):
        assert rel(ours, ref) < 2e-4, (name, rel(ours, ref))
    assert (att.double().sum(-1) - 1).abs().max().item() < 1e-5      # every source-attention row is a distribution


@pytest.mark.parametrize("adim", [256, 384])
def test_forward_matches_the_fp64_oracle_at_wide_heads(adim):
    """The eval forward and teacher-forced inference on ot.golden_batch with two heads of 128 or 192 against ot.forward in fp64:
    the causal and cross modes of pk_fused_attention_ex and the source weights of batched_matmul_nt at those widths.  1e-3
    relative, the bound of the fixture comparisons (split-bf16 GEMMs over the same chain)."""
    m, p, cfg = build(ot.SMALL, 130 + adim, adim=adim, aheads=2)
    text, tl, speech, sl = ot.golden_batch(cfg, 140 + adim)
    out = m(text.to(DEV), tl.to(DEV), speech.to(DEV), sl.to(DEV), seed=2 ** 62 - 1)
    with torch.no_grad():
        ref = ot.forward(p, cfg, text, tl, speech, sl, seed=2 ** 62 - 1)
    for name, ours in zip(("after_outs", "before_outs", "logits", "ys", "labels", "olens", "ilens"), out[:7]):
        assert tuple(ours.shape) == tuple(ref[name].shape), name
        if name in ("ys", "labels", "olens", "ilens"):
            assert torch.equal(ours.cpu().to(ref[name].dtype), ref[name]), name
        else:
            assert rel(ours, ref[name]) < 1e-3, (name, rel(ours, ref[name]))
    n, f = int(tl[0]), int(sl[0])
    outs, _, att = m.inference(text[0, :n].to(DEV), speech=speech[0, :f].to(DEV), use_teacher_forcing=True, seed=3)
    with torch.no_grad():
        one = ot.forward(p, cfg, text[:1, :n], tl[:1], speech[:1, :f], sl[:1], seed=3)
    assert rel(outs, one["after_outs"][0]) < 1e-3 and rel(att, one["att_ws"][0]) < 1e-3


def test_long_run_past_1000_steps():
    m, p, cfg = build(ot.SMALL, 41, reduction_factor=1)
    text = ot.golden_text(cfg, 42, 100)
    outs, probs, att = m.inference(text.to(DEV), threshold=2.0, maxlenratio=10.0, seed=9)
    a64, p64, att64, _ = ot.inference(p, cfg, text, threshold=2.0, maxlenratio=10.0, seed=9)
    assert probs.numel() == 1010 == p64.numel()
    for name, ours, ref in (("outs", outs, a64), ("probs", probs, p64), ("att_ws", att, att64)):
        assert rel(ours, ref) < 2e-4, (name, rel(ours, ref))


@pytest.mark.parametrize("minlen_extra", [0, 4])
def test_stop_step_from_the_fp64_trajectory(minlen_extra):
    """The threshold is placed between two steps' fp64 stop probabilities with the widest margin; the stop (or, with minlen past
    it, the next crossing) must land on the oracle's step.  Probabilities are within 2e-4 relative of fp64 (above), so a margin
    under 2e-4 x max prob could flip the decision: the test then skips and says so."""
    m, p, cfg = build(ot.SMALL, 71, reduction_factor=1)
    text = ot.golden_text(cfg, 72, 20)
    T = 21
    _, p64, _, _ = ot.inference(p, cfg, text, threshold=2.0, maxlenratio=3.0, seed=2)
    traj = p64.tolist()
    best = None
    for s in range(3, len(traj) - 1):
        gap = traj[s] - max(traj[:s])
        if best is None or gap > best[2]:
            best = (max(traj[:s]) + gap / 2, s + 1, gap / 2)
    th, stop, margin = best
    if margin < 2e-4 * max(traj):
        pytest.skip(f"the fp64 stop decision is within the error bound of its threshold (margin {margin:.1e})")
    minlen = stop + minlen_extra if minlen_extra else 0
    kw = dict(threshold=th, maxlenratio=3.0, minlenratio=(minlen + 0.5) / T if minlen else 0.0, seed=2)
    _, want, _, _ = ot.inference(p, cfg, text, **kw)
    _, probs, _ = m.inference(text.to(DEV), **kw)
    assert probs.numel() == want.numel()
    if minlen_extra:
        assert want.numel() >= minlen                         # minlen held the stop at `stop` off


def test_forward_fed_inference_frames_reproduces_inference():
    """Position-keyed prenet masks: forward on inference's own pre-postnet frames with the same seed sees the same decoder inputs.
    The two paths differ only in arithmetic (fp32 FFMA against split-bf16 GEMMs, ~2^-16 relative per product over the same chain
    as above): 1e-3 relative."""
    m, _, cfg = build(ot.SMALL, 81, reduction_factor=2)
    text = ot.golden_text(cfg, 82, 12).to(DEV)
    after, probs, _, before = m._inference(text, None, None, 2.0, 0.0, 3.0, False, 6)
    L = before.shape[0]
    f_after, f_before, logits, *_ = m(text[None], torch.tensor([12], device=DEV), before[None], torch.tensor([L], device=DEV), seed=6)
    assert rel(f_before[0], before) < 1e-3 and rel(f_after[0], after) < 1e-3 and rel(torch.sigmoid(logits[0]), probs) < 1e-3


def test_graph_replay_equals_eager():
    m, _, cfg = build(ot.SMALL, 91)
    text = ot.golden_text(cfg, 92, 10).to(DEV)
    pk = m._pack()
    A = cfg["adim"]
    mem = torch.randn(11, cfg["dlayers"] * 2 * A, device=DEV) * 0.5
    pe = ops.embed_pe(None, None, torch.zeros(1, 30, A, device=DEV), pk["dec_alpha"], None)[0]
    run_dec = lambda: ops.tts_decode(pk["dec"], mem, pe, heads=cfg["aheads"], steps=30, minlen=0, maxlen=30, threshold=2.0, seed=4)  # noqa
    speech = torch.randn(1, 14, cfg["odim"], device=DEV)
    lens, olens = torch.tensor([10], dtype=torch.int32, device=DEV), torch.tensor([14], dtype=torch.int32, device=DEV)
    run_fwd = lambda: m._forward(text[None], lens, speech, olens, 4)[:3]  # noqa: E731
    for run in (run_dec, run_fwd):
        eager = [t.clone() for t in run()]
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            outs = run()
        graph.replay()
        torch.cuda.synchronize()
        assert all(torch.equal(a, b) for a, b in zip(eager, outs))


def test_seed_gives_bit_identical_output():
    m, _, cfg = build(ot.SMALL, 51)
    text = ot.golden_text(cfg, 52, 9).to(DEV)
    a = m.inference(text, threshold=2.0, maxlenratio=4.0, seed=3)
    b = m.inference(text, threshold=2.0, maxlenratio=4.0, seed=3)
    c = m.inference(text, threshold=2.0, maxlenratio=4.0, seed=4)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert not torch.equal(a[0], c[0])


def test_inference_wrapper_denormalises():
    m, _, cfg = build(ot.SMALL, 61)
    g = torch.Generator().manual_seed(0)
    mu, sigma = torch.randn(cfg["odim"], generator=g), torch.rand(cfg["odim"], generator=g) + 0.5
    text = ot.golden_text(cfg, 62, 9).to(DEV)
    torch.manual_seed(7)
    mel = TransformerTTSInference(ZScore(mu, sigma, device=DEV), m)(text)
    torch.manual_seed(7)
    want = m.inference(text)[0] * sigma.to(DEV) + mu.to(DEV)
    assert rel(mel, want) < 1e-6
