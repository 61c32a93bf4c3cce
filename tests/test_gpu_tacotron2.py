"""Tacotron2 on the GPU against the reference's own Tacotron2 executed on the Paddle stand-in and against the fp64 oracle: the
persistent decoder in both modes, the stop rules, determinism, graph replay, pk_lstm_fwd at the encoder's row counts, the loss,
and the aishell3 voice-cloning chain."""
import os

import numpy as np
import pytest
import torch

import oracle.tacotron2 as ot
from parakeet_b200 import ops
from parakeet_b200.models import Tacotron2, Tacotron2Loss

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


def rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return ((a - b).abs().max() / b.abs().max().clamp_min(1e-30)).item()


def row_rel(a, b, floor=1e-3):
    """worst over rows (the last axis; each element of a 2-D tensor) of max |a - b| / max |b| in the row, the denominator at least
    floor x the tensor's max |b| (so a row of near-zeros is held to the tensor's scale, not to its own)."""
    a, b = torch.as_tensor(a).double().cpu(), torch.as_tensor(b).double().cpu()
    if b.dim() == 2:
        a, b = a.unsqueeze(-1), b.unsqueeze(-1)
    den = b.abs().amax(-1).clamp_min(floor * b.abs().max().item() + 1e-30)
    return ((a - b).abs().amax(-1) / den).max().item()


GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_executed_tacotron2.npz")


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_forward_infer_and_loss_match_the_reference_executed_fixture(tag):
    g = np.load(GOLD)
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    m, p = model(cfg, seed)
    x = ot.golden_inputs(cfg, seed + 100)
    got = {}
    for suffix, olens in (("", None), ("_olens", x["output_lens"])):
        o = m.forward(cuda(x["text"]), cuda(x["text_lens"]), cuda(x["mels"]), cuda(olens), cuda(x["tones"]), cuda(x["gc"]), seed=0)
        got.update({f"fwd{suffix}/{k}": v for k, v in o.items()})
    losses = Tacotron2Loss(cfg["use_stop_token"], True, 0.2)(o["mel_output"], o["mel_outputs_postnet"], cuda(x["mels"]), o["alignments"],
                                                             cuda(x["output_lens"]), cuda(x["text_lens"]), o.get("stop_logits"))
    got.update({f"loss/{k}": v for k, v in losses.items()})
    first = lambda v, n: None if v is None else cuda(v[:1, :n])
    gc1 = None if x["gc"] is None else cuda(x["gc"][:1])
    if cfg["use_stop_token"]:
        ms, _ = model(cfg, seed, stop_bias=1e4)
        o = ms.infer(cuda(x["text"][:1, :5]), 30, first(x["tones"], 5), gc1, seed=0)
        got.update({f"infer_stop/{k}": v for k, v in o.items()})
    else:
        # infer_t1 stops early (22 of 60 frames): the postnet then runs on the max-length buffer with the device-side frame count
        for name, n, steps in (("infer_t1", 1, 60), ("infer", 7, 30)):
            o = m.infer(cuda(x["text"][:1, :n]), steps, first(x["tones"], n), gc1, seed=0)
            got.update({f"{name}/{k}": v for k, v in o.items()})
    stored = sorted(k[len(tag) + 1:] for k in g.files if k.startswith(tag + "/") and "/in/" not in k and not k.endswith("/keys"))
    assert sorted(got) == stored
    for k in stored:
        ref = torch.from_numpy(np.asarray(g[f"{tag}/{k}"]))
        assert tuple(got[k].shape) == tuple(ref.shape), k
        err = row_rel(got[k], ref) if ref.dim() else abs(float(got[k]) - float(ref)) / abs(float(ref))
        assert err < 1e-3, (k, err)


def model(cfg, seed=0, stop_bias=None):
    p = ot.synth_params(seed, cfg, stop_bias=stop_bias)
    m = Tacotron2(device=DEV, **cfg)
    m.set_state_dict(p)
    return m, p


def inputs(cfg, B, T, seed=1):
    text, tones = ot.synth_text(seed, B, T, cfg["vocab_size"], cfg["n_tones"])
    gc = torch.randn(B, cfg["d_global_condition"], generator=torch.Generator().manual_seed(seed)) if cfg["d_global_condition"] else None
    return text, tones, gc


def cuda(x):
    return None if x is None else x.to(DEV)


CONFIGS = {"ljspeech": dict(ot.LJSPEECH, use_stop_token=True), "aishell3": dict(ot.AISHELL3, use_stop_token=True)}


@pytest.mark.parametrize("name", list(CONFIGS))
@pytest.mark.parametrize("B", [1, 32])
def test_teacher_forced_forward_matches_fp64_oracle(name, B):
    cfg = CONFIGS[name]
    m, p = model(cfg)
    T, T_mel = 13, 24
    text, tones, gc = inputs(cfg, B, T)
    lens = torch.tensor([T] + [int(x) for x in torch.randint(1, T + 1, (B - 1,), generator=torch.Generator().manual_seed(5))])
    mels = torch.randn(B, T_mel, 80, generator=torch.Generator().manual_seed(6)) - 2
    olens = torch.full((B,), T_mel)
    olens[-1] = T_mel - 5
    got = m.forward(cuda(text), cuda(lens), cuda(mels), cuda(olens), cuda(tones), cuda(gc), seed=11)
    with torch.no_grad():
        ref = ot.forward(p, cfg, text, lens, mels, olens, tones, gc, seed=11)
    for k in ("mel_output", "mel_outputs_postnet", "alignments", "stop_logits"):
        assert got[k].shape == ref[k].shape, k
        assert row_rel(got[k], ref[k]) < 1e-3, (k, row_rel(got[k], ref[k]))      # every step of every utterance
    # positions past text_lens get exactly zero weight
    for b in range(B):
        assert torch.all(got["alignments"][b, :, int(lens[b]):] == 0)


def test_infer_matches_oracle_at_p05_within_the_fp32_drift():
    cfg = dict(ot.LJSPEECH, use_stop_token=True)
    m, p = model(cfg, stop_bias=-1e4)
    text, _, _ = inputs(cfg, 1, 17)
    got = m.infer(cuda(text), max_decoder_steps=40, seed=3)
    with torch.no_grad():
        r64 = ot.infer(p, cfg, text, max_decoder_steps=40, seed=3)
        r32 = ot.infer(p, cfg, text, max_decoder_steps=40, seed=3, dtype=torch.float32)
    assert got["mel_output"].shape == r64["mel_output"].shape == (1, 40, 80)
    for k in ("mel_output", "mel_outputs_postnet", "alignments", "stop_logits"):
        e_k, e_32 = rel(got[k], r64[k]), rel(r32[k], r64[k])
        print(f"{k}: kernel vs fp64 {e_k:.2e}, fp32 oracle vs fp64 {e_32:.2e}")
        assert e_k < max(1e-3, 10 * e_32), (k, e_k, e_32)


@pytest.mark.parametrize("name", list(CONFIGS))
def test_infer_fed_to_forward_reproduces_it_bit_for_bit(name):
    cfg = dict(CONFIGS[name], use_stop_token=False)
    m, _ = model(cfg)
    T = 11
    text, tones, gc = inputs(cfg, 1, T)
    a = m.infer(cuda(text), max_decoder_steps=24, tones=cuda(tones), global_condition=cuda(gc), seed=9)
    b = m.forward(cuda(text), cuda(torch.tensor([T])), a["mel_output"], tones=cuda(tones), global_condition=cuda(gc), seed=9)
    assert torch.equal(a["mel_output"], b["mel_output"])
    assert torch.equal(a["alignments"], b["alignments"])
    assert torch.equal(a["mel_outputs_postnet"], b["mel_outputs_postnet"])


def test_same_seed_is_bit_identical_and_graph_replay_equals_eager():
    cfg = dict(ot.LJSPEECH, use_stop_token=True)
    m, _ = model(cfg)
    text, _, _ = inputs(cfg, 4, 9)
    lens, mels = torch.tensor([9, 7, 3, 9]), torch.randn(4, 12, 80)
    a = m.forward(cuda(text), cuda(lens), cuda(mels), seed=5)
    b = m.forward(cuda(text), cuda(lens), cuda(mels), seed=5)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    keys, pkeys = m._encode(cuda(text), None, cuda(lens).int(), None)
    w = m._packs()["dec"]
    kw = dict(teacher=True, mels=cuda(mels), text_lens=cuda(lens).int(), seed=5)
    eager = ops.taco2_decode(w, keys, pkeys, 12, **kw)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g):
            out = ops.taco2_decode(w, keys, pkeys, 12, **kw)
    for _ in range(2):
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(x, y)
    assert torch.equal(eager[0], a["mel_output"])


def test_stop_rules_stop_at_the_reference_frame():
    cfg = dict(ot.LJSPEECH)
    m, p = model(cfg)
    one = torch.tensor([[3]])
    assert m.infer(cuda(one), max_decoder_steps=100, seed=0)["mel_output"].shape[1] == 22      # T_enc = 1: fires at step 0
    assert m.infer(cuda(one), max_decoder_steps=9, seed=0)["mel_output"].shape[1] == 9
    text, _, _ = inputs(cfg, 1, 8)
    got = m.infer(cuda(text), max_decoder_steps=60, seed=2)
    with torch.no_grad():
        ref = ot.infer(p, cfg, text, max_decoder_steps=60, seed=2)
    assert got["mel_output"].shape == ref["mel_output"].shape
    cfg = dict(ot.LJSPEECH, use_stop_token=True)
    m, _ = model(cfg, stop_bias=1e4)
    assert m.infer(cuda(text), max_decoder_steps=60, seed=0)["mel_output"].shape[1] == 1


def test_errors_before_any_launch():
    from parakeet_b200 import _lib
    cfg = dict(ot.LJSPEECH, use_stop_token=True, reduction_factor=2)
    m, _ = model(cfg)
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        m.infer(torch.zeros(2, 5, dtype=torch.int64, device=DEV))                  # stop token with B > 1
    with pytest.raises(ValueError):
        m.forward(torch.zeros(1, 5, dtype=torch.int64, device=DEV), torch.tensor([5], device=DEV), torch.zeros(1, 7, 80, device=DEV))
    with pytest.raises(ValueError):
        m.infer(torch.full((1, 5), 99, dtype=torch.int64, device=DEV))              # id out of range
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("rows", [1, 32])
def test_lstm_fwd_rows_against_lstm_cell(rows):
    from parakeet_b200.models.lstm_speaker_encoder import start_states
    H, T = 256, 6
    g = torch.Generator().manual_seed(rows)
    wih, whh = (torch.rand(4 * H, 512, generator=g) - 0.5) / 8, (torch.rand(4 * H, H, generator=g) - 0.5) / 8
    bih, bhh = torch.rand(4 * H, generator=g) - 0.5, torch.rand(4 * H, generator=g) - 0.5
    x = torch.randn(T, rows, 512, generator=g)
    g_in = (x.reshape(T * rows, 512) @ wih.t() + bih).reshape(T, rows, 4 * H)
    h_all, hs, c = start_states(T, rows, H, DEV)
    ops.lstm_fwd(g_in.to(DEV), bhh.to(DEV), ops.lstm_pack_fwd(whh.to(DEV), ops.lstm_gate_perm(H, DEV)), h_all, hs, c)
    h, cc = torch.zeros(rows, H, dtype=torch.float64), torch.zeros(rows, H, dtype=torch.float64)
    for t in range(T):
        h, cc = torch._VF.lstm_cell(x[t].double(), (h, cc), wih.double(), whh.double(), bih.double(), bhh.double())
        assert rel(h_all[t + 1], h) < 1e-4, t


def test_loss_matches_oracle():
    g = torch.Generator().manual_seed(0)
    B, T, C, Te = 3, 20, 80, 9
    mel, post, tgt = (torch.randn(B, T, C, generator=g) for _ in range(3))
    align = torch.softmax(torch.randn(B, T, Te, generator=g), -1)
    stop = torch.randn(B, T, generator=g)
    slens, plens = torch.tensor([20, 14, 9]), torch.tensor([9, 5, 7])
    got = Tacotron2Loss(True, True, 0.2)(cuda(mel), cuda(post), cuda(tgt), cuda(align), cuda(slens), cuda(plens), cuda(stop))
    ref = ot.loss(*(x.double() for x in (mel, post, tgt, align)), slens, plens, stop.double(), use_guided_attention_loss=True)
    for k in ref:
        assert abs(float(got[k]) - float(ref[k])) <= 1e-5 * abs(float(ref[k])) + 1e-7, k


def test_voice_cloning_chain_at_recipe_shapes():
    from parakeet_b200.models import ConditionalWaveFlow, LSTMSpeakerEncoder
    enc = LSTMSpeakerEncoder(40, 3, 256, 256, device=DEV)
    embed = enc.embed_utterance(torch.randn(3, 160, 40, device=DEV))
    cfg = dict(ot.AISHELL3)
    m, _ = model(cfg)
    text, tones, _ = inputs(cfg, 1, 20)
    out = m.infer(cuda(text), max_decoder_steps=40, tones=cuda(tones), global_condition=embed.reshape(1, 256), seed=1)
    mel = out["mel_outputs_postnet"]
    n = mel.shape[1]
    voc = ConditionalWaveFlow([16, 16], 8, 8, 16, 128, 80, (3, 3), device=DEV)
    wav = voc.infer(mel.transpose(1, 2).contiguous())
    assert wav.shape[-1] == n * 256 - 272             # each of the two transposed convs trims its factor
    assert torch.isfinite(wav).all()
