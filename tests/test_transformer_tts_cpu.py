"""TransformerTTS without a GPU: the oracle against the reference's own TransformerTTS.inference executed on the Paddle stand-in
(scripts/make_golden_ref.py transformer_tts), the state-dict keys, the checks that run before any launch, and what ptxas makes of
the decoder kernel."""
import os

import numpy as np
import pytest
import torch

import _ptxas
import oracle.transformer_tts as ot
from parakeet_b200 import _lib
from parakeet_b200.models import TransformerTTS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "ref_executed_transformer_tts.npz")
CASES = ("maxlen", "stop", "minlen")


def model_kwargs(cfg, **over):
    cfg = dict(cfg, **over)
    kw = {k: v for k, v in cfg.items() if k not in ("idim", "odim")}
    return cfg["idim"], cfg["odim"], kw


def case_kwargs(g, tag, case):
    return {k: float(g[f"{tag}/{case}/{k}"]) for k in ("threshold", "maxlenratio", "minlenratio") if f"{tag}/{case}/{k}" in g.files}


def rel(a, b):
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    return ((a - b).abs().max() / b.abs().max()).item()


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_oracle_matches_the_reference_executed_fixture(tag):
    g = np.load(GOLD)
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    text = torch.from_numpy(g[f"{tag}/text"])
    stops = {}
    for case in CASES:
        after, probs, att, _ = ot.inference(ot.synth_params(seed, cfg), cfg, text, seed=seed, **case_kwargs(g, tag, case))
        ref = {k: torch.from_numpy(g[f"{tag}/{case}/{k}"]) for k in ("outs", "probs", "att_ws")}
        assert after.shape == ref["outs"].shape and att.shape == ref["att_ws"].shape, case       # the same stop step
        # fp64 against the reference's fp32: a few fp32 roundings per layer, amplified by the autoregressive feedback
        for name, ours in (("outs", after), ("probs", probs), ("att_ws", att)):
            assert rel(ours, ref[name]) < 1e-5, (case, name)
        stops[case] = probs.numel() // cfg["reduction_factor"]
    maxlen = int((len(text) + 1) * float(g[f"{tag}/maxlen/maxlenratio"]) / cfg["reduction_factor"])
    assert stops["maxlen"] == maxlen and stops["stop"] < maxlen          # the stop case stops on the threshold
    # the minlen case: without minlen its threshold stops earlier; with it the loop still ends by the rule, before maxlen
    kw = case_kwargs(g, tag, "minlen")
    minlen = int((len(text) + 1) * kw["minlenratio"] / cfg["reduction_factor"])
    early = ot.inference(ot.synth_params(seed, cfg), cfg, text, seed=seed, threshold=kw["threshold"], maxlenratio=kw["maxlenratio"])[1]
    assert early.numel() // cfg["reduction_factor"] < minlen <= stops["minlen"] < maxlen


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_oracle_forward_and_teacher_forcing_match_the_fixture(tag):
    g = np.load(GOLD)
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    p = ot.synth_params(seed, cfg)
    x = {k: torch.from_numpy(g[f"{tag}/fwd/in/{k}"]) for k in ("text", "text_lengths", "speech", "speech_lengths")}
    for k, v in zip(("text", "text_lengths", "speech", "speech_lengths"), ot.golden_batch(cfg, seed + 200)):
        assert torch.equal(x[k], v), k                                      # inputs regenerate from their seeds
    o = ot.forward(p, cfg, x["text"], x["text_lengths"], x["speech"], x["speech_lengths"], seed=seed)
    for k in ("after_outs", "before_outs", "logits", "ys", "labels", "olens", "ilens"):
        ref = torch.from_numpy(g[f"{tag}/fwd/{k}"])
        assert tuple(o[k].shape) == tuple(ref.shape), k
        assert rel(o[k], ref) < 1e-5, k                                     # padded rows included
    text, sp = torch.from_numpy(g[f"{tag}/text"]), torch.from_numpy(g[f"{tag}/tf/speech"])
    o = ot.forward(p, cfg, text[None], torch.tensor([len(text)]), sp[None], torch.tensor([sp.shape[0]]), seed=seed)
    assert rel(o["after_outs"][0], g[f"{tag}/tf/outs"]) < 1e-5 and rel(o["att_ws"][0], g[f"{tag}/tf/att_ws"]) < 1e-5


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_eos_and_labels_match_the_reference(tag):
    """eos at column text_lengths[b] of the text padded by one column; labels pad(make_pad_mask(olens - 1), 1) (cut for r > 1)."""
    g = np.load(GOLD)
    cfg, _ = ot.GOLDEN_CONFIGS[tag]
    x = {k: torch.from_numpy(g[f"{tag}/fwd/in/{k}"]) for k in ("text", "text_lengths", "speech_lengths")}
    xs, ilens, labels, olens = ot.eos_and_labels(x["text"], x["text_lengths"], x["speech_lengths"], cfg["idim"] - 1,
                                                  cfg["reduction_factor"])
    assert torch.equal(ilens, torch.from_numpy(g[f"{tag}/fwd/ilens"]))
    assert torch.equal(labels, torch.from_numpy(g[f"{tag}/fwd/labels"]).float())
    assert torch.equal(olens, torch.from_numpy(g[f"{tag}/fwd/olens"]))
    for b, n in enumerate(x["text_lengths"].tolist()):
        assert xs[b, n] == cfg["idim"] - 1 and torch.equal(xs[b, :n], x["text"][b, :n]) and not xs[b, n + 1:].any()


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_keys_are_those_of_the_executed_reference(tag):
    cfg, _ = ot.GOLDEN_CONFIGS[tag]
    ref_keys = sorted(str(k) for k in np.load(GOLD)[f"{tag}/keys"])
    assert sorted(ot.param_shapes(cfg)) == ref_keys
    idim, odim, kw = model_kwargs(cfg)
    m = TransformerTTS(idim, odim, device="cpu", **kw)
    assert sorted(m.state_dict()) == ref_keys
    want = ot.param_shapes(cfg)
    assert all(tuple(v.shape) == want[k] for k, v in m.state_dict().items())


def test_state_dict_round_trip():
    idim, odim, kw = model_kwargs(ot.SMALL)
    p = ot.synth_params(3, ot.SMALL)
    m = TransformerTTS(idim, odim, device="cpu", **kw)
    m.set_state_dict(p)
    assert all(torch.equal(m.state_dict()[k], v) for k, v in p.items())


@pytest.mark.parametrize("over", [dict(eprenet_conv_layers=3), dict(spk_embed_dim=64), dict(use_gst=True), dict(encoder_concat_after=True),
                                  dict(decoder_concat_after=True), dict(encoder_normalize_before=False),
                                  dict(decoder_normalize_before=False), dict(positionwise_layer_type="linear"), dict(dprenet_layers=0),
                                  dict(aheads=4), dict(adim=256, aheads=1), dict(use_scaled_pos_enc=False), dict(use_batch_norm=False), dict(postnet_filts=4),
                                  dict(odim=10), dict(dprenet_units=30), dict(reduction_factor=17)],
                         ids=lambda d: next(iter(d)))
def test_unsupported_configs_raise_in_the_constructor(over):
    idim, odim, kw = model_kwargs(ot.SMALL, **over)             # aheads=4: 32-wide heads at adim 128; adim=256: one 256-wide head
    with pytest.raises(ValueError):
        TransformerTTS(idim, odim, device="cpu", **kw)


def test_inference_refusals_come_before_any_launch():
    idim, odim, kw = model_kwargs(ot.SMALL)
    m = TransformerTTS(idim, odim, device="cpu", **kw)
    text = torch.tensor([3, 4, 5])
    n0 = _lib.launch_count()
    with pytest.raises(_lib.PkError):
        m.inference(text)                                      # CPU tensors: no fallback
    with pytest.raises(ValueError):
        m.inference(text, speech=torch.zeros(4, odim))
    with pytest.raises(ValueError):
        m.inference(text, spembs=torch.zeros(8))
    with pytest.raises(ValueError):
        m.inference(text, use_teacher_forcing=True)              # teacher forcing needs speech
    with pytest.raises(_lib.PkError):
        m.inference(text, speech=torch.zeros(4, odim), use_teacher_forcing=True)
    with pytest.raises(_lib.PkError):
        m(text[None], torch.tensor([3]), torch.zeros(1, 4, odim), torch.tensor([4]))
    with pytest.raises(ValueError):
        m(text[None], torch.tensor([3]), torch.zeros(1, 4, odim), torch.tensor([4]), spembs=torch.zeros(1, 8))
    with pytest.raises(NotImplementedError):
        m.train()
    assert _lib.launch_count() == n0


def test_prenet_rate_is_not_a_model_input():
    """DecoderPrenet.forward calls F.dropout with its default p = 0.5 and never reads dprenet_dropout_rate: two models that differ
    only in the rate hold the same weights, and the oracle (like the decoder kernel) takes no rate at all."""
    idim, odim, kw = model_kwargs(ot.SMALL)
    a = TransformerTTS(idim, odim, device="cpu", **dict(kw, dprenet_dropout_rate=0.2))
    b = TransformerTTS(idim, odim, device="cpu", **dict(kw, dprenet_dropout_rate=0.5))
    assert all(torch.equal(v, b.state_dict()[k]) for k, v in a.state_dict().items())
    assert ot.P_PRENET == 0.5


def test_prenet_masks_are_keyed_by_position():
    m = ot.prenet_masks(7, 6, 32, 2)
    assert torch.equal(m[:, :, :4], ot.prenet_masks(7, 4, 32, 2))       # a row's mask does not depend on how many rows follow
    assert not torch.equal(m[0], m[1]) and 0.3 < m.mean().item() < 0.7


@_ptxas.needs_nvcc
def test_decoder_kernel_compiles_for_sm90a_without_spills():
    rep = _ptxas.report("transformer_tts.cu")
    _ptxas.entry(rep, "tts_decode_kernel")
    for e in rep["entries"]:
        assert (e["stack"], e["spill_stores"], e["spill_loads"]) == (0, 0, 0), e
