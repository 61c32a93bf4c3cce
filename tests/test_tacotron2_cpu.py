"""Tacotron2 without a GPU: the oracle against the reference's own Tacotron2 executed on the Paddle stand-in
(scripts/make_golden_ref.py tacotron2), state-dict keys (both LSTM key formats), the checks that run before any launch, the
oracle's own consistency and stop rules, and what ptxas makes of the decoder kernel."""
import os

import numpy as np
import pytest
import torch

import _ptxas
import oracle.tacotron2 as ot
from parakeet_b200 import _lib
from parakeet_b200.models import Tacotron2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SMALL = ot.cfg_of(vocab_size=20, d_mels=8)
GOLD = os.path.join(ROOT, "tests", "golden", "ref_executed_tacotron2.npz")


def gold():
    return np.load(GOLD)


def golden_call(tag):
    """-> (cfg, params, inputs, {case: kwargs}) of a fixture config."""
    cfg, seed = ot.GOLDEN_CONFIGS[tag]
    return cfg, ot.synth_params(seed, cfg), ot.golden_inputs(cfg, seed + 100)


def row_rel(a, b, floor=1e-3):
    """worst over rows (last axis) of max |a - b| / max |b| in the row, the denominator at least floor x the tensor's max |b|."""
    a, b = torch.as_tensor(a).double(), torch.as_tensor(b).double()
    if b.dim() == 2:
        a, b = a.unsqueeze(-1), b.unsqueeze(-1)
    den = b.abs().amax(-1).clamp_min(floor * b.abs().max().item() + 1e-30)
    return ((a - b).abs().amax(-1) / den).max().item()


def oracle_cases(tag, dtype=torch.float64):
    """The oracle's outputs for every case the fixture stores under `tag`."""
    cfg, p, x = golden_call(tag)
    out = {}
    with torch.no_grad():
        for suffix, olens in (("", None), ("_olens", x["output_lens"])):
            o = ot.forward(p, cfg, x["text"], x["text_lens"], x["mels"], olens, x["tones"], x["gc"], dtype=dtype)
            out.update({f"fwd{suffix}/{k}": v for k, v in o.items()})
        losses = ot.loss(o["mel_output"], o["mel_outputs_postnet"], x["mels"].to(dtype), o["alignments"], x["output_lens"], x["text_lens"],
                         o.get("stop_logits"), use_stop_token_loss=cfg["use_stop_token"], use_guided_attention_loss=True)
        out.update({f"loss/{k}": v for k, v in losses.items()})
        first = lambda v, n: None if v is None else v[:1, :n]
        if cfg["use_stop_token"]:
            p2 = dict(p, **{"decoder.stop_layer.bias": torch.full((1,), 1e4)})
            o = ot.infer(p2, cfg, x["text"][:1, :5], 30, first(x["tones"], 5), (None if x["gc"] is None else x["gc"][:1]), dtype=dtype)
            out.update({f"infer_stop/{k}": v for k, v in o.items()})
        else:
            for name, n, steps in (("infer_t1", 1, 60), ("infer", 7, 30)):
                o = ot.infer(p, cfg, x["text"][:1, :n], steps, first(x["tones"], n), (None if x["gc"] is None else x["gc"][:1]), dtype=dtype)
                out.update({f"{name}/{k}": v for k, v in o.items()})
    return out


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_oracle_matches_the_reference_executed_fixture(tag):
    g = gold()
    cfg, p, x = golden_call(tag)
    for k, v in x.items():
        if v is not None:
            assert np.array_equal(g[f"{tag}/in/{k}"], v.numpy()), k          # inputs regenerate from their seeds
    ours = oracle_cases(tag)
    stored = sorted(k[len(tag) + 1:] for k in g.files if k.startswith(tag + "/") and "/in/" not in k and not k.endswith("/keys"))
    assert sorted(ours) == stored
    for k in stored:
        ref = torch.from_numpy(np.asarray(g[f"{tag}/{k}"]))
        assert tuple(ours[k].shape) == tuple(ref.shape), k
        err = row_rel(ours[k], ref) if ref.dim() else abs(float(ours[k]) - float(ref)) / abs(float(ref))
        assert err < 1e-4, (k, err)


@pytest.mark.parametrize("tag", list(ot.GOLDEN_CONFIGS))
def test_keys_are_those_of_the_executed_reference(tag):
    cfg, _ = ot.GOLDEN_CONFIGS[tag]
    ref_keys = sorted(str(k) for k in gold()[f"{tag}/keys"])
    assert sorted(ot.param_shapes(cfg)) == ref_keys
    assert sorted(Tacotron2(device="cpu", **cfg).state_dict()) == ref_keys


@pytest.mark.parametrize("cfg", [ot.LJSPEECH, dict(ot.AISHELL3, use_stop_token=True)], ids=["ljspeech", "aishell3_stop"])
def test_keys_and_shapes_match_the_reference_layout(cfg):
    m = Tacotron2(device="cpu", **cfg)
    want = ot.param_shapes(cfg)
    assert list(m.state_dict()) == list(want)
    assert all(tuple(v.shape) == want[k] for k, v in m.state_dict().items())


def test_both_lstm_key_formats_load():
    p = ot.synth_params(0, ot.LJSPEECH)
    flat = ot.flat_lstm_keys(p)
    assert "encoder.lstm.weight_hh_l0_reverse" in flat and "encoder.lstm.0.cell_bw.weight_hh" not in flat
    for state in (p, flat):
        m = Tacotron2(device="cpu", **ot.LJSPEECH)
        m.set_state_dict(state)
        for k, v in p.items():
            assert torch.equal(m.state_dict()[k], v), k


@pytest.mark.parametrize("kw", [dict(d_encoder=256), dict(d_attention_rnn=512), dict(d_prenet=128), dict(d_global_condition=128),
                                dict(d_mels=79), dict(attention_kernel_size=30), dict(p_prenet_dropout=1.0)])
def test_unsupported_configs_raise(kw):
    with pytest.raises(ValueError):
        Tacotron2(device="cpu", **dict(ot.LJSPEECH, **kw))


def test_cpu_inputs_raise_before_any_launch():
    m = Tacotron2(device="cpu", **ot.LJSPEECH)
    text = torch.zeros(1, 5, dtype=torch.int64)
    with pytest.raises(_lib.PkError):
        m.infer(text)
    with pytest.raises(_lib.PkError):
        m.forward(text, torch.tensor([5]), torch.zeros(1, 4, 80))
    with pytest.raises(NotImplementedError):
        m.train()


def test_oracle_fp32_and_fp64_draw_the_same_prenet_masks():
    cfg = dict(SMALL, use_stop_token=True)
    p = ot.synth_params(1, cfg, stop_bias=-1e4)
    text, _ = ot.synth_text(2, 1, 9, cfg["vocab_size"])
    a = ot.infer(p, cfg, text, max_decoder_steps=12, seed=7, dtype=torch.float32)
    b = ot.infer(p, cfg, text, max_decoder_steps=12, seed=7, dtype=torch.float64)
    assert a["mel_output"].shape == b["mel_output"].shape == (1, 12, 8)
    for k in a:
        err = (a[k].double() - b[k]).abs().max() / b[k].abs().max()
        assert err < 1e-4, (k, err)
    c = ot.infer(p, cfg, text, max_decoder_steps=12, seed=8, dtype=torch.float64)
    assert not torch.equal(b["mel_output"], c["mel_output"])          # the dropout is on: another seed, other frames


def test_stop_rules():
    p = ot.synth_params(3, SMALL)
    one, _ = ot.synth_text(4, 1, 1, SMALL["vocab_size"])
    # T_enc = 1: argmax is always the last position, so the rule fires at step 0 and the loop breaks after frame 21
    assert ot.infer(p, SMALL, one, max_decoder_steps=100, seed=0)["mel_output"].shape[1] == 22
    assert ot.infer(p, SMALL, one, max_decoder_steps=22, seed=0)["mel_output"].shape[1] == 22
    assert ot.infer(p, SMALL, one, max_decoder_steps=7, seed=0)["mel_output"].shape[1] == 7
    assert ot.infer(p, SMALL, one, max_decoder_steps=1, seed=0)["mel_output"].shape[1] == 1
    cfg = dict(SMALL, use_stop_token=True)
    ps = ot.synth_params(3, cfg, stop_bias=1e4)
    text, _ = ot.synth_text(5, 1, 6, cfg["vocab_size"])
    assert ot.infer(ps, cfg, text, max_decoder_steps=50, seed=0)["mel_output"].shape[1] == 1


def test_oracle_loss_terms():
    g = torch.Generator().manual_seed(0)
    mel, post, tgt = (torch.randn(2, 6, 4, generator=g, dtype=torch.float64) for _ in range(3))
    align = torch.softmax(torch.randn(2, 6, 5, generator=g, dtype=torch.float64), -1)
    stop = torch.randn(2, 6, generator=g, dtype=torch.float64)
    slens, plens = torch.tensor([6, 4]), torch.tensor([5, 3])
    out = ot.loss(mel, post, tgt, align, slens, plens, stop, use_guided_attention_loss=True, sigma=0.2)
    gal = 0.0
    for b in range(2):
        for n in range(int(slens[b])):
            for t in range(int(plens[b])):
                w = 1 - torch.exp(torch.tensor(-(n / float(slens[b]) - t / float(plens[b])) ** 2 / (2 * 0.04), dtype=torch.float64))
                gal += float(w * align[b, n, t]) / float(slens[b] * plens[b])
    assert abs(float(out["guided_attn_loss"]) - gal / 2) < 1e-12
    assert torch.isclose(out["loss"], out["mel_loss"] + out["post_mel_loss"] + out["guided_attn_loss"] + out["stop_loss"])


@_ptxas.needs_nvcc
def test_decoder_kernels_compile_for_sm90a_without_spills():
    entries = _ptxas.report("tacotron2.cu")["entries"]
    assert sum("taco2_decode_kernel" in e["name"] for e in entries) == 2, [e["name"] for e in entries]
    for e in entries:
        assert (e["stack"], e["spill_stores"], e["spill_loads"]) == (0, 0, 0), e
