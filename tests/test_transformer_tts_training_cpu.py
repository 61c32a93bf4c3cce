"""The TransformerTTS training step without a GPU: the fp64 oracle against the reference executed on the Paddle stand-in
(scripts/make_golden_ref.py transformer_tts_train), the guided-attention mask's documented values, the step's refusals, its C
entry points and what ptxas makes of its kernels."""
import os
import re

import numpy as np
import pytest
import torch

import _ptxas
from oracle import transformer_tts_train as ot

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "ref_executed_transformer_tts_train.npz")
ENTRY_POINTS = ("pk_masked_softmax", "pk_softmax_bwd", "pk_tts_guided_loss", "pk_tts_loss_workspace", "pk_tts_loss",
                "pk_tts_loss_bwd")


def test_oracle_matches_executed_reference():
    """fp64 oracle vs the reference's fp32 update_core: losses within 2e-6 relative, every gradient within 2e-3 relative L2 (on
    the stored elements) and its norm within 2e-3.  The attention key biases' true gradient is zero (the softmax does not see a
    per-row shift): those two are held to 1e-6 absolute."""
    ref = np.load(GOLDEN)
    cfg = ot.TRAIN_SMALL
    batch = {k: torch.from_numpy(ref[f"batch/{k}"]) for k in ("text", "text_lengths", "speech", "speech_lengths")}
    keep = ot.train_prenet_masks(ot.TRAIN_SEED, 1, batch["speech"].shape[0], batch["speech"].shape[1], cfg["dprenet_units"],
                                 cfg["dprenet_layers"])
    losses, grads, _ = ot.train_step_grads(ot.synth_params(13, cfg), cfg, batch, keep, lam=ot.TRAIN_LAMBDA)
    for k in ("loss", "l1_loss", "l2_loss", "bce_loss", "enc_dec_attn_loss"):
        assert abs(losses[k] - float(ref[k])) <= 2e-6 * abs(float(ref[k])), (k, losses[k], float(ref[k]))
    names = [k[len("grad/"):] for k in ref.files if k.startswith("grad/")]
    assert sorted(names) == sorted(grads), set(names) ^ set(grads)
    for k in names:
        g = grads[k].reshape(-1)
        got, want = g[::max(1, g.numel() // 1024)].numpy(), ref[f"grad/{k}"].astype(np.float64)
        if "linear_k.bias" in k:
            assert np.abs(got).max() < 1e-6 and np.abs(want).max() < 1e-6, k
            continue
        err = np.linalg.norm(got - want) / max(np.linalg.norm(want), 1e-30)
        assert err < 2e-3, (k, err)
        assert abs(float(g.norm()) - float(ref[f"gradnorm/{k}"])) <= 2e-3 * float(ref[f"gradnorm/{k}"]), k


def test_guided_mask_known_answers():
    """The 5 x 5 and 6 x 3 tables of GuidedAttentionLoss._make_guided_attention_mask's docstring (sigma 0.4)."""
    t55 = [[0.0000, 0.1175, 0.3935, 0.6753, 0.8647], [0.1175, 0.0000, 0.1175, 0.3935, 0.6753], [0.3935, 0.1175, 0.0000, 0.1175, 0.3935],
           [0.6753, 0.3935, 0.1175, 0.0000, 0.1175], [0.8647, 0.6753, 0.3935, 0.1175, 0.0000]]
    t63 = [[0.0000, 0.2934, 0.7506], [0.0831, 0.0831, 0.5422], [0.2934, 0.0000, 0.2934], [0.5422, 0.0831, 0.0831],
           [0.7506, 0.2934, 0.0000], [0.8858, 0.5422, 0.0831]]
    assert np.allclose(ot.guided_mask(5, 5, 0.4).numpy(), t55, atol=5e-5)
    assert np.allclose(ot.guided_mask(3, 6, 0.4).numpy(), t63, atol=5e-5)


def _cpu_model(**kw):
    from parakeet_b200.models import TransformerTTS
    cfg = {k: v for k, v in dict(ot.TRAIN_SMALL, **kw).items() if k not in ("idim", "odim")}
    return TransformerTTS(ot.TRAIN_SMALL["idim"], ot.TRAIN_SMALL["odim"], device="cpu", **cfg)


@pytest.mark.parametrize("model_kw, step_kw, what", [
    (dict(reduction_factor=2), {}, "reduction_factor"),
    ({}, dict(use_weighted_masking=True), "use_weighted_masking"),
    ({}, dict(modules_applied_guided_attn=("encoder-decoder", "encoder")), "encoder"),
    ({}, dict(modules_applied_guided_attn=("decoder",)), "decoder"),
])
def test_constructor_refuses_before_device_memory(model_kw, step_kw, what):
    """Each uncovered option raises NotImplementedError naming it, before the step touches the model (its parameters are not yet
    views of a flat buffer) or any device: the model here lives on the CPU."""
    from parakeet_b200.training import TransformerTTSTrainStep
    m = _cpu_model(**model_kw)
    before = dict(m._params)
    with pytest.raises(NotImplementedError, match=what):
        TransformerTTSTrainStep(m, **step_kw)
    assert all(m._params[k] is v for k, v in before.items())


def test_model_still_refuses_train_mode_and_speaker_embeddings():
    m = _cpu_model()
    with pytest.raises(NotImplementedError):
        m.train()
    with pytest.raises(ValueError, match="speaker"):
        _cpu_model(spk_embed_dim=16)


def test_step_entry_points_in_header_and_binding():
    from parakeet_b200 import _lib
    with open(_lib.HEADER) as f:
        header = f.read()
    for name in ENTRY_POINTS:
        assert re.search(rf"\b{name}\s*\(", header), name
        assert name in _lib.exported_symbols(), name
    assert len(_lib.PROTOTYPES["pk_softmax_bwd"].argtypes) == 19
    assert len(_lib.PROTOTYPES["pk_masked_softmax"].argtypes) == 11


@_ptxas.needs_nvcc
def test_step_kernels_compile_for_sm90a_without_spills():
    kernels = {"fs2.cu": ("masked_softmax_kernel",), "train.cu": ("softmax_bwd_kernel",),
               "transformer_tts_train.cu": ("guided_loss_kernel", "tts_loss_partial_kernel", "tts_loss_final_kernel", "tts_loss_bwd_kernel")}
    for src, names in kernels.items():
        entries = _ptxas.report(src)["entries"]
        for k in names:
            found = [e for e in entries if k in e["name"]]          # softmax_bwd_kernel: with and without the guided loss
            assert found, f"ptxas reported no entry function {k} in {src}"
            assert all((e["spill_stores"], e["spill_loads"]) == (0, 0) for e in found), found
