"""Golden vectors produced by EXECUTING THE REFERENCE'S OWN PYTHON for the hot path.

PaddlePaddle cannot be installed in the build container, so the reference cannot run as is.  Its model code is plain Python
that calls ~60 Paddle primitives; `scripts/refexec/paddle_standin.py` maps those primitives onto torch (same mathematical
definitions; the few Paddle-specific semantics are the ones oracle/README.md lists), `scripts/refexec/loader.py` imports the
reference's files from /root/reference without running `parakeet/__init__.py`.  Under that stand-in this script builds the
reference's own FastSpeech2 / PWGGenerator / ConditionalWaveFlow classes, loads the oracle's seeded Paddle-layout state dicts
into them (which also checks every state-dict key and shape against the reference's class tree) and records what the
REFERENCE code computes.  tests/test_oracle_cpu.py then holds the oracle to these vectors.

    python scripts/make_golden_ref.py        # needs /root/reference; writes tests/golden/ref_executed*.npz
    python scripts/make_golden_ref.py waveflow_forward   # only tests/golden/ref_executed_waveflow_forward.npz
    python scripts/make_golden_ref.py waveflow_configs   # only tests/golden/ref_executed_waveflow_configs.npz
    python scripts/make_golden_ref.py speedyspeech       # only tests/golden/ref_executed_speedyspeech.npz
    python scripts/make_golden_ref.py waveflow_train     # only tests/golden/ref_executed_waveflow_train.npz
    python scripts/make_golden_ref.py fs2ms_train        # only tests/golden/ref_executed_fs2ms_train.npz
    python scripts/make_golden_ref.py speedyspeech_train # only tests/golden/ref_executed_speedyspeech_train.npz
    python scripts/make_golden_ref.py ge2e               # only tests/golden/ref_executed_ge2e.npz
    python scripts/make_golden_ref.py tacotron2          # only tests/golden/ref_executed_tacotron2.npz
    python scripts/make_golden_ref.py transformer_tts    # only tests/golden/ref_executed_transformer_tts.npz
    python scripts/make_golden_ref.py transformer_tts_train    # only tests/golden/ref_executed_transformer_tts_train.npz
"""
import importlib.util
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from _golden import sample_index  # noqa: E402
from refexec import loader, paddle_standin  # noqa: E402

REF = "/root/reference/parakeet"
GOLD = os.path.join(ROOT, "tests", "golden")
T = paddle_standin.T


def load_by_path(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def small_pieces(out):
    # numpy-only collate padding (parakeet/data/batch.py:170-189)
    batch = load_by_path(os.path.join(REF, "data", "batch.py"), "ref_batch")
    rng = np.random.RandomState(20260923)
    lengths = [5, 11, 3, 8]
    seqs = {"text": [rng.randint(1, 70, size=n).astype(np.int64) for n in lengths],
            "speech": [rng.randn(3 * n, 7).astype(np.float32) for n in lengths],
            "pitch": [rng.randn(n, 1).astype(np.float32) for n in lengths]}
    for name, ss in seqs.items():
        for i, s in enumerate(ss):
            out[f"{name}_in{i}"] = s
        out[f"{name}_out"] = batch.batch_sequences(ss)
    out["n"] = np.asarray(len(lengths))
    # padding masks (modules/nets_utils.py:54-125) and the length regulator (fastspeech2_predictor/length_regulator.py:46-89)
    from parakeet.modules import nets_utils as nets
    from parakeet.modules.fastspeech2_predictor.length_regulator import LengthRegulator
    for i, lens in enumerate(([5, 3, 2], [1], [7, 7, 4, 9])):
        out[f"mask_len{i}"] = np.asarray(lens, dtype=np.int64)
        out[f"mask_pad{i}"] = nets.make_pad_mask(T(torch.tensor(lens))).numpy()
        out[f"mask_nonpad{i}"] = nets.make_non_pad_mask(lens).numpy()
    lr = LengthRegulator()
    rng = np.random.RandomState(7)
    cases = {"a": ([[1, 2, 2, 1], [3, 1, 4, 0]], 3),                                  # tests/unit/test_expansion.py:20-24
             "b": (rng.randint(0, 6, size=(3, 17)).tolist(), 8), "c": ([[0, 0, 5], [2, 0, 0]], 4)}
    for name, (ds, c) in cases.items():
        d = np.asarray(ds, dtype=np.int64)
        x = rng.randn(d.shape[0], d.shape[1], c).astype(np.float32)
        y = lr(T(torch.from_numpy(x)), T(torch.from_numpy(d)))
        out[f"lr_{name}_x"], out[f"lr_{name}_d"], out[f"lr_{name}_y"] = x, d, y.numpy()


def check_keys(ref, params, what):
    own = dict(ref.named_parameters())
    own.update(dict(ref.named_buffers()))
    own = {k: v for k, v in own.items() if "generated_tensor_" not in k}
    missing, extra = [k for k in own if k not in params], [k for k in params if k not in own]
    bad = [k for k in own if k in params and tuple(own[k].shape) != tuple(params[k].shape)]
    assert not missing and not extra and not bad, (what, missing[:5], extra[:5], bad[:5])
    return sorted(own)


def fastspeech2(out):
    from oracle import fastspeech2 as ofs
    from parakeet.models.fastspeech2.fastspeech2 import FastSpeech2, FastSpeech2Loss
    cfg = dict(ofs.LJSPEECH_MODEL_CFG)
    ref = FastSpeech2(idim=80, odim=80, **cfg)
    ref.eval()
    params = ofs.synth_params(1)
    out["fs2_keys"] = np.asarray(check_keys(ref, params, "FastSpeech2"))
    ref.set_state_dict(params)
    with torch.no_grad():
        xs, _ = ofs.synth_text(1, [100])                                               # cfg1
        out["fs2_inf_text"] = xs[0].numpy()
        out["fs2_inf_mel"] = ref.inference(T(xs[0])).numpy()
        out["fs2_inf_mel_alpha"] = ref.inference(T(xs[0]), alpha=1.3).numpy()        # uses the stand-in's round (restated)
        b = ofs.synth_train_batch(5, [23, 31, 17])
        for k, v in b.items():
            out[f"fs2_fwd_{k}"] = v.numpy()
        before, after, d_outs, p_outs, e_outs, ys, olens = ref(T(b["text"]), T(b["text_lengths"]), T(b["speech"]), T(b["speech_lengths"]),
                                                               T(b["durations"]), T(b["pitch"]), T(b["energy"]))
        for k, v in (("before", before), ("after", after), ("d_outs", d_outs), ("p_outs", p_outs), ("e_outs", e_outs)):
            out[f"fs2_fwd_out_{k}"] = v.numpy()
        crit = FastSpeech2Loss(use_masking=True, use_weighted_masking=False)
        l1, dur, pitch, energy = crit(after_outs=after, before_outs=before, d_outs=d_outs, p_outs=p_outs, e_outs=e_outs, ys=ys,
                                      ds=T(b["durations"]), ps=T(b["pitch"]), es=T(b["energy"]), ilens=T(b["text_lengths"]), olens=olens)
        out["fs2_loss"] = np.asarray([float(l1), float(dur), float(pitch), float(energy)], dtype=np.float64)


def fastspeech2_multispeaker(out):
    """The aishell3 / vctk shape of the model (conf/default.yaml:76-77: spk_embed_dim 256, concat) plus tone embeddings ("add"):
    the reference's own inference(spk_id, tone_id) and batched forward(..., spk_id, tone_id) - including its F.normalize(axis=1)
    over TIME for the batched (B, T, D) tone embeddings."""
    from oracle import fastspeech2 as ofs
    from parakeet.models.fastspeech2.fastspeech2 import FastSpeech2
    for tag, (st, tt) in (("a", ("concat", "add")), ("b", ("add", "concat"))):
        cfg = dict(ofs.LJSPEECH_MODEL_CFG, num_speakers=6, spk_embed_dim=256, spk_embed_integration_type=st, num_tones=7, tone_embed_dim=32,
                   tone_embed_integration_type=tt)
        ref = FastSpeech2(idim=80, odim=80, **cfg)
        ref.eval()
        params = ofs.add_speaker_tone_params(ofs.synth_params(1), 1, spk_type=st, tone_type=tt)
        out[f"fs2ms_{tag}_keys"] = np.asarray(check_keys(ref, params, "FastSpeech2(multi-speaker)"))
        ref.set_state_dict(params)
        g = torch.Generator().manual_seed(77)
        with torch.no_grad():
            xs, _ = ofs.synth_text(21, [37])
            tone = torch.randint(0, 7, (37,), generator=g)
            spk = torch.tensor([4])
            out[f"fs2ms_{tag}_inf_text"], out[f"fs2ms_{tag}_inf_tone"] = xs[0].numpy(), tone.numpy()
            # tone "concat" cannot run through the reference's inference(): it expands the (T, D) embeddings with
            # shape=[-1, T, -1], a -1 in a dimension that does not exist (fastspeech2.py:611-612) - speaker only there
            out[f"fs2ms_{tag}_inf_mel"] = ref.inference(T(xs[0]), spk_id=T(spk), tone_id=T(tone) if tt == "add" else None).numpy()
            b = ofs.synth_train_batch(22, [14, 19])
            tone_b = torch.randint(0, 7, tuple(b["text"].shape), generator=g)
            spk_b = torch.tensor([1, 5])
            for k, v in b.items():
                out[f"fs2ms_{tag}_fwd_{k}"] = v.numpy()
            out[f"fs2ms_{tag}_fwd_tone"], out[f"fs2ms_{tag}_fwd_spk"] = tone_b.numpy(), spk_b.numpy()
            res = ref(T(b["text"]), T(b["text_lengths"]), T(b["speech"]), T(b["speech_lengths"]), T(b["durations"]), T(b["pitch"]),
                      T(b["energy"]), tone_id=T(tone_b), spk_id=T(spk_b))
            out[f"fs2ms_{tag}_fwd_after"], out[f"fs2ms_{tag}_fwd_d"] = res[1].numpy(), res[2].numpy()


def fastspeech2_training(out):
    """The reference model in TRAIN mode (dropout rates set to 0, BatchNorm on batch statistics), its own FastSpeech2Loss, the
    sum of the four losses as in fastspeech2_updater.py:83, torch autograd through the reference's code: the gradients the
    CUDA training step is checked against (via the oracle), now produced by the reference's wiring."""
    from oracle import fastspeech2 as ofs
    from parakeet.models.fastspeech2.fastspeech2 import FastSpeech2, FastSpeech2Loss
    zero = dict(transformer_enc_dropout_rate=0.0, transformer_enc_positional_dropout_rate=0.0, transformer_enc_attn_dropout_rate=0.0,
                transformer_dec_dropout_rate=0.0, transformer_dec_positional_dropout_rate=0.0, transformer_dec_attn_dropout_rate=0.0,
                duration_predictor_dropout_rate=0.0, postnet_dropout_rate=0.0, pitch_predictor_dropout=0.0, pitch_embed_dropout=0.0,
                energy_predictor_dropout=0.0, energy_embed_dropout=0.0, stop_gradient_from_pitch_predictor=True,
                stop_gradient_from_energy_predictor=False)
    ref = FastSpeech2(idim=80, odim=80, **ofs.LJSPEECH_MODEL_CFG, **zero)
    ref.train()
    params = ofs.synth_params(1)
    ref.set_state_dict(params)
    b = ofs.synth_train_batch(9, [19, 27, 22])
    for k, v in b.items():
        out[f"fs2_train_{k}"] = v.numpy()
    before, after, d_outs, p_outs, e_outs, ys, olens = ref(T(b["text"]), T(b["text_lengths"]), T(b["speech"]), T(b["speech_lengths"]),
                                                           T(b["durations"]), T(b["pitch"]), T(b["energy"]))
    l1, dur, pitch, energy = FastSpeech2Loss()(after_outs=after, before_outs=before, d_outs=d_outs, p_outs=p_outs, e_outs=e_outs, ys=ys,
                                               ds=T(b["durations"]), ps=T(b["pitch"]), es=T(b["energy"]), ilens=T(b["text_lengths"]),
                                               olens=olens)
    (l1 + dur + pitch + energy).backward()
    out["fs2_train_loss"] = np.asarray([float(l1), float(dur), float(pitch), float(energy)], dtype=np.float64)
    # a representative subset of gradients (all 198 would be 150 MB): every kind of tensor on the path
    keep = ["encoder.embed.0.weight", "encoder.embed.1.alpha", "encoder.encoders.0.self_attn.linear_q.weight",
            "encoder.encoders.3.feed_forward.w_1.weight", "encoder.encoders.2.norm1.bias", "encoder.after_norm.weight",
            "duration_predictor.conv.0.0.weight", "duration_predictor.linear.bias", "pitch_predictor.conv.4.0.bias",
            "pitch_embed.0.weight", "energy_embed.0.bias", "decoder.embed.0.alpha", "decoder.encoders.1.self_attn.linear_out.weight",
            "decoder.encoders.3.feed_forward.w_2.bias", "feat_out.weight", "postnet.postnet.0.0.weight", "postnet.postnet.2.1.weight",
            "postnet.postnet.4.1.bias"]
    named = dict(ref.named_parameters())
    for k in keep:
        gk = named[k].grad
        gk = (gk if gk is not None else torch.zeros_like(named[k])).detach().reshape(-1)
        stride = max(1, gk.numel() // 20000)                          # big tensors: every stride-th element + the L2 norm
        out["fs2_train_grad/" + k] = gk[::stride].numpy()
        out["fs2_train_gradnorm/" + k] = np.asarray(float(gk.double().norm()))
    bufs = dict(ref.named_buffers())
    for k in ("postnet.postnet.0.1._mean", "postnet.postnet.0.1._variance", "postnet.postnet.4.1._variance"):
        out["fs2_train_stat/" + k] = bufs[k].detach().numpy()


FS2MS_TRAIN_SPK = (3, 0, 3)          # a repeated speaker and the padding id 0; speakers 1, 2, 4, 5 are absent
FS2MS_TRAIN_KEEP = ("encoder.embed.0.weight", "encoder.encoders.3.feed_forward.w_2.weight", "encoder.after_norm.weight",
                    "encoder.after_norm.bias", "duration_predictor.conv.0.0.weight", "pitch_predictor.conv.0.0.bias",
                    "energy_predictor.conv.0.0.weight", "pitch_embed.0.weight", "decoder.encoders.0.self_attn.linear_q.weight",
                    "feat_out.weight", "postnet.postnet.0.0.weight")


def fastspeech2_multispeaker_training(out):
    """The multi-speaker training gradients (aishell3 / vctk: spk_embed_dim 256, conf/default.yaml:76-77): the reference in
    TRAIN mode (dropout 0), forward(..., spk_id=) as fastspeech2_updater.py:51-99 calls it, its FastSpeech2Loss and the sum of
    the four losses, differentiated by autograd through the reference's code, for "concat" (a) and "add" (b).  3 utterances,
    spk_id = FS2MS_TRAIN_SPK of 6 speakers.  The gradients of the speaker table and the projection bias are stored in full; the
    projection weight and the tensors in FS2MS_TRAIN_KEEP as every stride-th element (stride = numel // 2048) plus their L2 norm."""
    from oracle import fastspeech2 as ofs
    from parakeet.models.fastspeech2.fastspeech2 import FastSpeech2, FastSpeech2Loss
    zero = {k: 0.0 for k in ofs.DROPOUT_DEFAULTS}
    for tag, st in (("a", "concat"), ("b", "add")):
        ref = FastSpeech2(idim=80, odim=80, **ofs.LJSPEECH_MODEL_CFG, **zero, num_speakers=6, spk_embed_dim=256,
                          spk_embed_integration_type=st, stop_gradient_from_pitch_predictor=True, stop_gradient_from_energy_predictor=False)
        ref.train()
        params = {k: v for k, v in ofs.add_speaker_tone_params(ofs.synth_params(1), 1, spk_type=st).items() if not k.startswith("tone_")}
        check_keys(ref, params, f"FastSpeech2(spk {st})")
        ref.set_state_dict(params)
        b = ofs.synth_train_batch(13, [19, 27, 22])
        spk = torch.tensor(FS2MS_TRAIN_SPK, dtype=torch.int64)
        for k, v in b.items():
            out[f"{tag}_{k}"] = v.numpy()
        out[f"{tag}_spk_id"] = spk.numpy()
        before, after, d_outs, p_outs, e_outs, ys, olens = ref(T(b["text"]), T(b["text_lengths"]), T(b["speech"]), T(b["speech_lengths"]),
                                                               T(b["durations"]), T(b["pitch"]), T(b["energy"]), spk_id=T(spk))
        l1, dur, pitch, energy = FastSpeech2Loss()(after_outs=after, before_outs=before, d_outs=d_outs, p_outs=p_outs, e_outs=e_outs,
                                                   ys=ys, ds=T(b["durations"]), ps=T(b["pitch"]), es=T(b["energy"]),
                                                   ilens=T(b["text_lengths"]), olens=olens)
        (l1 + dur + pitch + energy).backward()
        out[f"{tag}_loss"] = np.asarray([float(l1), float(dur), float(pitch), float(energy)], dtype=np.float64)
        named = dict(ref.named_parameters())
        for k in ("spk_embedding_table.weight", "spk_projection.weight", "spk_projection.bias") + FS2MS_TRAIN_KEEP:
            gk = named[k].grad
            gk = (gk if gk is not None else torch.zeros_like(named[k])).detach().reshape(-1)
            stride = 1 if k in ("spk_embedding_table.weight", "spk_projection.bias") else max(1, gk.numel() // 2048)
            out[f"{tag}_grad/{k}"] = gk[::stride].numpy().astype(np.float32)
            out[f"{tag}_gradnorm/{k}"] = np.asarray(float(gk.double().norm()))


def parallel_wavegan(out):
    from oracle import pwg as opwg
    from parakeet.models.parallel_wavegan.parallel_wavegan import PWGGenerator
    cfg = dict(opwg.DEFAULT_GENERATOR_PARAMS)
    cfg["use_weight_norm"] = False                                                    # the folded weights are loaded
    ref = PWGGenerator(**cfg)
    ref.eval()
    folded = opwg.fold_weight_norm(opwg.synth_params(2, weight_norm=True))
    out["pwg_keys"] = np.asarray(check_keys(ref, folded, "PWGGenerator"))
    ref.set_state_dict(folded)
    x, c = opwg.synth_inputs(2, batch=2, mel_frames=10)
    with torch.no_grad():
        out["pwg_x"], out["pwg_c"] = x.numpy(), c.numpy()
        out["pwg_y"] = ref(T(x), T(c)).numpy()
    # with weight norm applied by the reference's own apply_weight_norm: the g / v parametrisation and its 1-D weight_g
    cfg["use_weight_norm"] = True
    ref2 = PWGGenerator(**cfg)
    ref2.eval()
    wn = opwg.synth_params(2, weight_norm=True)
    out["pwg_wn_keys"] = np.asarray(check_keys(ref2, wn, "PWGGenerator(weight_norm)"))
    ref2.set_state_dict(wn)
    with torch.no_grad():
        out["pwg_y_weight_norm"] = ref2(T(x), T(c)).numpy()


def pwg_discriminator(out):
    from oracle import pwg as opwg
    from parakeet.models.parallel_wavegan.parallel_wavegan import PWGDiscriminator
    cfg = dict(opwg.DEFAULT_DISCRIMINATOR_PARAMS)
    cfg["use_weight_norm"] = False
    ref = PWGDiscriminator(**cfg)
    ref.eval()
    dp = opwg.synth_discriminator_params(12)
    out["pwgd_keys"] = np.asarray(check_keys(ref, dp, "PWGDiscriminator"))
    ref.set_state_dict(dp)
    x = torch.randn(2, 1, 900, generator=torch.Generator().manual_seed(21))
    with torch.no_grad():
        out["pwgd_x"], out["pwgd_y"] = x.numpy(), ref(T(x)).numpy()


def waveflow(out):
    from oracle import waveflow as owf
    from parakeet.models.waveflow import ConditionalWaveFlow
    ref = ConditionalWaveFlow(upsample_factors=[16, 16], n_flows=8, n_layers=8, n_group=16, channels=64, n_mels=80, kernel_size=[3, 3])
    ref.eval()
    params = owf.synth_params(4)
    out["wf_keys"] = np.asarray(check_keys(ref, params, "ConditionalWaveFlow"))
    ref.set_state_dict(params)
    g = torch.Generator().manual_seed(4)
    mel = torch.randn(2, 80, 9, generator=g) * 0.5 - 3
    with torch.no_grad():
        cond = ref.encoder(T(mel), trim_conv_artifact=True)
        z = torch.randn(2, cond.shape[-1], generator=g)
        out["wf_mel"], out["wf_z"] = mel.numpy(), z.numpy()
        out["wf_cond"] = cond.numpy()
        out["wf_x"] = ref.decoder.inverse(T(z), cond).numpy()
        # second vector: 22 mel frames -> W = 335 columns > 2 x 128, so the +-128 width taps of layer 7 land on live data
        # (the 9-frame vector above has W = 127: its widest taps only ever see zero padding)
        mel2 = torch.randn(1, 80, 22, generator=g) * 0.5 - 3
        cond2 = ref.encoder(T(mel2), trim_conv_artifact=True)
        z2 = torch.randn(1, cond2.shape[-1], generator=g)
        out["wf2_mel"], out["wf2_z"] = mel2.numpy(), z2.numpy()
        out["wf2_x"] = ref.decoder.inverse(T(z2), cond2).numpy()
    # third vector: the SHIPPED config (examples/waveflow/config.py: 128 residual channels), W = 335 columns
    ref128 = ConditionalWaveFlow(upsample_factors=[16, 16], n_flows=8, n_layers=8, n_group=16, channels=128, n_mels=80, kernel_size=[3, 3])
    ref128.eval()
    params128 = owf.synth_params(5, channels=128)
    check_keys(ref128, params128, "ConditionalWaveFlow(128)")
    ref128.set_state_dict(params128)
    g = torch.Generator().manual_seed(45)
    with torch.no_grad():
        mel3 = torch.randn(1, 80, 22, generator=g) * 0.5 - 3
        cond3 = ref128.encoder(T(mel3), trim_conv_artifact=True)
        z3 = torch.randn(1, cond3.shape[-1], generator=g)
        out["wf128_mel"], out["wf128_z"] = mel3.numpy(), z3.numpy()
        out["wf128_x"] = ref128.decoder.inverse(T(z3), cond3).numpy()


def waveflow_forward(out):
    """The density direction: the reference's own ConditionalWaveFlow.forward (encoder without trim, WaveFlow.forward with its
    permutations and log-det sum) and WaveFlowLoss at two sigmas.  (a) 64 channels, seed-4 parameters, B = 2, 22 mel frames,
    audio of 22 * 256 - 5 samples (shorter than the condition, not a multiple of 16: W = 351); (b) the shipped 128-channel
    config, seed-5 parameters, B = 1, 22 frames."""
    from oracle import waveflow as owf
    from parakeet.models.waveflow import ConditionalWaveFlow, WaveFlowLoss
    g = torch.Generator().manual_seed(46)
    for tag, channels, seed, batch, samples in (("a", 64, 4, 2, 22 * 256 - 5), ("b", 128, 5, 1, 22 * 256)):
        ref = ConditionalWaveFlow(upsample_factors=[16, 16], n_flows=8, n_layers=8, n_group=16, channels=channels, n_mels=80,
                                  kernel_size=[3, 3])
        ref.eval()
        params = owf.synth_params(seed, channels=channels)
        check_keys(ref, params, f"ConditionalWaveFlow({channels})")
        ref.set_state_dict(params)
        mel = torch.randn(batch, 80, 22, generator=g) * 0.5 - 3
        audio = (torch.rand(batch, samples, generator=g) * 2 - 1) * 0.5
        with torch.no_grad():
            z, log_det = ref(T(audio), T(mel))
            out[f"{tag}_mel"], out[f"{tag}_audio"] = mel.numpy(), audio.numpy()
            out[f"{tag}_z"], out[f"{tag}_log_det"] = z.numpy(), log_det.numpy().reshape(1)
            for sigma in (1.0, 0.7):
                out[f"{tag}_loss_sigma{sigma}"] = np.asarray(WaveFlowLoss(sigma)(z, log_det).numpy(), dtype=np.float32).reshape(1)


WAVEFLOW_CONFIGS = dict(upsample_factors=[8, 32], n_flows=4, n_layers=8, n_group=8, channels=128, n_mels=128)


def waveflow_configs(out):
    """A config away from the shipped one in every dimension the CUDA kernels branch on: n_group 8 (7 row steps), 128 mel
    bands (4 condition K-steps in the last chunk), 4 flows (the permutations split at 2), upsample factors 8 x 32, 128
    channels and 8 layers (the only count the reference's ResidualNet takes).  Seed-7 parameters, B = 2, 10 mel frames:
    the reference's inverse from a given z (W = 284 > 2 x 128) and its forward (audio of 10 * 256 - 5 samples, W = 319) with
    WaveFlowLoss at two sigmas."""
    from oracle import waveflow as owf
    from parakeet.models.waveflow import ConditionalWaveFlow, WaveFlowLoss
    cfg = WAVEFLOW_CONFIGS
    ref = ConditionalWaveFlow(kernel_size=[3, 3], **cfg)
    ref.eval()
    params = owf.synth_params(7, **cfg)
    check_keys(ref, params, "ConditionalWaveFlow(waveflow_configs)")
    ref.set_state_dict(params)
    g = torch.Generator().manual_seed(48)
    mel = torch.randn(2, cfg["n_mels"], 10, generator=g) * 0.5 - 3
    audio = (torch.rand(2, 10 * 256 - 5, generator=g) * 2 - 1) * 0.5
    with torch.no_grad():
        cond = ref.encoder(T(mel), trim_conv_artifact=True)
        z = torch.randn(2, cond.shape[-1], generator=g)
        out["mel"], out["z"], out["audio"] = mel.numpy(), z.numpy(), audio.numpy()
        out["x"] = ref.decoder.inverse(T(z), cond).numpy()
        fz, log_det = ref(T(audio), T(mel))
        out["fwd_z"], out["fwd_log_det"] = fz.numpy(), log_det.numpy().reshape(1)
        for sigma in (1.0, 0.7):
            out[f"loss_sigma{sigma}"] = np.asarray(WaveFlowLoss(sigma)(fz, log_det).numpy(), dtype=np.float32).reshape(1)


def waveflow_train(out):
    """The training gradients: torch autograd through the reference's own ConditionalWaveFlow.forward (its weight-normed
    Conv2D / Conv2DTranspose layers, so the gradients are those of weight_g / weight_v) and WaveFlowLoss (sigma 1), as
    examples/waveflow/train.py:95-118 runs them.  64 channels, 2 flows x 8 layers (the reference's Flow takes its height
    dilations from a table of 8), n_group 16, 2 clips x 6 frames of 6 * 256 - 3 samples (W = 95).  Tensors of up to 4096
    elements are stored in full, larger ones as every stride-th element (stride = numel // 4096) plus their L2 norm."""
    from oracle import waveflow as owf
    from parakeet.models.waveflow import ConditionalWaveFlow, WaveFlowLoss
    g = torch.Generator().manual_seed(47)
    ref = ConditionalWaveFlow(upsample_factors=[16, 16], n_flows=2, n_layers=8, n_group=16, channels=64, n_mels=80, kernel_size=[3, 3])
    params = owf.synth_params(6, n_flows=2, n_layers=8, channels=64)
    check_keys(ref, params, "ConditionalWaveFlow(64, 2 flows)")
    ref.set_state_dict(params)
    mel = torch.randn(2, 80, 6, generator=g) * 0.5 - 3
    audio = (torch.rand(2, 6 * 256 - 3, generator=g) * 2 - 1) * 0.5
    z, log_det = ref(T(audio), T(mel))
    loss = WaveFlowLoss(1.0)(z, log_det)
    loss.backward()
    out["mel"], out["audio"] = mel.numpy(), audio.numpy()
    out["loss"] = np.asarray(loss.detach().numpy(), dtype=np.float32).reshape(1)
    for k, v in ref.named_parameters():
        gk = (v.grad if v.grad is not None else torch.zeros_like(v)).detach().reshape(-1)
        out["grad/" + k] = gk[::max(1, gk.numel() // 4096)].numpy().astype(np.float32)
        out["gradnorm/" + k] = np.asarray(float(gk.double().norm()))


def speedyspeech(out):
    """The reference's own SpeedySpeech (eval), SpeedySpeechInference (+ ZScore) and expand: (small) 3 encoder / 2 decoder
    blocks with tones - inference with and without tones, the wrapper, and the batched teacher-forced forward over padded
    tokens; (shipped) the baker yaml's 10 / 18 blocks at one short utterance."""
    from oracle import speedyspeech as oss
    from parakeet.models.speedyspeech.speedyspeech import SpeedySpeech, SpeedySpeechInference
    from parakeet.modules.normalizer import ZScore
    g = torch.Generator().manual_seed(31)
    for tag, cfg, seed, tone_size in (("small", oss.SMALL_CFG, 6, 7), ("shipped", oss.SHIPPED_CFG, 7, None)):
        ref = SpeedySpeech(vocab_size=40, tone_size=tone_size, **cfg)
        ref.eval()
        params = oss.synth_params(seed, cfg, tone_size=tone_size)
        keys = check_keys(ref, params, f"SpeedySpeech({tag})")
        out[f"{tag}_keys"] = np.asarray(keys)
        out[f"{tag}_shapes"] = np.asarray([",".join(map(str, params[k].shape)) for k in keys])
        ref.set_state_dict(params)
        text = torch.randint(1, 40, (12 if tag == "shipped" else 23,), generator=g)
        out[f"{tag}_inf_text"] = text.numpy()
        with torch.no_grad():
            out[f"{tag}_inf_mel"] = ref.inference(T(text)).numpy()
            if tone_size:
                tones = torch.randint(1, tone_size, tuple(text.shape), generator=g)
                out[f"{tag}_inf_tones"] = tones.numpy()
                out[f"{tag}_inf_tone_mel"] = ref.inference(T(text), T(tones)).numpy()
                mu, sigma = torch.randn(80, generator=g), torch.rand(80, generator=g) + 0.5
                out[f"{tag}_wr_mu"], out[f"{tag}_wr_sigma"] = mu.numpy(), sigma.numpy()
                out[f"{tag}_wr_logmel"] = SpeedySpeechInference(ZScore(T(mu), T(sigma)), ref)(T(text), T(tones)).numpy()
                lengths = [17, 9, 14]
                text_b = torch.zeros(3, 17, dtype=torch.int64)
                tones_b = torch.zeros(3, 17, dtype=torch.int64)
                dur_b = torch.zeros(3, 17, dtype=torch.int64)
                for i, n in enumerate(lengths):
                    text_b[i, :n] = torch.randint(1, 40, (n,), generator=g)
                    tones_b[i, :n] = torch.randint(1, tone_size, (n,), generator=g)
                    dur_b[i, :n] = torch.randint(0, 7, (n,), generator=g)
                decoded, pred = ref(T(text_b), T(tones_b), T(dur_b))
                out[f"{tag}_fwd_text"], out[f"{tag}_fwd_tones"], out[f"{tag}_fwd_durations"] = text_b.numpy(), tones_b.numpy(), dur_b.numpy()
                out[f"{tag}_fwd_decoded"], out[f"{tag}_fwd_pred_durations"] = decoded.numpy(), pred.numpy()


def speedyspeech_train(out):
    """The training gradients: torch autograd through the reference's own SpeedySpeech in train() mode (batch-statistics
    BatchNorm1D, encodings.detach() in front of the duration predictor) and the reference's own masked_l1_loss, weighted_mean
    and ssim, composed exactly as SpeedySpeechUpdater.update_core does (speedyspeech_updater.py:52-80; the updater class itself
    needs the Trainer runtime and is not imported).  Small config (3 encoder / 2 decoder blocks), two tone table sizes
    and batches with padded tokens, zero durations and utterances shorter than the longest; always with tones, because the
    reference's forward casts `tones` unconditionally (speedyspeech.py:169) and cannot run without them.  Stored: the batch, the four losses,
    every parameter gradient (tensors of up to 1024 elements in full, larger ones as every stride-th element, stride = numel //
    1024, plus their L2 norm) and the new running statistics."""
    import paddle
    import paddle.nn.functional as F
    from paddle.fluid.layers import huber_loss
    from oracle import speedyspeech as oss
    from oracle import speedyspeech_train as ost
    from parakeet.models.speedyspeech.speedyspeech import SpeedySpeech
    from parakeet.modules.losses import masked_l1_loss, weighted_mean
    from parakeet.modules.ssim import ssim
    cfg = oss.SMALL_CFG
    for tag, seed, tone_size, lens in (("a", 8, 7, [13, 7, 10]), ("b", 9, 5, [16, 9, 12, 14])):
        ref = SpeedySpeech(vocab_size=40, tone_size=tone_size, **cfg)
        ref.train()
        params = oss.synth_params(seed, cfg, tone_size=tone_size)
        check_keys(ref, params, f"SpeedySpeech(train, {tag})")
        ref.set_state_dict(params)
        out[f"{tag}/seed"], out[f"{tag}/tone_size"] = np.asarray(seed), np.asarray(tone_size)
        batch = ost.synth_batch(seed + 100, lens, tone_size=tone_size)
        for k, v in batch.items():
            out[f"{tag}/batch/{k}"] = v.numpy()
        decoded, predicted_durations = ref(text=T(batch["phones"]), tones=T(batch["tones"]),
                                           durations=T(batch["durations"]))
        target_mel = T(batch["feats"])
        spec_mask = F.sequence_mask(T(batch["num_frames"]), dtype=target_mel.dtype).unsqueeze(-1)
        text_mask = F.sequence_mask(T(batch["num_phones"]), dtype=predicted_durations.dtype)
        l1_loss = masked_l1_loss(decoded, target_mel, spec_mask)
        target_durations = paddle.maximum(T(batch["durations"]).astype(predicted_durations.dtype), paddle.to_tensor([1.0]))
        duration_loss = weighted_mean(huber_loss(predicted_durations, paddle.log(target_durations), delta=1.0), text_mask)
        ssim_loss = 1.0 - ssim((decoded * spec_mask).unsqueeze(1), (target_mel * spec_mask).unsqueeze(1))
        loss = l1_loss + ssim_loss + duration_loss
        loss.backward()
        for k, v in dict(loss=loss, l1_loss=l1_loss, duration_loss=duration_loss, ssim_loss=ssim_loss).items():
            out[f"{tag}/{k}"] = np.asarray(float(v.detach().reshape(-1)[0]))
        for k, v in ref.named_parameters():
            gk = (v.grad if v.grad is not None else torch.zeros_like(v)).detach().reshape(-1)
            out[f"{tag}/grad/{k}"] = gk[::max(1, gk.numel() // 1024)].numpy().astype(np.float32)
            out[f"{tag}/gradnorm/{k}"] = np.asarray(float(gk.double().norm()))
        for k, v in ref.named_buffers():
            if k.endswith(("_mean", "_variance")):
                out[f"{tag}/stat/{k}"] = v.detach().numpy().astype(np.float32)


def ge2e(out):
    """The reference's own LSTMSpeakerEncoder (its nn.LSTM on the stand-in's LSTM, Paddle 2.1 keys): embed_sequences (also with
    initial states and reduce=True), the forward's loss and EER (its reshape to [N, -1, N]), loss / similarity matrix on the plain
    (N, M, C) grouping, and every parameter gradient after do_gradient_ops.  (small) 40 mels / 3 layers / hidden 64 / output 64
    at 4 speakers x 3 utterances x 20 frames; (shipped) 40 / 3 / 256 / 256 at 4 x 5 x 160.  The weights and utterances are
    regenerated from their seeds (oracle.ge2e); a sample of the utterances is stored to check that.  Gradients of up to 1024
    elements are stored in full, larger ones as every stride-th element (stride = numel // 1024) plus their L2 norm.
    The reference module imports scipy (interp1d, brentq) and sklearn (roc_curve) for its EER: regenerating this fixture needs
    both installed (the stored EER comes from sklearn's roc_curve)."""
    import numpy
    from oracle import ge2e as og
    from parakeet.models.lstm_speaker_encoder import LSTMSpeakerEncoder
    if not hasattr(numpy, "int"):
        numpy.int = int                  # inv_argmax's np.int (removed from numpy 1.24 on; the reference ran on older numpy)
    for tag, (cfg, (N, M, T_), seed) in og.GOLDEN_CONFIGS.items():
        ref = LSTMSpeakerEncoder(*cfg)
        params = og.synth_params(seed, *cfg)
        keys = check_keys(ref, params, f"LSTMSpeakerEncoder({tag})")
        out[f"{tag}/keys"] = np.asarray(keys)
        ref.set_state_dict(params)
        x = og.synth_utterances(seed + 100, N * M, T_, cfg[0])
        out[f"{tag}/x_sample"] = x.reshape(-1)[::97].numpy()
        with torch.no_grad():
            out[f"{tag}/embeds"] = ref.embed_sequences(T(x)).numpy()
            out[f"{tag}/embed_reduce"] = ref.embed_utterance(T(x)).numpy()
            h0, c0 = og.synth_states(seed + 200, cfg[1], N * M, cfg[2])
            out[f"{tag}/embeds_init"] = ref.embed_sequences(T(x), (T(h0), T(c0))).numpy()
            plain = ref.embed_sequences(T(x)).reshape([N, M, -1])
            out[f"{tag}/plain_sim"] = ref.similarity_matrix(plain)[0].numpy()
            out[f"{tag}/plain_loss"] = np.asarray(float(ref.loss(plain)[0]))
            grouped = ref.embed_sequences(T(x)).reshape([N, -1, N])
            out[f"{tag}/sim"] = ref.similarity_matrix(grouped)[0].numpy()
        loss, eer = ref(T(x), N)
        loss.backward()
        ref.do_gradient_ops()
        out[f"{tag}/loss"], out[f"{tag}/eer"] = np.asarray(float(loss)), np.asarray(float(eer))
        for k, v in ref.named_parameters():
            gk = v.grad.detach().reshape(-1)
            out[f"{tag}/grad/{k}"] = gk[::max(1, gk.numel() // 1024)].numpy().astype(np.float32)
            out[f"{tag}/gradnorm/{k}"] = np.asarray(float(gk.double().norm()))


def tacotron2(out):
    """The reference's own Tacotron2 (its BiRNN encoder LSTM on the stand-in, Paddle 2.1 keys) with p_prenet_dropout = 0 at the
    configs of oracle.tacotron2.GOLDEN_CONFIGS: the teacher-forced forward with and without output_lens, Tacotron2Loss with the
    guided attention term (and the stop term where the model has a stop token), and infer under both stop rules: the alignment
    rule (no stop token; T_enc = 1 gives 22 frames, and a 7-token text), the stop token with its bias at +1e4 (fires at the
    first frame).  Weights are regenerated from their seeds (oracle.tacotron2.synth_params), inputs are stored."""
    from oracle import tacotron2 as ot
    from parakeet.models.tacotron2 import Tacotron2, Tacotron2Loss
    for tag, (cfg, seed) in ot.GOLDEN_CONFIGS.items():
        kw = {k: v for k, v in cfg.items() if k != "vocab_size"}
        ref = Tacotron2(cfg["vocab_size"], **kw)
        params = ot.synth_params(seed, cfg)
        out[f"{tag}/keys"] = np.asarray(check_keys(ref, params, f"Tacotron2({tag})"))
        ref.set_state_dict(params)
        ref.eval()
        x = ot.golden_inputs(cfg, seed + 100)
        for k, v in x.items():
            if v is not None:
                out[f"{tag}/in/{k}"] = v.numpy()
        opt = lambda v: None if v is None else T(v)
        with torch.no_grad():
            for suffix, olens in (("", None), ("_olens", x["output_lens"])):
                o = ref(T(x["text"]), T(x["text_lens"]), T(x["mels"]), opt(olens), opt(x["tones"]), opt(x["gc"]))
                for k, v in o.items():
                    out[f"{tag}/fwd{suffix}/{k}"] = v.numpy()
            stop = cfg["use_stop_token"]
            crit = Tacotron2Loss(use_stop_token_loss=stop, use_guided_attention_loss=True, sigma=0.2)
            losses = crit(o["mel_output"], o["mel_outputs_postnet"], T(x["mels"]), o["alignments"], T(x["output_lens"]),
                          T(x["text_lens"]), o.get("stop_logits"))
            for k, v in losses.items():
                out[f"{tag}/loss/{k}"] = np.asarray(float(v))
            if stop:
                p2 = dict(params)
                p2["decoder.stop_layer.bias"] = torch.full((1,), 1e4)
                ref.set_state_dict(p2)
                o = ref.infer(T(x["text"][:1, :5]), max_decoder_steps=30, tones=opt(None if x["tones"] is None else x["tones"][:1, :5]),
                              global_condition=opt(None if x["gc"] is None else x["gc"][:1]))
                for k, v in o.items():
                    out[f"{tag}/infer_stop/{k}"] = v.numpy()
                ref.set_state_dict(params)
            else:
                for name, n in (("infer_t1", 1), ("infer", 7)):
                    o = ref.infer(T(x["text"][:1, :n]), max_decoder_steps=60 if n == 1 else 30,
                                  tones=opt(None if x["tones"] is None else x["tones"][:1, :n]),
                                  global_condition=opt(None if x["gc"] is None else x["gc"][:1]))
                    for k, v in o.items():
                        out[f"{tag}/{name}/{k}"] = v.numpy()


def stop_threshold(probs, r, first=3):
    """A threshold the stop rule crosses with the widest margin at a step >= first: -> (threshold, stop step, margin)."""
    m = torch.from_numpy(np.asarray(probs.numpy())).reshape(-1, r).amax(1)
    best = None
    for s in range(first, len(m)):
        gap = float(m[s] - m[:s].max())
        if best is None or gap > best[2]:
            best = (float(m[:s].max()) + gap / 2, s + 1, gap / 2)
    return best


class _ListEqShape(tuple):
    def __eq__(self, other):
        return tuple.__eq__(self, tuple(other) if isinstance(other, list) else other)

    __hash__ = tuple.__hash__


def minlen_threshold(probs, r):
    """A threshold crossed first at step idx a and again at a later idx b >= a + 2 (before the run's end), with the widest margin:
    -> (threshold, minlen = a + 2, margin).  With that minlen the early stop at a is held off and the loop ends at b by the rule."""
    m = torch.from_numpy(np.asarray(probs.numpy())).reshape(-1, r).amax(1)
    cands = sorted(set(float(v) for v in m))
    best = None
    for lo, hi in zip(cands, cands[1:]):
        th = (lo + hi) / 2
        idx = [i + 1 for i, v in enumerate(m.tolist()) if v >= th]
        if len(idx) >= 2 and any(b >= idx[0] + 2 for b in idx[1:]) and max(idx) < len(m):
            if best is None or (hi - lo) / 2 > best[2]:
                best = (th, idx[0] + 2, (hi - lo) / 2)
    assert best is not None, "no threshold gives a minlen case that stops by the rule"
    return best


def transformer_tts(out):
    """The reference's own TransformerTTS.inference at oracle.transformer_tts.GOLDEN_CONFIGS, its prenet F.dropout supplied with
    the position-keyed Philox masks (prenet layer i = site i, row = step, element b * units + j; oracle.transformer_tts.prenet_masks):
    under maxlen (threshold 2), under the stop rule (a threshold placed from that run with the widest margin) and with minlenratio
    holding an early stop off until the threshold is crossed again before maxlen; the eval forward on a ragged batch and
    inference(use_teacher_forcing=True).  Weights regenerate from their seeds; inputs are stored."""
    import types
    from oracle import transformer_tts as ot
    from parakeet.models.transformer_tts.transformer_tts import TransformerTTS
    from parakeet.modules.tacotron2 import decoder as prenet_mod
    for tag, (cfg, seed) in ot.GOLDEN_CONFIGS.items():
        kw = {k: v for k, v in cfg.items() if k not in ("idim", "odim")}
        ref = TransformerTTS(cfg["idim"], cfg["odim"], **kw)
        params = ot.synth_params(seed, cfg)
        out[f"{tag}/keys"] = np.asarray(check_keys(ref, params, f"TransformerTTS({tag})"))
        ref.set_state_dict(params)
        ref.eval()
        text = ot.golden_text(cfg, seed + 100, 9 if tag == "small" else 12)
        out[f"{tag}/text"] = text.numpy()
        calls = [0]

        def dropout(x, p=0.5, training=True, **k):
            assert p == ot.P_PRENET and training and x.dim() == 3
            i = calls[0] % cfg["dprenet_layers"]
            calls[0] += 1
            keep = ot.prenet_masks(seed, x.shape[1], x.shape[2], cfg["dprenet_layers"], batch=x.shape[0])[i]
            return T(x * keep * (1.0 / (1.0 - p)))

        saved = prenet_mod.F
        prenet_mod.F = types.SimpleNamespace(dropout=dropout)
        # DecoderLayer's cache check compares a shape with a list, as Paddle's list-valued shapes allow
        paddle_standin.Tensor.shape = property(lambda self: _ListEqShape(torch.Tensor.shape.__get__(self)))
        try:
            with torch.no_grad():
                T_in = len(text) + 1
                mlr = 4.0 if tag == "small" else 2.0
                cases = {"maxlen": dict(threshold=2.0, maxlenratio=mlr)}
                o = ref.inference(T(text), threshold=2.0, maxlenratio=mlr)
                th, stop, margin = stop_threshold(o[1], cfg["reduction_factor"])
                cases["stop"] = dict(threshold=th, maxlenratio=mlr)
                th2, minlen, m2 = minlen_threshold(o[1], cfg["reduction_factor"])
                cases["minlen"] = dict(threshold=th2, maxlenratio=mlr, minlenratio=(minlen + 0.5) * cfg["reduction_factor"] / T_in)
                out[f"{tag}/minlen/margin"] = np.asarray(m2)
                for case, ckw in cases.items():
                    calls[0] = 0
                    o = ref.inference(T(text), **ckw)
                    for k, v in ckw.items():
                        out[f"{tag}/{case}/{k}"] = np.asarray(v)
                    for k, v in zip(("outs", "probs", "att_ws"), o):
                        out[f"{tag}/{case}/{k}"] = v.numpy()
                out[f"{tag}/stop/margin"] = np.asarray(margin)
                # the teacher-forced forward on a ragged batch (padded rows live) and inference(use_teacher_forcing=True)
                text_b, tl, sp, sl = ot.golden_batch(cfg, seed + 200)
                for k, v in (("text", text_b), ("text_lengths", tl), ("speech", sp), ("speech_lengths", sl)):
                    out[f"{tag}/fwd/in/{k}"] = v.numpy()
                calls[0] = 0
                o = ref(T(text_b), T(tl), T(sp), T(sl))
                for k, v in zip(("after_outs", "before_outs", "logits", "ys", "labels", "olens", "ilens"), o[:7]):
                    out[f"{tag}/fwd/{k}"] = np.asarray(v.numpy())
                out[f"{tag}/fwd/need_dict"] = np.asarray(sorted(k for k, v in o[7].items() if not hasattr(v, "parameters")))
                calls[0] = 0
                tf_speech = sp[0, :int(sl[0])]
                o = ref.inference(T(text), speech=T(tf_speech), use_teacher_forcing=True)
                out[f"{tag}/tf/speech"] = tf_speech.numpy()
                out[f"{tag}/tf/outs"], out[f"{tag}/tf/att_ws"] = o[0].numpy(), o[2].numpy()
        finally:
            prenet_mod.F = saved
            del paddle_standin.Tensor.shape


def transformer_tts_train(out):
    """The training losses and gradients: torch autograd through the reference's own TransformerTTS in train() mode, its own
    TransformerTTSLoss and GuidedMultiHeadAttentionLoss, composed as TransformerTTSUpdater.update_core does
    (transformer_tts_updater.py:73-170; the updater class itself needs the Trainer runtime and is not imported), at
    oracle.transformer_tts_train.TRAIN_SMALL and one ragged batch.  Transformer and postnet dropout rates are 0; the decoder prenet's
    always-on F.dropout is supplied with the training step's Philox masks (oracle.transformer_tts_train.train_prenet_masks, step 1).
    Stored: the batch, the losses, every parameter gradient (tensors of up to 1024 elements in full, larger ones as every
    stride-th element, stride = numel // 1024, plus their L2 norm)."""
    import types
    from oracle import transformer_tts_train as ot
    from parakeet.models.transformer_tts.transformer_tts import (GuidedMultiHeadAttentionLoss, TransformerTTS,
                                                                 TransformerTTSLoss)
    from parakeet.modules.tacotron2 import decoder as prenet_mod
    cfg, seed = ot.TRAIN_SMALL, 13
    kw = {k: v for k, v in cfg.items() if k not in ("idim", "odim")}
    ref = TransformerTTS(cfg["idim"], cfg["odim"], **kw)
    params = ot.synth_params(seed, cfg)
    check_keys(ref, params, "TransformerTTS(train)")
    ref.set_state_dict(params)
    ref.train()
    text, tl, sp, sl = ot.golden_batch(cfg, seed + 300, lens=(9, 4, 6), frames=(14, 9, 11))
    for k, v in (("text", text), ("text_lengths", tl), ("speech", sp), ("speech_lengths", sl)):
        out[f"batch/{k}"] = v.numpy()
    keep = ot.train_prenet_masks(ot.TRAIN_SEED, 1, sp.shape[0], sp.shape[1], cfg["dprenet_units"], cfg["dprenet_layers"])
    calls = [0]

    def dropout(x, p=0.5, training=True, **k):
        assert p == ot.P_PRENET and training and x.dim() == 3
        i = calls[0] % cfg["dprenet_layers"]
        calls[0] += 1
        return T(x * keep[i] * (1.0 / (1.0 - p)))

    saved = prenet_mod.F
    prenet_mod.F = types.SimpleNamespace(dropout=dropout)
    try:
        after, before, logits, ys, labels, olens, ilens, need = ref(T(text), T(tl), T(sp), T(sl))
        l1, l2, bce = TransformerTTSLoss(use_masking=True, bce_pos_weight=5.0)(after, before, logits, ys, labels, olens)
        loss = l1 + bce
        att = []
        for idx, layer_idx in enumerate(reversed(range(len(need["decoder"].decoders)))):
            att += [need["decoder"].decoders[layer_idx].src_attn.attn[:, :need["num_heads_applied_guided_attn"]]]
            if idx + 1 == need["num_layers_applied_guided_attn"]:
                break
        g = GuidedMultiHeadAttentionLoss(sigma=0.4, alpha=ot.TRAIN_LAMBDA)(torch.cat(att, 1), ilens, olens)
        loss = loss + g
        loss.backward()
    finally:
        prenet_mod.F = saved
    for k, v in dict(loss=loss, l1_loss=l1, l2_loss=l2, bce_loss=bce, enc_dec_attn_loss=g).items():
        out[k] = np.asarray(float(v.detach().reshape(-1)[0]))
    for k, v in ref.named_parameters():
        gk = (v.grad if v.grad is not None else torch.zeros_like(v)).detach().reshape(-1)
        out[f"grad/{k}"] = gk[::max(1, gk.numel() // 1024)].numpy().astype(np.float32)
        out[f"gradnorm/{k}"] = np.asarray(float(gk.double().norm()))


def wrappers_and_stft(out):
    """FastSpeech2Inference / PWGInference (normaliser wrappers, PWG's replicate padding and transposes) and modules/audio.STFT."""
    import paddle
    from oracle import fastspeech2 as ofs
    from oracle import pwg as opwg
    from parakeet.models.fastspeech2.fastspeech2 import FastSpeech2, FastSpeech2Inference
    from parakeet.models.parallel_wavegan.parallel_wavegan import PWGGenerator, PWGInference
    from parakeet.modules.audio import STFT
    from parakeet.modules.normalizer import ZScore
    g = torch.Generator().manual_seed(11)
    mu, sigma = torch.randn(80, generator=g), torch.rand(80, generator=g) + 0.5
    out["wr_mu"], out["wr_sigma"] = mu.numpy(), sigma.numpy()
    fs = FastSpeech2(idim=80, odim=80, **ofs.LJSPEECH_MODEL_CFG)
    fs.eval()
    fs.set_state_dict(ofs.synth_params(1))
    text = torch.randint(1, 79, (20,), generator=g)
    with torch.no_grad():
        logmel = FastSpeech2Inference(ZScore(T(mu), T(sigma)), fs)(T(text))
    out["wr_text"], out["wr_logmel"] = text.numpy(), logmel.numpy()
    cfg = dict(opwg.DEFAULT_GENERATOR_PARAMS)
    cfg["use_weight_norm"] = False
    gen = PWGGenerator(**cfg)
    gen.eval()
    gen.set_state_dict(opwg.fold_weight_norm(opwg.synth_params(2, weight_norm=True)))
    mel = torch.randn(6, 80, generator=g)
    noise = torch.randn(1, 1, 6 * 300, generator=g)
    real_randn = paddle.randn
    paddle.randn = lambda shape, dtype=None: T(noise)                 # inference() draws its own noise: supply ours
    try:
        with torch.no_grad():
            wav = PWGInference(ZScore(T(mu), T(sigma)), gen)(T(mel))
    finally:
        paddle.randn = real_randn
    out["wr_pwg_logmel"], out["wr_pwg_noise"], out["wr_pwg_wav"] = mel.numpy(), noise.numpy(), wav.numpy()
    wavs = torch.randn(2, 3000, generator=g)
    out["stft_x"] = wavs.numpy()
    for tag, (n_fft, hop, win) in (("a", (512, 128, 512)), ("b", (1024, 120, 600))):
        st = STFT(n_fft, hop, win, window="hann")
        with torch.no_grad():
            re, im = st(T(wavs))
            mag = st.magnitude(T(wavs))
        out[f"stft_{tag}_re"], out[f"stft_{tag}_im"], out[f"stft_{tag}_mag"] = re.numpy(), im.numpy(), mag.numpy()
    # MultiResolutionSTFTLoss (modules/stft_loss.py:163-219): paddle.signal.stft mapped to torch.stft; the clipping, the
    # transposes, the Frobenius ratio, the log-magnitude L1 and the mean over resolutions are the reference's code
    from parakeet.modules.stft_loss import MultiResolutionSTFTLoss
    other = torch.randn(2, 3000, generator=g) * 0.3
    out["mrstft_y"] = other.numpy()
    with torch.no_grad():
        sc, mag = MultiResolutionSTFTLoss()(T(wavs), T(other))
    out["mrstft_loss"] = np.asarray([float(sc), float(mag)], dtype=np.float64)
# Large arrays of the models file are stored as a fixed sample of their elements (tests/_golden.py reads them back), which keeps
# the file under 1 MB: the compared-against outputs, the seeded speech targets (regenerated by the tests) and the gradients.
SAMPLED = ("wf_cond", "fs2_fwd_out_before", "fs2_fwd_out_after", "fs2_inf_mel", "fs2_inf_mel_alpha", "fs2ms_a_inf_mel", "fs2ms_b_inf_mel",
           "fs2ms_a_fwd_after", "fs2ms_b_fwd_after", "stft_a_re", "stft_a_im", "stft_a_mag", "stft_b_re", "stft_b_im", "stft_b_mag",
           "fs2_fwd_speech", "fs2_train_speech", "fs2ms_a_fwd_speech", "fs2ms_b_fwd_speech")


def sampled(models):
    out = {}
    for k, v in models.items():
        if k in SAMPLED or k.startswith("fs2_train_grad/"):
            flat = np.asarray(v).reshape(-1)
            out[k + "@sample"] = flat[sample_index(flat.size, 1024 if k.startswith("fs2_train_grad/") else 2048)]
            out[k + "@shape"] = np.asarray(np.shape(v), dtype=np.int64)
        else:
            out[k] = v
    return out


def main():
    single = {"waveflow_forward": waveflow_forward, "waveflow_configs": waveflow_configs, "speedyspeech": speedyspeech, "waveflow_train": waveflow_train,
              "fs2ms_train": fastspeech2_multispeaker_training, "speedyspeech_train": speedyspeech_train, "ge2e": ge2e,
              "tacotron2": tacotron2, "transformer_tts": transformer_tts, "transformer_tts_train": transformer_tts_train}
    if len(sys.argv) == 2 and sys.argv[1] in single:
        uninstall = loader.install(paddle_standin.build())
        try:
            vecs = {}
            single[sys.argv[1]](vecs)
        finally:
            uninstall()
        name = f"ref_executed_{sys.argv[1]}.npz"
        np.savez_compressed(os.path.join(GOLD, name), **vecs)
        print(name, os.path.getsize(os.path.join(GOLD, name)) // 1024, "KB")
        return
    uninstall = loader.install(paddle_standin.build())
    try:
        small, models = {}, {}
        small_pieces(small)
        fastspeech2(models)
        fastspeech2_multispeaker(models)
        fastspeech2_training(models)
        parallel_wavegan(models)
        pwg_discriminator(models)
        waveflow(models)
        wrappers_and_stft(models)
    finally:
        uninstall()
    np.savez(os.path.join(GOLD, "ref_executed.npz"), **small)
    models = sampled(models)
    np.savez_compressed(os.path.join(GOLD, "ref_executed_models.npz"), **models)
    for name, d in (("ref_executed.npz", small), ("ref_executed_models.npz", models)):
        print(name, os.path.getsize(os.path.join(GOLD, name)) // 1024, "KB", len(d), "arrays")


if __name__ == "__main__":
    main()
