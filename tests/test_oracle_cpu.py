"""CPU tests: the oracle against its golden vectors and against independent cross-checks (SURVEY.md 8c)."""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import fastspeech2 as ofs
from oracle import pwg as opwg

GOLD = os.path.join(os.path.dirname(__file__), "golden")


def test_paddle_round_is_half_away_from_zero():
    x = torch.tensor([0.5, 1.5, 2.5, -0.5, -1.5, 2.4999, 3.0])
    assert ofs.paddle_round(x).tolist() == [1.0, 2.0, 3.0, -1.0, -2.0, 2.0, 3.0]
    assert torch.round(x).tolist()[:3] == [0.0, 2.0, 2.0]  # torch rounds half to even: the hazard this guards against


def test_length_regulator_reference_case_and_gather_equivalence():
    # tests/unit/test_expansion.py:20-24 of the reference pins only the shape [2, 8, 3]
    g = np.load(os.path.join(GOLD, "length_regulator.npz"))
    enc, dur = torch.from_numpy(g["enc"]), torch.from_numpy(g["dur"])
    out = ofs.length_regulator_expand(enc, dur)
    assert list(out.shape) == [2, 8, 3]
    assert torch.equal(out, torch.from_numpy(g["out"]))
    # the 0/1-matrix matmul is bit-identical to a gather (what the CUDA kernel does)
    torch.manual_seed(0)
    x = torch.randn(4, 100, 384)
    d = torch.randint(0, 13, (4, 100))
    ref = ofs.length_regulator_expand(x, d)
    for b in range(4):
        idx = torch.repeat_interleave(torch.arange(100), d[b])
        assert torch.equal(ref[b, :idx.numel()], x[b, idx])
        assert ref[b, idx.numel():].abs().max() == 0 if idx.numel() < ref.shape[1] else True


def test_attention_matches_torch_sdpa():
    torch.manual_seed(1)
    p = {}
    for nm in ("linear_q", "linear_k", "linear_v", "linear_out"):
        p[f"a.{nm}.weight"] = torch.randn(64, 64) / 8
        p[f"a.{nm}.bias"] = torch.randn(64) * 0.1
    x = torch.randn(3, 17, 64)
    lens = [17, 9, 13]
    mask = ofs.make_non_pad_mask(lens, 17).unsqueeze(-2)
    out = ofs.attention(p, "a.", x, mask, n_head=4)
    q = (x @ p["a.linear_q.weight"] + p["a.linear_q.bias"]).reshape(3, 17, 4, 16).transpose(1, 2)
    k = (x @ p["a.linear_k.weight"] + p["a.linear_k.bias"]).reshape(3, 17, 4, 16).transpose(1, 2)
    v = (x @ p["a.linear_v.weight"] + p["a.linear_v.bias"]).reshape(3, 17, 4, 16).transpose(1, 2)
    ref = F.scaled_dot_product_attention(q, k, v, attn_mask=mask.unsqueeze(1))
    ref = ref.transpose(1, 2).reshape(3, 17, 64) @ p["a.linear_out.weight"] + p["a.linear_out.bias"]
    assert torch.allclose(out, ref, atol=1e-5)


def test_fully_masked_attention_row_is_zero_not_nan():
    scores = torch.randn(1, 1, 2, 3)
    m = torch.ones(1, 1, 1, 3, dtype=torch.bool)
    s = ofs.masked_fill(scores, m, float(np.finfo(np.float32).min))
    attn = ofs.masked_fill(torch.softmax(s, dim=-1), m, 0.0)
    assert torch.isfinite(attn).all() and attn.abs().max() == 0


def test_positional_encoding_formula():
    pe = ofs.positional_encoding(50, 8)[0]
    for t in (0, 1, 7, 49):
        for i in range(4):
            div = math.exp(2 * i * -(math.log(10000.0) / 8))
            assert abs(pe[t, 2 * i].item() - math.sin(t * div)) < 1e-5
            assert abs(pe[t, 2 * i + 1].item() - math.cos(t * div)) < 1e-5


def test_pwg_weight_norm_fold_and_upsample_shapes():
    pw = opwg.synth_params(2, weight_norm=True)
    assert pw["first_conv.weight_g"].dim() == 1  # paddle weight_g is 1-D [out] (tests/unit/test_pwg.py:131-132)
    pf = opwg.fold_weight_norm(pw)
    v, g = pw["conv_layers.3.conv.weight_v"], pw["conv_layers.3.conv.weight_g"]
    ref = v * (g / v.reshape(128, -1).norm(dim=1)).reshape(-1, 1, 1)
    assert torch.allclose(pf["conv_layers.3.conv.weight"], ref)
    c = torch.randn(2, 80, 9 + 4)
    up = opwg.conv_in_upsample_net(pf, c, [4, 5, 3, 5])
    assert list(up.shape) == [2, 80, 9 * 300]


def test_pwg_generator_reference_test_config_runs():
    # shapes of tests/unit/test_pwg.py:120-136: layers 9, stacks 3, upsample [4,4,4,4], x [4,1,80*256], c [4,80,84]
    cfg = dict(layers=9, stacks=3, upsample_scales=[4, 4, 4, 4])
    p = opwg.synth_params(3, cfg)
    x, c = torch.randn(1, 1, 8 * 256), torch.randn(1, 80, 8 + 4)
    with torch.no_grad():
        y = opwg.generator_forward(p, x, c, cfg)
    assert list(y.shape) == [1, 1, 8 * 256] and torch.isfinite(y).all()


def test_oracle_matches_golden_pwg():
    g = np.load(os.path.join(GOLD, "pwg_small.npz"))
    params = opwg.fold_weight_norm(opwg.synth_params(2, weight_norm=True))
    with torch.no_grad():
        y, inter = opwg.generator_forward(params, torch.from_numpy(g["x"]), torch.from_numpy(g["c"]), return_intermediates=True)
    assert np.abs(y.numpy() - g["y"]).max() <= 1e-5 * np.abs(g["y"]).max()
    assert abs(inter["skips"].double().sum().item() - float(g["skips_checksum"])) < 1e-2


def test_oracle_matches_golden_fs2():
    fp = ofs.synth_params(1)
    g = np.load(os.path.join(GOLD, "fs2_infer_small.npz"))
    with torch.no_grad():
        out = ofs.fs2_inference(fp, None, torch.from_numpy(g["text"])[0])
    assert out.shape[0] == int(g["durations"].sum())
    assert np.abs(out.numpy() - g["after"][0]).max() <= 2e-5 * np.abs(g["after"]).max()
    g = np.load(os.path.join(GOLD, "fs2_forward_small.npz"))
    b = {k: torch.from_numpy(g[k]) for k in ("text", "text_lengths", "speech", "speech_lengths", "durations", "pitch", "energy")}
    with torch.no_grad():
        ref = ofs.fs2_forward(fp, None, b["text"], b["text_lengths"], b["speech_lengths"], b["durations"], b["pitch"], b["energy"])
        losses = ofs.fs2_loss(ref[1], ref[0], ref[2], ref[3], ref[4], b["speech"], b["durations"], b["pitch"], b["energy"],
                              b["text_lengths"], b["speech_lengths"])
    assert np.abs(ref[1].numpy() - g["after"]).max() <= 2e-5 * np.abs(g["after"]).max()
    assert np.allclose([float(v) for v in losses], g["losses"], rtol=1e-4)


def test_fs2_padding_rows_do_not_leak_in_single_utterance_semantics():
    # an utterance decoded alone equals itself: inference is deterministic and length = sum of rounded durations
    fp = ofs.synth_params(1)
    xs, il = ofs.synth_text(3, [15])
    with torch.no_grad():
        b, a, d, p, e = ofs.fs2_forward(fp, None, xs, il, is_inference=True)
    assert a.shape[1] == int(d.sum()) and (d >= 0).all() and torch.equal(d, torch.round(d))


def test_waveflow_oracle_shapes_and_identity_flow():
    """With the reference's zero-initialised output_proj every flow is the identity up to the row permutations, so
    inverse(z) is a pure permutation of z - a known answer that pins fold / permutation / unfold index arithmetic."""
    from oracle import waveflow as owf
    p = owf.fold_weight_norm(owf.synth_params(4))
    for k in list(p):
        if "output_proj" in k:
            p[k] = torch.zeros_like(p[k])
    mel = torch.randn(1, 80, 4)
    cond = owf.encoder(p, mel, 2)
    assert cond.shape[-1] == 256 * 4 - 272
    z = torch.arange(cond.shape[-1], dtype=torch.float32)[None]
    with torch.no_grad():
        x = owf.infer(p, mel, z)
    # 8 flows: 4 full reversals + 4 half reversals of the 16 rows compose to the identity permutation
    assert torch.equal(x, z)


def test_waveflow_flow_forward_inverse_identity():
    """SURVEY 8c cross-check 4: Flow.inverse (incremental 3-row cache) undoes Flow.forward (full causal convolution) -
    a known-answer test the reference's own math guarantees, tying the row-cache restatement to the conv definition."""
    from oracle import waveflow as owf
    torch.manual_seed(0)
    p = owf.fold_weight_norm(owf.synth_params(4, n_flows=2, n_layers=8))
    x = torch.randn(2, 1, 16, 23)
    cond = torch.randn(2, 80, 16, 23)
    with torch.no_grad():
        z, logs = owf.flow_forward(p, "decoder.0.", x, cond, 8, 16)
        x_back = owf.flow_inverse(p, "decoder.0.", z, cond, 8, 16)
    assert logs.abs().max() > 1e-3                      # the flow is not the identity
    assert (x_back - x).abs().max().item() < 1e-4


def test_pwg_discriminator_matches_module_restatement_and_gan_step_differentiates():
    """SURVEY 8f.1 groundwork: the discriminator restatement against torch.nn modules carrying the same weights, the
    dilation rule of parallel_wavegan.py:571-576, and the two losses of PWGUpdater.update_core being differentiable."""
    import torch.nn as nn
    from oracle import pwg as opwg
    assert opwg.discriminator_dilations() == [1, 1, 2, 3, 4, 5, 6, 7, 8, 1]
    dp = opwg.synth_discriminator_params(12)
    mods, cin = [], 1
    for i, d in enumerate(opwg.discriminator_dilations()):
        cout = 1 if i == 9 else 64
        c = nn.Conv1d(cin, cout, 3, padding=d, dilation=d)
        c.weight.data.copy_(dp[f"conv_layers.{2 * i}.weight"]); c.bias.data.copy_(dp[f"conv_layers.{2 * i}.bias"])
        mods.append(c)
        if i < 9:
            mods.append(nn.LeakyReLU(0.2))
        cin = 64
    x = torch.randn(2, 1, 600, generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        assert torch.allclose(opwg.discriminator_forward(dp, x), nn.Sequential(*mods)(x), atol=1e-6)
    cfg = dict(layers=4, stacks=2, upsample_scales=[2, 3])                  # small generator: hop 6
    gp = {k: v.clone().requires_grad_(True) for k, v in opwg.fold_weight_norm(opwg.synth_params(2, cfg, weight_norm=True)).items()}
    dq = {k: v.clone().requires_grad_(True) for k, v in dp.items()}
    g = torch.Generator().manual_seed(3)
    mel = torch.randn(2, 80, 500 + 4, generator=g); noise = torch.randn(2, 1, 3000, generator=g); wav = torch.randn(2, 1, 3000, generator=g) * 0.1
    out = opwg.gan_step_losses(gp, dq, noise, mel, wav, gen_cfg=cfg)
    out["generator_loss"].backward(retain_graph=True)
    no_grad = [k for k, v in gp.items() if v.grad is None]
    assert all(k.startswith("conv_layers.3.conv1x1_out") for k in no_grad)   # the last block's residual output is unused (:469)
    assert all(torch.isfinite(v.grad).all() and float(v.grad.abs().sum()) > 0 for v in gp.values() if v.grad is not None)
    for v in dq.values():
        v.grad = None
    out["discriminator_loss"].backward()
    assert all(torch.isfinite(v.grad).all() and float(v.grad.abs().sum()) > 0 for v in dq.values())
    assert float(out["generator_loss"].detach()) > float((out["spectral_convergence_loss"] + out["log_stft_magnitude_loss"]).detach()) - 1e-6


def test_adam_restatement_equals_torch_adam():
    """Paddle's Adam form (lr_t = lr*sqrt(1-b2^t)/(1-b1^t), eps scaled by sqrt(1-b2^t)) is algebraically torch.optim.Adam:
    an independent implementation of the optimiser the training step is checked against."""
    from oracle.fastspeech2 import adam_step
    g = torch.Generator().manual_seed(7)
    p0 = {"w": torch.randn(6, 5, generator=g), "b": torch.randn(5, generator=g)}
    tp = {k: v.clone().requires_grad_(True) for k, v in p0.items()}
    opt = torch.optim.Adam(list(tp.values()), lr=1e-3, betas=(0.9, 0.999), eps=1e-8)
    p, state = {k: v.clone() for k, v in p0.items()}, {}
    for step in range(4):
        grads = {k: torch.randn(v.shape, generator=g) * (10.0 ** -step) for k, v in p0.items()}
        for k in tp:
            tp[k].grad = grads[k].clone()
        opt.step()
        p = adam_step(p, grads, state, 1e-3, 0.9, 0.999, 1e-8)
        for k in p:
            assert torch.allclose(p[k], tp[k].detach(), atol=1e-7, rtol=1e-6), (step, k)


def test_weight_norm_fold_equals_torch_weight_norm_and_train_bn_equals_torch_batch_norm():
    """w = g * v / ||v|| over all dims but the first (paddle weight_norm dim 0) against torch's own weight_norm; the
    train-mode BatchNorm normalisation against torch.nn.BatchNorm1d (the running variance differs by design: Paddle keeps the
    biased batch variance, torch the unbiased one - SURVEY 8a hazards)."""
    import torch.nn as nn
    from oracle import fastspeech2 as ofs
    from oracle import pwg as opwg
    import warnings
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")                     # torch deprecates this spelling; it is the reference's semantics
        conv = nn.utils.weight_norm(nn.Conv1d(5, 7, 3), dim=0)
    with torch.no_grad():
        conv.weight_g.mul_(torch.rand(7, 1, 1) + 0.5)
    folded = opwg.fold_weight_norm({"c.weight_g": conv.weight_g.detach().reshape(-1), "c.weight_v": conv.weight_v.detach(),
                                    "c.bias": conv.bias.detach()})
    x = torch.randn(2, 5, 11)
    with torch.no_grad():
        assert torch.allclose(torch.nn.functional.conv1d(x, folded["c.weight"], folded["c.bias"]), conv(x), atol=1e-6)
    # one postnet layer in train mode
    g = torch.Generator().manual_seed(2)
    w = torch.randn(6, 4, 5, generator=g) * 0.3
    p = {"postnet.postnet.0.0.weight": w, "postnet.postnet.0.1.weight": torch.rand(6, generator=g) + 0.5,
         "postnet.postnet.0.1.bias": torch.randn(6, generator=g), "postnet.postnet.0.1._mean": torch.randn(6, generator=g),
         "postnet.postnet.0.1._variance": torch.rand(6, generator=g) + 0.5}
    xs = torch.randn(3, 4, 20, generator=g)
    stats = {}
    y = ofs.postnet(p, xs, 1, train_bn=True, new_stats=stats)
    bn = nn.BatchNorm1d(6, eps=1e-5, momentum=0.1)
    with torch.no_grad():
        bn.weight.copy_(p["postnet.postnet.0.1.weight"]); bn.bias.copy_(p["postnet.postnet.0.1.bias"])
        bn.running_mean.copy_(p["postnet.postnet.0.1._mean"]); bn.running_var.copy_(p["postnet.postnet.0.1._variance"])
        h = torch.nn.functional.conv1d(xs, w, None, padding=2)
        ref = bn.train()(h)
    assert torch.allclose(y, ref, atol=1e-5)
    assert torch.allclose(stats["postnet.postnet.0.1._mean"], bn.running_mean, atol=1e-6)
    n = h.numel() // 6
    biased = (bn.running_var - 0.9 * p["postnet.postnet.0.1._variance"]) * (n - 1) / n + 0.9 * p["postnet.postnet.0.1._variance"]
    assert torch.allclose(stats["postnet.postnet.0.1._variance"], biased, atol=1e-6)


def _frame_rate_table_errors(scales):
    """max |band rows @ P window - conv1x1_aux(upsample(m'))| / max |reference| per utterance length (fp64), with the rows read
    from the compact table through source_row and the window start floor8(t0 // hop - 2) of the pair tile, exactly as the
    layer kernel reads them (frames outside [0, frames) read as zero)."""
    from oracle import pwg as opwg
    from parakeet_b200.models import _pwg_frame_cond as fc
    cfg = {"upsample_scales": scales, "layers": 3, "stacks": 1}
    hop = math.prod(scales)
    params = {k: v.double() for k, v in opwg.fold_weight_norm(opwg.synth_params(2, cfg, weight_norm=True)).items()}
    firs = [params[f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"].reshape(-1) for i in range(len(scales))]
    w_aux = params["conv_layers.1.conv1x1_aux.weight"][:, :, 0]                        # (128, 80)
    g = torch.Generator().manual_seed(0)
    frames_list = [1, 2, 3, 9, 21, 40]                                                  # > 8 frames: the end blocks' shortcut
    table, lay, _ = fc.compact_band_tables(firs, scales, frames_list)
    assert lay["hop"] == hop
    worst = {}
    for b, frames in enumerate(frames_list):
        mel = torch.randn(1, 80, frames + 4, generator=g, dtype=torch.float64)
        m1 = torch.nn.functional.conv1d(mel, params["upsample_net.conv_in.weight"])     # (1, 80, frames)
        c_up = opwg.upsample_net(params, m1, scales)[0]                                # (80, T)
        ref = (w_aux @ c_up).transpose(0, 1)                                           # (T, 128)
        P = (w_aux @ m1[0]).transpose(0, 1)                                            # (frames, 128)
        T = frames * hop
        Ppad = torch.zeros(frames + 2 * fc.KWIN, 128, dtype=torch.float64)
        Ppad[fc.KWIN:fc.KWIN + frames] = P
        err = 0.0
        for m in range(0, T, fc.HALF):
            r = fc.source_row(m, T, b, lay)
            j0 = fc.window_start(m // fc.TILE * fc.TILE, hop)
            win = Ppad[fc.KWIN + j0:fc.KWIN + j0 + fc.KWIN]                           # zero outside [0, frames)
            n = min(fc.HALF, T - m)
            got = table[r:r + n] @ win
            err = max(err, float((got - ref[m:m + n]).abs().max()))
        worst[frames] = err / float(ref.abs().max())
    return worst


def test_pwg_frame_rate_conditioning_tables_reproduce_the_aux_path():
    """conv1x1_aux(upsample(m')) == band rows @ (W_aux m')[window], half tile by half tile, for every upsample config below.
    Where frame_rate_exact holds the tables must be exact to 1e-12; where it does not, they must be wrong for some length,
    so the predicate is checked against this comparison rather than trusted.  Every config is checked before the assertion,
    so a failure names all configs that disagree."""
    from parakeet_b200.models import _pwg_frame_cond as fc
    wrong = {}
    for scales in ([4, 5, 3, 5], [4, 4, 4, 4], [16, 16], [4, 4, 16], [2, 16, 8], [3, 16, 16]):
        worst = _frame_rate_table_errors(scales)
        if fc.frame_rate_exact(scales) != (max(worst.values()) < 1e-12):
            wrong[str(scales)] = (fc.edge_reach(scales), worst)
    assert not wrong, wrong


def test_pwg_compact_band_tables_equal_the_per_length_tables():
    """The kernel reads a compact table (one interior period + start block + 384 end rows per utterance, indexed by
    _pwg_frame_cond.source_row): every half tile of utterances of several lengths must equal the per-length table above."""
    from oracle import pwg as opwg
    from parakeet_b200.models import _pwg_frame_cond as fc
    cfg = opwg.DEFAULT_GENERATOR_PARAMS
    scales = cfg["upsample_scales"]
    params = {k: v.double() for k, v in opwg.fold_weight_norm(opwg.synth_params(2, weight_norm=True)).items()}
    firs = [params[f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"].reshape(-1) for i in range(len(scales))]
    frames_list = [1, 2, 3, 7, 9, 40, 64, 65, 129, 400]
    table, lay, base = fc.compact_band_tables(firs, scales, frames_list)
    again, _, _ = fc.compact_band_tables(firs, scales, frames_list[::-1], base)            # cached base + end blocks: same rows
    assert torch.equal(again[:lay["end_base"]], table[:lay["end_base"]]) and torch.equal(again[-384:], table[lay["end_base"]:lay["end_base"] + 384])
    for nf in (9, 40, 129):                                                                 # the O(384) end block == the full per-length table's tail
        L, full = nf * 300, fc.tile_band_table(firs, scales, nf)
        m1 = fc.end_tile_start(L)
        assert torch.equal(fc.end_block(firs, scales, nf)[:L - m1], full[m1:])
    assert lay["period"] == 19200 and table.shape[0] == 19200 + 128 + 384 * len(frames_list)
    for b, nf in enumerate(frames_list):
        L = nf * lay["hop"]
        full = fc.tile_band_table(firs, scales, nf)
        for m in range(0, (L + 255) // 256 * 256, 128):                 # every half tile of every pair tile with a valid row
            r = fc.source_row(m, L, b, lay)
            got = table[r:r + 128].clone()
            want = torch.zeros(128, fc.KWIN, dtype=torch.float64)
            n = max(0, min(128, L - m))
            want[:n] = full[m:m + n]
            # entry k of a row multiplies frame window_start(pair tile) + k of P; frames outside [0, nf) read as zero (TMA
            # bounds / zero padding), so coefficients for them are "don't care" (short utterances keep them at zero, the
            # interior period carries the coefficient a longer utterance would use)
            j = fc.window_start(m // fc.TILE * fc.TILE, lay["hop"]) + torch.arange(fc.KWIN)
            live = ((j >= 0) & (j < nf)).to(torch.float64)
            got, want = got * live, want * live
            assert torch.equal(got[:n], want[:n]), (nf, m)
            if m + 128 > L - fc.EDGE:                                    # end blocks are zero past the utterance
                assert got[n:].abs().max() == 0 if n < 128 else True


def test_length_regulator_against_vectors_produced_by_the_reference_code():
    """tests/golden/ref_executed.npz: outputs of the reference's own LengthRegulator.forward (its numpy expansion-matrix loop,
    length_regulator.py:46-89) executed by scripts/make_golden_ref.py behind a ten-line torch stand-in for the four paddle
    names it touches.  The oracle (and through tests/test_gpu_kernels.py the CUDA kernel) must reproduce them bit for bit,
    including zero durations and the zero rows past each utterance's total."""
    import os
    from oracle import fastspeech2 as ofs
    g = np.load(os.path.join(GOLD, "ref_executed.npz"))
    for name in ("a", "b", "c"):
        x, d, y = (torch.from_numpy(g[f"lr_{name}_{k}"]) for k in ("x", "d", "y"))
        got = ofs.length_regulator(x, d)
        assert tuple(got.shape) == tuple(y.shape) and torch.equal(got, y), name
        # rows past an utterance's own total are exactly zero, rows before it are exact copies
        tot = d.sum(1)
        for b in range(d.shape[0]):
            assert y[b, int(tot[b]):].abs().sum() == 0
    assert list(g["lr_a_y"].shape) == [2, 8, 3]                      # tests/unit/test_expansion.py:24


def test_pad_masks_against_vectors_produced_by_the_reference_code():
    """make_pad_mask / make_non_pad_mask (modules/nets_utils.py:54-125) executed by scripts/make_golden_ref.py."""
    import os
    from oracle import fastspeech2 as ofs
    g = np.load(os.path.join(GOLD, "ref_executed.npz"))
    for i in range(3):
        lens = torch.from_numpy(g[f"mask_len{i}"])
        assert np.array_equal(ofs.make_pad_mask(lens).numpy(), g[f"mask_pad{i}"])
        assert np.array_equal(ofs.make_non_pad_mask(lens).numpy(), g[f"mask_nonpad{i}"])


def test_philox_restatement_known_answers():
    """oracle.fastspeech2.philox4x32_10 against the Random123 known-answer vectors for philox4x32-10 (kat_vectors)."""
    from oracle import fastspeech2 as ofs
    kat = [((0, 0, 0, 0), (0, 0), (0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8)),
           ((0xffffffff,) * 4, (0xffffffff, 0xffffffff), (0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd)),
           ((0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344), (0xa4093822, 0x299f31d0), (0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1))]
    for ctr, key, want in kat:
        got = ofs.philox4x32_10(*[np.array([c]) for c in ctr], *key)
        assert tuple(int(v[0]) for v in got) == want
    d = ofs.PhiloxDropout(5, 1)
    x = torch.ones(4, 1000)
    y = d(17, x, 0.25)
    assert abs(float((y != 0).float().mean()) - 0.75) < 0.03 and torch.all((y == 0) | (y - 1 / 0.75).abs().lt(1e-6))
