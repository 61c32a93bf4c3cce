"""Host-side API pieces of SURVEY.md 8b that need no GPU: spectrogram normalisers (audio/spec_normalizer.py), token-averaged
energy (data/get_feats.py:205-220), checkpoint writer round trip, ConditionalWaveFlow.from_pretrained (models/waveflow.py:827-852)
and the known-answer checks that pin the Slaney mel filterbank to librosa's documented output."""
import os

import numpy as np
import pytest
import torch


def test_log_and_unit_magnitude_match_the_reference_formulas():
    from parakeet_b200.audio import LogMagnitude, UnitMagnitude
    rng = np.random.default_rng(0)
    x = np.abs(rng.normal(size=(80, 37))).astype(np.float32) * 3
    x[0, :5] = 0.0
    lm = LogMagnitude(min=1e-5)
    ref = np.log(np.maximum(x, 1e-5))                                   # spec_normalizer.py:47-50
    assert np.array_equal(lm.transform(x), ref)
    assert np.allclose(lm.inverse(ref), np.maximum(x, 1e-5), rtol=1e-6)
    t = lm.transform(torch.from_numpy(x))
    assert torch.is_tensor(t) and np.allclose(t.numpy(), ref, rtol=1e-6, atol=1e-6)
    um = UnitMagnitude(min=1e-5)
    ref_u = np.clip((20 * np.log10(np.maximum(1e-5, x)) - 20 + 100) / 100, 0, 1)   # :66-69
    assert np.allclose(um.transform(x), ref_u)
    assert np.allclose(um.transform(torch.from_numpy(x)).numpy(), ref_u, atol=1e-6)
    back = um.inverse(ref_u)
    ref_back = np.exp((np.clip(ref_u, 0, 1) * 100 - 100 + 20) / 20 * np.log(10))  # :71-74
    assert np.allclose(back, ref_back) and np.allclose(um.inverse(torch.from_numpy(ref_u)).numpy(), ref_back, rtol=1e-5)


def test_token_averaged_energy_equals_the_reference_loop():
    from parakeet_b200.modules.audio import Energy
    rng = np.random.default_rng(1)
    energy = np.abs(rng.normal(size=57)).astype(np.float32)
    d = np.array([3, 0, 10, 1, 7, 0, 20, 16, 5])                        # sums to 62 > 57: the last slices are clipped / empty

    def ref_average(inp, d):                                             # get_feats.py:205-213 restated
        cs = np.pad(d.cumsum(0), (1, 0), "constant")
        out = []
        for a, b in zip(cs[:-1], cs[1:]):
            arr = inp[a:b]
            out.append(np.mean(arr, axis=0) if len(arr) != 0 else np.array(0))
        return np.expand_dims(np.array(out), 0).T
    got = Energy._average_by_duration(torch.from_numpy(energy), d).numpy()
    ref = ref_average(energy, d)
    assert got.shape == ref.shape == (9, 1)
    assert np.allclose(got, ref, rtol=1e-6, atol=1e-7)


def test_checkpoint_writer_round_trip_and_waveflow_from_pretrained(tmp_path):
    from parakeet_b200 import checkpoint
    from parakeet_b200.models import ConditionalWaveFlow
    src = ConditionalWaveFlow([16, 16], 2, 2, 16, 64, 80, (3, 3), device="cpu", seed=3)
    path = tmp_path / "step-100"
    checkpoint.save(src.state_dict(), str(path) + ".pdparams")
    cfg = {"model": {"upsample_factors": [16, 16], "n_flows": 2, "n_layers": 2, "n_group": 16, "channels": 64, "kernel_size": [3, 3]},
           "data": {"n_mels": 80}}
    m = ConditionalWaveFlow.from_pretrained(cfg, str(path), device="cpu")    # the reference passes the path without extension
    for k, v in src.state_dict().items():
        assert torch.equal(m.state_dict()[k], v), k

    class Node(dict):                                                        # yacs CfgNode style attribute access
        __getattr__ = dict.__getitem__
    m2 = ConditionalWaveFlow.from_pretrained(Node(model=Node(cfg["model"]), data=Node(cfg["data"])), str(path), device="cpu")
    assert sorted(m2.state_dict()) == sorted(src.state_dict())
    # nested snapshot layout (updater.state_dict()) survives the writer
    snap = {"main_params": src.state_dict(), "main_optimizer": {"w_moment1_0": torch.ones(3), "step_count": 7}, "epoch": 2, "iteration": 7}
    checkpoint.save(snap, str(tmp_path / "snapshot_iter_7.pdz"))
    back = checkpoint.load(str(tmp_path / "snapshot_iter_7.pdz"))
    assert back["epoch"] == 2 and back["iteration"] == 7 and back["main_optimizer"]["step_count"] == 7
    assert np.array_equal(back["main_optimizer"]["w_moment1_0"], np.ones(3, dtype=np.float32))
    assert sorted(back["main_params"]) == sorted(src.state_dict())


def test_set_state_dict_is_in_place():
    """A training step turns the parameters into views of its flat buffer; loading a snapshot afterwards (the reference's
    resume order: build the updater, then updater.set_state_dict) must write through those views."""
    from collections import OrderedDict
    from parakeet_b200.layer import Layer
    from parakeet_b200.training import FlatBuffers
    lay = Layer(device="cpu")
    lay._register("w", torch.zeros(4, 3))
    lay._register("b", torch.zeros(5))
    fb = FlatBuffers(lay._params, ["w", "b"], "cpu")
    lay.set_state_dict(OrderedDict(w=torch.full((4, 3), 2.0), b=np.full(5, 3.0, dtype=np.float32)))
    assert lay._params["w"].data_ptr() == fb.flat.data_ptr()
    assert fb.flat[:12].eq(2).all() and fb.flat[12:17].eq(3).all()


def test_mel_filterbank_known_answers():
    """librosa is not installable here, so the Slaney filterbank (modules/audio.py: mel_filterbank, what the reference gets from
    librosa.filters.mel(sr, n_fft, n_mels, fmin, fmax), data/get_feats.py:71-74 / audio/audio.py:54-60) is pinned to what
    librosa documents about it: (1) the docstring example `librosa.filters.mel(sr=22050, n_fft=2048)` prints
    `[[0., 0.016, ..., 0., 0.], ..., [0., 0., ..., 0., 0.]]` (128 filters; second weight of the first filter 0.016);
    (2) Slaney's scale: linear below 1 kHz at 200/3 Hz per mel, 1 kHz = mel 15, log-spaced above with step log(6.4)/27;
    (3) area normalisation: every triangle has weight 2 / (f_hi - f_lo) at its centre frequency."""
    from parakeet_b200.modules.audio import _hz_to_mel, _mel_to_hz, mel_filterbank
    fb = mel_filterbank(22050, 2048, n_mels=128)
    assert fb.shape == (128, 1025) and fb.dtype == np.float32
    assert fb[0, 0] == 0 and round(float(fb[0, 1]), 3) == 0.016 and fb[-1, -1] == 0 and fb[0, -1] == 0
    assert abs(float(_hz_to_mel(1000.0)) - 15.0) < 1e-12 and abs(float(_hz_to_mel(200.0)) - 3.0) < 1e-12
    assert abs(float(_mel_to_hz(15.0 + 27.0)) - 6400.0) < 1e-6             # 27 log-steps above 1 kHz = a factor 6.4
    # the PWG / FastSpeech2 configs of the reference: sr 24000, n_fft 2048, 80 mels, 80..7600 Hz
    fb = mel_filterbank(24000, 2048, 80, 80, 7600).astype(np.float64)
    edges = _mel_to_hz(np.linspace(_hz_to_mel(80.0), _hz_to_mel(7600.0), 82))
    freqs = np.linspace(0, 12000, 1025)
    for i in (0, 17, 40, 79):
        lo, c, hi = edges[i], edges[i + 1], edges[i + 2]
        nz = np.nonzero(fb[i])[0]
        assert freqs[nz[0]] > lo and freqs[nz[-1]] < hi                    # support inside (f_lo, f_hi)
        assert fb[i].max() <= 2.0 / (hi - lo) + 1e-12                      # Slaney area normalisation bounds the peak
        k = np.argmin(np.abs(freqs - c))
        tri = max(0.0, min((freqs[k] - lo) / (c - lo), (hi - freqs[k]) / (hi - c))) * 2.0 / (hi - lo)
        assert abs(fb[i, k] - tri) < 1e-7


@pytest.mark.parametrize("channels", [64, 128])
def test_waveflow_fused_operand_layout(channels):
    """The packed operands of pk_waveflow_flow / pk_waveflow_forward_layer (include/parakeet_b200.h) restated on the CPU: one
    ResidualBlock.add_input evaluated as the kernel does it - GEMM1 over [tap][ring slot][channel] | condition columns with the
    row-step variant's weight, gate per 64-channel block, GEMM2 with the reordered out_proj - against conv2d on the 3-row buffer
    (reference parakeet/models/waveflow.py:248-285).  Host logic only: no CUDA."""
    import torch.nn.functional as F
    from parakeet_b200.models import ConditionalWaveFlow
    C, M, W = channels, 80, 23
    m = ConditionalWaveFlow([16, 16], 2, 3, 16, C, M, (3, 3), device="cpu", seed=9)
    sd = dict(m.state_dict())
    g = torch.Generator().manual_seed(9)
    pk = m._pack()
    nb = C // 64
    a_rows = torch.cat([torch.cat([torch.arange(64 * k, 64 * k + 64), torch.arange(C + 64 * k, C + 64 * k + 64)]) for k in range(nb)])
    o_rows = torch.cat([torch.cat([torch.arange(C + 64 * k, C + 64 * k + 64), torch.arange(64 * k, 64 * k + 64)]) for k in range(nb)])
    from parakeet_b200.models.waveflow import _fold_wn
    p = {k: v.double() for k, v in _fold_wn({k: v.detach().float() for k, v in sd.items()}).items()}
    for layer, i in ((0, 1), (1, 5), (2, 15)):                        # width dilation 1, 2, 4; row-step variants 1, 2, 0
        dil, q = 2 ** layer, f"decoder.1.resnet.{layer}."
        fused = pk["flows"][1]["layers"][layer]["fused"]
        rows = {r: torch.randn(C, W, generator=g).double() for r in (i - 3, i - 2, i - 1)}
        cond = torch.randn(M, W, generator=g).double()
        # reference: conv2d over the 3-row buffer (causal in height, "same" in width), + condition_proj, gate, out_proj
        buf = torch.stack([rows[i - 3], rows[i - 2], rows[i - 1]], dim=1)[None]                    # (1, C, 3, W)
        y = F.conv2d(buf, p[q + "conv.weight"], p[q + "conv.bias"], padding=(0, dil), dilation=(1, dil))[0, :, 0]
        y = y + p[q + "condition_proj.weight"][:, :, 0, 0] @ cond + p[q + "condition_proj.bias"][:, None]
        z = torch.tanh(y[:C]) * torch.sigmoid(y[C:])
        o = p[q + "out_proj.weight"][:, :, 0, 0] @ z + p[q + "out_proj.bias"][:, None]             # res (C) | skip (C)
        # kernel view: ring slot s holds the row r with r % 3 == s; operand columns [tap][slot][c] then the condition channels
        w1 = fused["w1"][i % 3].float().sum(0).double()                                            # hi + lo planes
        w2 = fused["w2"].float().sum(0).double()
        a_op = torch.zeros(9 * C + 128, W, dtype=torch.float64)
        for tap in range(3):
            for s in range(3):
                r = next(r for r in rows if r % 3 == s)
                shifted = torch.zeros(C, W, dtype=torch.float64)
                lo, hi = max(0, -(tap - 1) * dil), min(W, W - (tap - 1) * dil)
                shifted[:, lo:hi] = rows[r][:, lo + (tap - 1) * dil:hi + (tap - 1) * dil]
                a_op[(3 * tap + s) * C:(3 * tap + s + 1) * C] = shifted
        a_op[9 * C:9 * C + M] = cond
        acc1 = w1 @ a_op + torch.from_numpy(fused["b1"]).double()[:, None]
        assert torch.allclose(acc1, y[a_rows], rtol=0, atol=2e-4 * y.abs().max().item())           # bf16x2 planes of the weights
        zk = torch.cat([torch.tanh(acc1[128 * k:128 * k + 64]) * torch.sigmoid(acc1[128 * k + 64:128 * k + 128]) for k in range(nb)])
        acc2 = w2 @ zk + torch.from_numpy(fused["b2"]).double()[:, None]
        assert torch.allclose(acc2, o[o_rows], rtol=0, atol=2e-4 * o.abs().max().item())


def test_vocoder_layer_path_follows_the_model_config(monkeypatch):
    """Which layer kernel Parallel WaveGAN runs follows from its upsample scales alone: with every PK_* environment variable
    reading "0", [4, 5, 3, 5] (hop 300) still runs the frame-rate kernel and [2, 16, 8] (whose band tables are not exact) the
    sample-rate kernel."""
    from parakeet_b200.models import PWGGenerator

    class PkOff(dict):
        def get(self, key, default=None):
            return "0" if key.startswith("PK_") else super().get(key, default)
    monkeypatch.setattr(os, "environ", PkOff(os.environ))
    assert PWGGenerator(upsample_scales=[4, 5, 3, 5], device="cpu")._uses_frame_cond()
    assert not PWGGenerator(upsample_scales=[2, 16, 8], device="cpu")._uses_frame_cond()


def test_waveflow_packs_only_the_operands_of_its_layer_path():
    """An eligible ConditionalWaveFlow packs the fused kernels' operands and none of the two-GEMM row loop's; an n_mels = 64
    model (outside the fused kernels' range) and a one-layer model (which pk_waveflow_flow refuses) the reverse."""
    from parakeet_b200.models import ConditionalWaveFlow
    for n_mels, n_layers, eligible in ((80, 3, True), (64, 3, False), (80, 1, False)):
        m = ConditionalWaveFlow([16, 16], 2, n_layers, 16, 64, n_mels, (3, 3), device="cpu", seed=9)
        assert m._eligible() == eligible
        for fw in m._pack()["flows"]:
            flow_keys = {"host", "in_w", "in_b", "layers"} | (set() if eligible else {"cond_all", "cond_all_b", "out_w", "out_b"})
            assert set(fw) == flow_keys
            for lay in fw["layers"]:
                assert set(lay) == ({"fused"} if eligible else {"conv", "conv_b", "out", "out_b"})
