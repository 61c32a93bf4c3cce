"""Reading the reference's checkpoint files without Paddle (parakeet_b200/checkpoint.py); layouts restated from paddle.save."""
import pickle

import numpy as np
import pytest
import torch

from parakeet_b200 import checkpoint


def _fs2(device="cpu"):
    from parakeet_b200.models import FastSpeech2
    return FastSpeech2(40, 80, adim=64, aheads=1, elayers=1, eunits=96, dlayers=1, dunits=96, positionwise_layer_type="conv1d",
                       positionwise_conv_kernel_size=3, duration_predictor_layers=1, duration_predictor_chans=32,
                       duration_predictor_kernel_size=3, postnet_layers=2, postnet_filts=5, postnet_chans=32,
                       pitch_predictor_layers=1, pitch_predictor_chans=32, pitch_predictor_kernel_size=3,
                       pitch_embed_kernel_size=1, energy_predictor_layers=1, energy_predictor_chans=32,
                       energy_predictor_kernel_size=3, energy_embed_kernel_size=1, device=device, seed=3)


def test_nested_archive_with_tensor_tuples_roundtrips_into_set_state_dict(tmp_path):
    m = _fs2()
    sd = {k: v.cpu().numpy() + 1.0 for k, v in m.state_dict().items()}
    # snapshot_iter_N.pdz: tensors reduced to (name, ndarray) tuples inside a nested archive
    archive = {"main_params": {k: (f"param_{i}", v) for i, (k, v) in enumerate(sd.items())}, "epoch": 3, "iteration": 1200,
               "main_optimizer": {"LR_Scheduler": {"last_epoch": 3}, "moment1_0": ("m1", np.zeros(4, np.float32))}}
    path = tmp_path / "snapshot_iter_1200.pdz"
    with open(path, "wb") as f:
        pickle.dump(archive, f, protocol=2)
    got = checkpoint.load(path)
    assert got["epoch"] == 3 and got["iteration"] == 1200 and isinstance(got["main_optimizer"]["moment1_0"], np.ndarray)
    m.set_state_dict(got["main_params"])
    for k, v in m.state_dict().items():
        assert np.array_equal(v.cpu().numpy(), sd[k]), k


def test_flat_pdparams_with_structured_names_and_big_param_slices(tmp_path):
    w = np.arange(24, dtype=np.float32).reshape(2, 3, 4)
    flat = {"conv.weight": None, "conv.bias": np.ones(2, np.float32),
            "StructuredToParameterName@@": {"conv.weight": "conv1d_0.w_0", "conv.bias": "conv1d_0.b_0"},
            "conv.weight@@.0": w.reshape(-1)[:10], "conv.weight@@.1": w.reshape(-1)[10:],
            "UnpackBigParamInfor@@": {"conv.weight": {"OriginShape": (2, 3, 4), "slices": ["conv.weight@@.0", "conv.weight@@.1"]}}}
    path = tmp_path / "step-10.pdparams"
    with open(path, "wb") as f:
        pickle.dump(flat, f, protocol=4)
    got = checkpoint.load(path)
    assert set(got) == {"conv.weight", "conv.bias"}
    assert np.array_equal(got["conv.weight"], w) and got["conv.weight"].shape == (2, 3, 4)


def test_checkpoint_is_data_not_code(tmp_path):
    class Evil:
        def __reduce__(self):
            import os
            return (os.system, ("echo pwned",))
    path = tmp_path / "evil.pdz"
    with open(path, "wb") as f:
        pickle.dump({"main_params": Evil()}, f)
    with pytest.raises(pickle.UnpicklingError):
        checkpoint.load(path)


def test_stats_file(tmp_path):
    mu, sd = np.random.randn(80), np.random.rand(80) + 0.5
    np.save(tmp_path / "speech_stats.npy", np.stack([mu, sd]))
    a, b = checkpoint.load_stats(tmp_path / "speech_stats.npy")
    assert a.dtype == np.float32 and np.allclose(a, mu, atol=1e-6) and np.allclose(b, sd, atol=1e-6)
    from parakeet_b200.modules.normalizer import ZScore
    z = ZScore(a, b, device="cpu")
    assert tuple(torch.as_tensor(z.mu).shape) == (80,)
    np.save(tmp_path / "bad.npy", np.zeros(5))
    with pytest.raises(ValueError):
        checkpoint.load_stats(tmp_path / "bad.npy")
