"""CPU side of the multi-speaker FastSpeech2 training step: the oracle held to the reference's own multi-speaker training
gradients, the multi-speaker collate and speaker map, and the C-ABI entry points of the speaker path."""
import ctypes
import os

import numpy as np
import pytest
import torch

import _fs2ms
from conftest import rel_err

GOLD = os.path.join(os.path.dirname(__file__), "golden")
FIELDS = ("text", "text_lengths", "speech", "speech_lengths", "durations", "pitch", "energy")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_executed_fs2ms_train.npz"))


@pytest.mark.parametrize("tag,spk_type", [("a", "concat"), ("b", "add")])
def test_multispeaker_training_gradients_equal_executed_reference(g, tag, spk_type):
    """tests/golden/ref_executed_fs2ms_train.npz: autograd through the reference's own train-mode FastSpeech2(spk_id) +
    FastSpeech2Loss on a batch with a repeated speaker and speaker 0.  Losses to 1e-5, gradients to the tolerance of the
    single-speaker executed-reference test; the table gradient exactly zero on row 0 and on the absent speakers."""
    b = {k: torch.from_numpy(g[f"{tag}_{k}"]) for k in FIELDS}
    spk = torch.from_numpy(g[f"{tag}_spk_id"])
    assert 0 in spk.tolist() and len(set(spk.tolist())) < len(spk)
    losses, grads, _ = _fs2ms.train_step_grads(_fs2ms.params(spk_type), spk_type, b, spk)
    assert np.allclose([losses["l1_loss"], losses["duration_loss"], losses["pitch_loss"], losses["energy_loss"]], g[f"{tag}_loss"], rtol=1e-5)
    keys = [k[len(f"{tag}_grad/"):] for k in g.files if k.startswith(f"{tag}_grad/")]
    assert len(keys) == 14
    for k in keys:
        ref = torch.from_numpy(g[f"{tag}_grad/{k}"])
        mine = grads[k].reshape(-1)
        stride = max(1, mine.numel() // ref.numel())
        assert mine[::stride].numel() == ref.numel(), k
        assert rel_err(mine[::stride], ref) < 2e-4, k
        norm = float(g[f"{tag}_gradnorm/{k}"])
        assert abs(float(mine.double().norm()) - norm) <= 2e-4 * max(norm, 1e-12), k
    table = torch.from_numpy(g[f"{tag}_grad/spk_embedding_table.weight"]).reshape(_fs2ms.NUM_SPEAKERS, -1)
    present = set(spk.tolist()) - {0}
    for r in range(_fs2ms.NUM_SPEAKERS):
        assert (table[r].abs().max() > 0) == (r in present), r
        assert (grads["spk_embedding_table.weight"][r].abs().max() > 0) == (r in present), r


def _examples(with_spk):
    rng = np.random.RandomState(3)
    out = []
    for i, n in enumerate((5, 9, 7)):
        d = rng.randint(1, 4, size=n)
        e = dict(text=rng.randint(1, 70, size=n), text_lengths=n, durations=d, speech=rng.randn(int(d.sum()), 80).astype(np.float32),
                 speech_lengths=int(d.sum()), pitch=rng.randn(n).astype(np.float32), energy=rng.randn(n, 1).astype(np.float32))
        if with_spk:
            e["spk_id"] = (4, 0, 4)[i]
        out.append(e)
    return out


def test_multispeaker_collate_adds_spk_id_and_leaves_single_speaker_batches_unchanged():
    from parakeet_b200.data import FS2_FIELDS, FS2_MS_FIELDS, batch_sequences, fastspeech2_batch
    assert FS2_MS_FIELDS == FS2_FIELDS + ("spk_id",)
    single, multi = fastspeech2_batch(_examples(False)), fastspeech2_batch(_examples(True))
    assert tuple(sorted(single)) == tuple(sorted(FIELDS))
    assert tuple(sorted(multi)) == tuple(sorted(FIELDS + ("spk_id",)))
    assert multi["spk_id"].dtype == torch.int64 and multi["spk_id"].tolist() == [4, 0, 4] and multi["spk_id"].shape == (3,)
    ex = _examples(False)
    expect = dict(text=batch_sequences([np.asarray(e["text"], np.int64) for e in ex]), text_lengths=np.asarray([5, 9, 7], np.int64),
                  durations=batch_sequences([np.asarray(e["durations"], np.int64) for e in ex]),
                  speech=batch_sequences([e["speech"] for e in ex]), speech_lengths=np.asarray([e["speech_lengths"] for e in ex], np.int64),
                  pitch=batch_sequences([e["pitch"][:, None] for e in ex]), energy=batch_sequences([e["energy"] for e in ex]))
    for k, v in expect.items():
        assert single[k].dtype == torch.from_numpy(v).dtype and single[k].numpy().tobytes() == v.tobytes(), k
        assert multi[k].numpy().tobytes() == v.tobytes(), k


def test_feature_table_with_multispeaker_fields(tmp_path):
    from parakeet_b200.data import FS2_MS_FIELDS, FeatureTable, fastspeech2_batch
    ex = _examples(True)
    data = []
    for i, e in enumerate(ex):
        row = dict(e, utt_id=f"u{i}", text=e["text"].tolist(), durations=e["durations"].tolist())
        for f in ("speech", "pitch", "energy"):
            np.save(tmp_path / f"{f}{i}.npy", e[f])
            row[f] = f"{f}{i}.npy"
        data.append(row)
    table = FeatureTable(data, fields=FS2_MS_FIELDS, root=str(tmp_path))
    batch = fastspeech2_batch([table[i] for i in range(3)])
    assert batch["spk_id"].tolist() == [4, 0, 4]
    assert torch.equal(batch["speech"], fastspeech2_batch(ex)["speech"])


def test_speaker_id_map_reader(tmp_path):
    from parakeet_b200.data import read_speaker_id_map
    p = tmp_path / "speaker_id_map.txt"
    p.write_text("SSB0005 0\nSSB0009 1\n\nSSB0011 2\n")
    m = read_speaker_id_map(str(p))
    assert m == {"SSB0005": 0, "SSB0009": 1, "SSB0011": 2} and list(m) == ["SSB0005", "SSB0009", "SSB0011"]
    bad = tmp_path / "bad.txt"
    bad.write_text("SSB0005\n")
    with pytest.raises(ValueError):
        read_speaker_id_map(str(bad))


def test_speaker_entry_points_are_exported_and_reject_bad_arguments():
    from parakeet_b200 import _lib
    L = _lib.lib()
    names = _lib.exported_symbols()
    for n in ("pk_spk_embed_fwd", "pk_spk_time_sum", "pk_spk_normalize_bwd", "pk_spk_table_grad"):
        assert n in names and hasattr(L, n), n
    buf = (ctypes.c_float * 64)()
    ids = (ctypes.c_int64 * 4)()
    p, pi = ctypes.cast(buf, ctypes.c_void_p), ctypes.cast(ids, ctypes.c_void_p)
    assert L.pk_spk_embed_fwd(None, 6, 8, pi, 4, 0, 1e-12, p, p, None) == -1
    assert L.pk_spk_embed_fwd(p, 0, 8, pi, 4, 0, 1e-12, p, p, None) == -1
    assert L.pk_spk_embed_fwd(p, 6, 8, pi, 4, 0, 0.0, p, p, None) == -1
    assert L.pk_spk_time_sum(p, 2, 3, 8, 4, 5, None, 0, p, None) == -1          # col0 + ncols > c
    assert L.pk_spk_time_sum(p, 2, 3, 8, 0, 8, p, 9, p, None) == -1             # dhs wider than the input
    assert L.pk_spk_time_sum(None, 2, 3, 8, 0, 8, None, 0, p, None) == -1
    assert L.pk_spk_normalize_bwd(p, p, None, pi, 4, 6, 0, 8, 1e-12, p, None) == -1
    assert L.pk_spk_normalize_bwd(p, p, p, pi, 0, 6, 0, 8, 1e-12, p, None) == -1
    assert L.pk_spk_table_grad(p, None, 4, 6, 8, 0, p, None) == -1
    assert L.pk_spk_table_grad(p, pi, 4, 0, 8, 0, p, None) == -1
    assert L.pk_spk_table_grad(p, pi, 4, 6, 8, 0, None, None) == -1 and b"NULL" in L.pk_last_error()


def test_training_step_refuses_cpu_models():
    from parakeet_b200 import _lib
    from parakeet_b200.training import FastSpeech2TrainStep
    m = _fs2ms.model("concat", _fs2ms.params("concat"), "cpu")
    with pytest.raises(_lib.PkError):
        FastSpeech2TrainStep(m)
