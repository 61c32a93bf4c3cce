"""The caller side of the training step (SURVEY.md 8f.2 / 8f.4): the reference's dumped-feature dataset layout, its collate
function and its per-rank batch sampler, without Paddle / jsonlines.

* `dump/{train,dev,test}/norm/metadata.jsonl` (examples/fastspeech2/normalize.py:143-175): one JSON object per line with
  `utt_id, text (phone ids), text_lengths, speech_lengths, durations, speech / pitch / energy (paths of .npy files)`
  [+ `spk_id`]; features are z-scored float32 arrays: speech (L, n_mels), pitch (T,) or (T, 1), energy likewise.
* `DataTable(data, fields, converters={"speech": np.load, ...})` (parakeet/datasets/data_table.py:47-120): lazy per-example
  conversion -> `FeatureTable`.
* `fastspeech2_single_spk_batch_fn` (parakeet/datasets/am_batch_fn.py:60-99) with `batch_sequences`
  (parakeet/data/batch.py:170-189: pad along axis 0 with zeros to the longest example) -> `fastspeech2_batch`; the dict it
  returns is exactly what `FastSpeech2TrainStep.step` / `FastSpeech2.forward` take.
* `paddle.io.DistributedBatchSampler(dataset, batch_size, shuffle=True, drop_last=True)`
  (examples/fastspeech2/train.py:101-105) -> `DistributedBatchSampler`: restated from Paddle 2.1 (python/paddle/fluid/
  dataloader/batch_sampler.py); the index order cannot be checked against Paddle here - what the tests pin is the contract
  (every rank sees the same number of batches, ranks are disjoint, an epoch covers the data once up to the wrap-around pad).
"""
import json
import os

import numpy as np
import torch

FS2_FIELDS = ("text", "text_lengths", "speech", "speech_lengths", "durations", "pitch", "energy")
FS2_MS_FIELDS = FS2_FIELDS + ("spk_id",)          # the multi-speaker recipes (train.py:66-71)


def read_metadata(path):
    """metadata.jsonl -> list of dicts."""
    with open(path, "rt", encoding="utf-8") as f:
        return [json.loads(line) for line in f if line.strip()]


class FeatureTable:
    """DataTable: `data[i]` restricted to `fields`, with `converters[field]` applied on access (default for the FastSpeech2
    dump: np.load for speech / pitch / energy).  Relative paths are resolved against `root`."""

    def __init__(self, data, fields=FS2_FIELDS, converters=None, root=None):
        if not data:
            raise ValueError("empty metadata")
        missing = [f for f in fields if f not in data[0]]
        if missing:
            raise ValueError(f"fields {missing} are not in the data; fields in the data: {sorted(data[0])}")
        self.data, self.fields, self.root = data, tuple(fields), root
        self.converters = {"speech": self._load, "pitch": self._load, "energy": self._load} if converters is None else converters

    def _load(self, path):
        if self.root is not None and not os.path.isabs(path):
            path = os.path.join(self.root, path)
        return np.load(path, allow_pickle=False)

    def __len__(self):
        return len(self.data)

    def __getitem__(self, i):
        item = self.data[i]
        return {f: (self.converters[f](item[f]) if f in self.converters else item[f]) for f in self.fields}


def batch_sequences(sequences, pad_value=0):
    """parakeet/data/batch.py:170-189 for axis 0: zero-pad every array to the longest first dimension and stack."""
    n = max(s.shape[0] for s in sequences)
    out = np.full((len(sequences), n) + tuple(sequences[0].shape[1:]), pad_value, dtype=sequences[0].dtype)
    for i, s in enumerate(sequences):
        out[i, :s.shape[0]] = s
    return out


def read_speaker_id_map(path):
    """The recipe's `speaker_id_map.txt` (one `<speaker> <id>` pair per line; examples/fastspeech2/train.py:67-71, which takes
    num_speakers = the number of lines) -> dict speaker name -> int id, in file order.  num_speakers = len(result)."""
    out = {}
    with open(path, "rt", encoding="utf-8") as f:
        for n, line in enumerate(f, 1):
            parts = line.strip().split()
            if not parts:
                continue
            if len(parts) != 2:
                raise ValueError(f"{path}:{n}: expected '<speaker> <id>', got {line.strip()!r}")
            out[parts[0]] = int(parts[1])
    return out


def fastspeech2_batch(examples, device=None):
    """fastspeech2_single_spk_batch_fn (am_batch_fn.py:60-99): list of examples -> dict of tensors
    text (B, Tmax) i64, text_lengths (B,) i64, durations (B, Tmax) i64, speech (B, Lmax, n_mels) f32, speech_lengths (B,) i64,
    pitch / energy (B, Tmax, 1) f32 (a trailing feature axis is added to 1-D pitch / energy, the shape the model expects).
    When the examples carry `spk_id` (FeatureTable(..., fields=FS2_MS_FIELDS)) this is fastspeech2_multi_spk_batch_fn
    (am_batch_fn.py:102-145) and the dict also holds spk_id (B,) i64."""
    def feat(name):
        arrs = [np.asarray(e[name], dtype=np.float32) for e in examples]
        return [a[:, None] if a.ndim == 1 else a for a in arrs]
    text = batch_sequences([np.asarray(e["text"], dtype=np.int64) for e in examples])
    durations = batch_sequences([np.asarray(e["durations"], dtype=np.int64) for e in examples])
    batch = {
        "text": text, "text_lengths": np.asarray([e["text_lengths"] for e in examples], dtype=np.int64),
        "durations": durations, "speech": batch_sequences([np.asarray(e["speech"], dtype=np.float32) for e in examples]),
        "speech_lengths": np.asarray([e["speech_lengths"] for e in examples], dtype=np.int64),
        "pitch": batch_sequences(feat("pitch")), "energy": batch_sequences(feat("energy")),
    }
    if "spk_id" in examples[0]:
        batch["spk_id"] = np.asarray([e["spk_id"] for e in examples], dtype=np.int64).reshape(len(examples))
    out = {k: torch.from_numpy(v) for k, v in batch.items()}
    if device is not None:
        out = {k: v.to(device, non_blocking=True) for k, v in out.items()}
    return out


class DistributedBatchSampler:
    """Per-rank batches of indices: the (optionally shuffled, seed = epoch) index list is padded by wrap-around to a multiple
    of `nranks`, then dealt out in blocks of `batch_size`, block k going to rank k % nranks; the tail that does not fill
    `batch_size * nranks` is split evenly.  `drop_last` drops a rank's final short batch."""

    def __init__(self, n_samples, batch_size, nranks=1, rank=0, shuffle=False, drop_last=False):
        assert batch_size > 0 and 0 <= rank < nranks
        self.n, self.batch_size, self.nranks, self.rank = n_samples, batch_size, nranks, rank
        self.shuffle, self.drop_last, self.epoch = shuffle, drop_last, 0
        self.num_samples = (n_samples + nranks - 1) // nranks
        self.total_size = self.num_samples * nranks

    def set_epoch(self, epoch):
        self.epoch = epoch

    def _local_indices(self):
        idx = list(range(self.n))
        idx += idx[:self.total_size - len(idx)]
        if self.shuffle:
            np.random.RandomState(self.epoch).shuffle(idx)
            self.epoch += 1
        bs, nr = self.batch_size, self.nranks
        last = self.total_size % (bs * nr)
        local = []
        for i in range(self.rank * bs, len(idx) - last, bs * nr):
            local.extend(idx[i:i + bs])
        tail = idx[len(idx) - last:]
        per = last // nr
        local.extend(tail[self.rank * per:(self.rank + 1) * per])
        return local

    def __iter__(self):
        local = self._local_indices()
        for i in range(0, len(local), self.batch_size):
            b = local[i:i + self.batch_size]
            if len(b) == self.batch_size or not self.drop_last:
                yield b

    def __len__(self):
        full, rem = divmod(self.num_samples, self.batch_size)
        return full if (self.drop_last or rem == 0) else full + 1


def synthetic_fastspeech2_batch(seed, lengths, odim=80, idim=80, dur_range=(2, 12)):
    """LJSpeech-shaped synthetic teacher-forced batch (no dataset is reachable offline): phoneme ids U{1..V-2}, durations
    U{dur_range}, speech / pitch / energy N(0, 1), zero padded like fastspeech2_single_spk_batch_fn pads - the dict
    FastSpeech2TrainStep.step takes.  Used by bench.py (cfg 5) and scripts/bench_train.py."""
    import torch
    g = torch.Generator().manual_seed(int(seed))
    B, Tmax = len(lengths), max(lengths)
    text = torch.zeros(B, Tmax, dtype=torch.int64)
    ds = torch.zeros(B, Tmax, dtype=torch.int64)
    ps, es = torch.zeros(B, Tmax, 1), torch.zeros(B, Tmax, 1)
    for b, n in enumerate(lengths):
        text[b, :n] = torch.randint(1, idim - 1, (n,), generator=g)
        ds[b, :n] = torch.randint(dur_range[0], dur_range[1] + 1, (n,), generator=g)
        ps[b, :n] = torch.randn(n, 1, generator=g)
        es[b, :n] = torch.randn(n, 1, generator=g)
    olens = ds.sum(1)
    ys = torch.zeros(B, int(olens.max()), odim)
    for b in range(B):
        ys[b, :int(olens[b])] = torch.randn(int(olens[b]), odim, generator=g)
    return dict(text=text, text_lengths=torch.tensor(lengths, dtype=torch.int64), speech=ys, speech_lengths=olens, durations=ds,
                pitch=ps, energy=es)
