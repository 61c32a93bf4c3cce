"""N > 1 path on CPU: world_size-2 gloo processes shard a ragged batch, 'synthesise' their slice and gather."""
import os
import socket

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from parakeet_b200.parallel import gather_variable, pad_batch, shard_indices


def test_shard_indices_partition_and_balance():
    lengths = [60, 140, 83, 71, 100, 97, 133, 65, 120]
    for world in (1, 2, 4, 8):
        parts = [shard_indices(lengths, world, r) for r in range(world)]
        flat = sorted(i for p in parts for i in p)
        assert flat == list(range(len(lengths)))                       # a partition: every utterance exactly once
        sizes = [len(p) for p in parts]
        assert max(sizes) - min(sizes) <= 1
        if world == 2:
            tot = [sum(lengths[i] for i in p) for p in parts]
            assert abs(tot[0] - tot[1]) <= max(lengths)


def test_pad_batch():
    seqs = [torch.arange(3), torch.arange(5), torch.arange(1)]
    x, lens = pad_batch(seqs)
    assert x.tolist() == [[0, 1, 2, 0, 0], [0, 1, 2, 3, 4], [0, 0, 0, 0, 0]] and lens.tolist() == [3, 5, 1]


def _worker(rank, world, port, lengths, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        mine = shard_indices(lengths, world, rank)
        # stand-in for FastSpeech2 -> PWG on this rank's slice: a deterministic function of (index, length)
        results = [torch.full((lengths[i] * 3,), float(i)) for i in mine]
        full = gather_variable(results, mine, len(lengths))
        ok = all(full[i].shape[0] == lengths[i] * 3 and float(full[i][0]) == float(i) for i in range(len(lengths)))
        # max-over-ranks timing reduction used by bench.py
        t = torch.tensor([10.0 + rank], dtype=torch.float64)
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        q.put((rank, ok, float(t.item()), mine))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_shard_and_gather():
    lengths = [60, 140, 83, 71, 100, 97, 133]
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, lengths, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = [q.get(timeout=120) for _ in procs]
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    assert all(ok for _, ok, _, _ in out)
    assert all(abs(tmax - 11.0) < 1e-9 for _, _, tmax, _ in out)
    assert sorted(i for _, _, _, mine in out for i in mine) == list(range(len(lengths)))


def _train_exchange_worker(rank, world, port, q):
    """The exchange step of the training path (FastSpeech2TrainStep.step): flat gradient all-reduce + Adam with 1/world."""
    from collections import OrderedDict

    from oracle.fastspeech2 import adam_step
    from parakeet_b200.training import FlatBuffers
    from parakeet_b200.training.flat import broadcast_from_rank0
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(0)                          # same initial weights on every rank
        params = OrderedDict(w1=torch.randn(5, 3, generator=g), b1=torch.randn(5, generator=g), bn_mean=torch.zeros(5),
                             w2=torch.randn(2, 5, 3, generator=g))
        fb = FlatBuffers(params, ["w1", "b1", "w2"], "cpu")           # buffers (bn_mean) stay out of the flat buffer
        assert params["w1"].data_ptr() == fb.flat.data_ptr() and fb.total == 16 + 8 + 32
        params["bn_variance"] = torch.ones(5)
        w1 = params["w1"].clone()
        if rank:                                                      # rank 0's parameters and BatchNorm buffers win
            fb.flat.add_(1.0)
            params["bn_mean"].fill_(3.0)
            params["bn_variance"].fill_(3.0)
        broadcast_from_rank0(fb.flat, params)
        bcast_ok = torch.equal(params["w1"], w1) and not params["bn_mean"].any() and params["bn_variance"].eq(1.0).all()
        grads = {}
        for r in range(world):                                        # what each rank's backward would have produced
            gr = torch.Generator().manual_seed(100 + r)
            grads[r] = {k: torch.randn(params[k].shape, generator=gr) for k in fb.names}
        for k in fb.names:
            fb.grads[k].copy_(grads[rank][k])
        fb.all_reduce_grads()
        mean = {k: sum(grads[r][k] for r in range(world)) / world for k in fb.names}
        ok = bool(bcast_ok) and all(torch.allclose(fb.grads[k] / world, mean[k], atol=1e-6) for k in fb.names)
        # Adam on the flat buffers with the DataParallel mean folded in as grad_scale = 1/world (what pk_adam does)
        new_p = adam_step({"flat": fb.flat}, {"flat": fb.gflat / world}, {}, 1e-3, 0.9, 0.999, 1e-8)["flat"]
        per_tensor = adam_step({k: params[k].clone() for k in fb.names}, mean, {}, 1e-3, 0.9, 0.999, 1e-8)
        fb.flat.copy_(new_p)
        # the flat update equals the per-tensor update with the mean gradient (padding lanes carry zero gradient)
        ok = ok and all(torch.allclose(params[k], per_tensor[k], atol=1e-7) for k in fb.names)
        # plain Python lists: a tensor on an mp queue is sent as a handle to shared storage that dies with this process
        q.put((rank, ok, params["w1"].tolist(), params["w2"].tolist()))
    finally:
        dist.destroy_process_group()


def test_two_rank_gloo_training_exchange():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_train_exchange_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    out = sorted([q.get(timeout=120) for _ in procs], key=lambda t: t[0])
    for p in procs:
        p.join(timeout=60)
    assert all(o[1] for o in out)
    # every rank applied the same update: replicas stay bit-identical, and the weights moved
    assert out[0][2] == out[1][2] and out[0][3] == out[1][3]
    g = torch.Generator().manual_seed(0)
    w1_init = torch.randn(5, 3, generator=g)
    w1_new = torch.tensor(out[0][2])
    assert not torch.equal(w1_new, w1_init) and (w1_new - w1_init).abs().max() < 2e-3   # |step| <= lr for the first Adam step
