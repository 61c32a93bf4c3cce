"""Flat parameter / gradient buffers for the data-parallel training step.

The reference wraps the model in `paddle.DataParallel` (examples/fastspeech2/*/train.py:117-119), which all-reduces
gradients bucket by bucket.  Here every trainable tensor is a view into ONE flat fp32 buffer (and its gradient into a second
one), so the exchange step of the path is a single `all_reduce(SUM)` of the flat gradient and the optimiser (`FlatAdam`, the
one every training step uses) is a single kernel over the flat buffers; it also applies the 1/world scale of the DataParallel
mean.
Device-agnostic on purpose: the CPU tests run the buffers over gloo (tests/test_dist_cpu.py) and the optimiser's checkpoint
entries on the CPU (tests/test_flat_adam_cpu.py); only `FlatAdam.update` needs the library.
The rest is what every training step shares around its buffers: rank 0's broadcast at construction, the snapshot container of
`StandardUpdater` and the switch of the step's CUDA graphs.
"""
import os
from collections import OrderedDict

import torch
import torch.distributed as dist

from .. import _lib
from ..graph import GraphRunner
from ..ops import _ptr, _stream

BUFFERS = ("_mean", "_variance")      # BatchNorm running statistics: state-dict entries that are not trained


def step_graphs(max_graphs, use_graphs=None):
    """The GraphRunner that replays a training step's forward + backward: on when `use_graphs` says so, else unless
    PK_TRAIN_GRAPH=0 (PK_CUDA_GRAPHS=0 turns every graph off)."""
    on = os.environ.get("PK_TRAIN_GRAPH", "1") != "0" if use_graphs is None else bool(use_graphs)
    return GraphRunner(max_graphs=max_graphs, enabled=on)


def broadcast_from_rank0(flat, params, group=None):
    """paddle.DataParallel broadcasts rank 0's parameters and buffers at construction (examples/fastspeech2/*/train.py:117-119):
    the flat parameter buffer, then every BUFFERS entry of `params`."""
    dist.broadcast(flat, src=0, group=group)
    for k, v in params.items():
        if k.endswith(BUFFERS):
            dist.broadcast(v, src=0, group=group)


def updater_state(model, opt, lr, epoch=0):
    """StandardUpdater.state_dict's container {"main_params", "main_optimizer", "epoch", "iteration"}: Adam moments per
    parameter under Paddle's accumulator suffixes (FlatAdam.moments) plus the step count the bias correction needs."""
    o = opt.moments()
    o["step_count"] = opt.steps
    o["LR_Scheduler"] = {"last_lr": lr}
    return {"main_params": model.state_dict(), "main_optimizer": o, "epoch": int(epoch), "iteration": int(opt.steps)}


def load_updater_state(model, opt, state):
    model.set_state_dict(state["main_params"])                  # in place: the parameters stay views of the flat buffer
    o = state.get("main_optimizer", {})
    opt.load_moments(o)
    opt.steps = int(o.get("step_count", state.get("iteration", opt.steps)))


class FlatBuffers:
    def __init__(self, params: "OrderedDict[str, torch.Tensor]", names, device):
        """params: name -> tensor (replaced in place by views of the flat buffer for every name in `names`)."""
        sizes = [params[k].numel() for k in names]
        offs, tot = [], 0
        for s in sizes:
            offs.append(tot)
            tot += (s + 3) // 4 * 4                      # keep every view 16-byte aligned
        self.names, self.offsets, self.sizes, self.total = list(names), offs, sizes, tot
        self.flat = torch.zeros(tot, dtype=torch.float32, device=device)
        self.gflat = torch.zeros(tot, dtype=torch.float32, device=device)
        self.grads = {}
        for k, o, s in zip(names, offs, sizes):
            shape = params[k].shape
            self.flat[o:o + s].copy_(params[k].reshape(-1))
            params[k] = self.flat[o:o + s].view(shape)      # the model now reads the flat buffer
            self.grads[k] = self.gflat[o:o + s].view(shape)

    def all_reduce_grads(self, group=None):
        """The one exchange step of the path: SUM over ranks (the optimiser divides by the world size)."""
        if dist.is_initialized() and dist.get_world_size(group) > 1:
            dist.all_reduce(self.gflat, op=dist.ReduceOp.SUM, group=group)


class FlatAdam:
    """paddle.optimizer.Adam (with ClipGradByGlobalNorm when `clip_norm` is given) over one FlatBuffers: both moments are flat
    buffers of the same layout and one kernel updates everything.  `clip_norm` 0.0 keeps the clipping kernels and never clips."""

    def __init__(self, params, names, device, beta1=0.9, beta2=0.999, epsilon=1e-8, clip_norm=None):
        self.buffers = FlatBuffers(params, names, device)
        self.flat, self.gflat, self.grads = self.buffers.flat, self.buffers.gflat, self.buffers.grads
        self.m = torch.zeros_like(self.flat)
        self.v = torch.zeros_like(self.flat)
        self.beta1, self.beta2, self.epsilon, self.clip_norm = beta1, beta2, epsilon, clip_norm
        self.sq = torch.zeros(1, dtype=torch.float64, device=device) if clip_norm is not None else None    # squared gradient norm
        self.steps = 0

    def update(self, lr, world=1, group=None):
        """One update from the gradient in `gflat`: SUM over the ranks and the DataParallel mean when world > 1, then Adam."""
        L, n = _lib.lib(), self.flat.numel()
        if world > 1:
            self.buffers.all_reduce_grads(group)
        self.steps += 1
        grad_scale = 1.0 / world
        if self.clip_norm is not None:
            if world > 1:
                self.gflat.mul_(1.0 / world)             # the mean comes before the clip, like paddle
            grad_scale = 1.0
            self.sq.zero_()
            _lib.check(L.pk_sq_sum(_ptr(self.gflat), n, _ptr(self.sq), _stream()), "pk_sq_sum")
        _lib.check(L.pk_adam(_ptr(self.flat), _ptr(self.gflat), _ptr(self.m), _ptr(self.v), n, lr, self.beta1, self.beta2, self.epsilon,
                             self.steps, grad_scale, _ptr(self.sq), float(self.clip_norm or 0.0), _stream()), "pk_adam")

    def _views(self):
        b = self.buffers
        for k, o, n in zip(b.names, b.offsets, b.sizes):
            shape = b.grads[k].shape
            yield k + "_moment1_0", self.m[o:o + n].view(shape)
            yield k + "_moment2_0", self.v[o:o + n].view(shape)

    def moments(self):
        """The moments per parameter under Paddle's accumulator suffixes (`<name>_moment1_0`, `<name>_moment2_0`; Paddle prefixes
        them with its internal tensor names, which do not exist here, so the structured names are used)."""
        return {key: view.clone() for key, view in self._views()}

    def load_moments(self, opt):
        """The reverse of moments(); entries that `opt` lacks keep their values."""
        for key, view in self._views():
            if key in opt:
                view.copy_(torch.as_tensor(opt[key]).reshape(view.shape).to(view.device, view.dtype))


class PdCheckpoint:
    """The old-style `step-N.pdparams` / `step-N.pdopt` pair of ExperimentBase (utils/checkpoint.py:61-138) for a training step
    that holds its model as `self.m` and its optimiser as `self.opt` (a FlatAdam): the model's state dict, and the Adam state
    under Paddle's accumulator suffixes (`<name>_moment1_0`, `<name>_moment2_0`, `<name>_beta1_pow_acc_0`, `<name>_beta2_pow_acc_0`)."""

    step_count = property(lambda self: self.opt.steps)

    def state_dict(self):
        """(params, opt)."""
        opt = self.opt.moments()
        for k in self.opt.buffers.names:
            opt[k + "_beta1_pow_acc_0"] = torch.tensor([self.opt.beta1 ** self.step_count])
            opt[k + "_beta2_pow_acc_0"] = torch.tensor([self.opt.beta2 ** self.step_count])
        opt["step_count"] = self.step_count
        return self.m.state_dict(), opt

    def set_state_dict(self, params, opt=None):
        self.m.set_state_dict(params)                # in place: the parameters stay views of the flat buffer
        if opt:
            self.opt.load_moments(opt)
            self.opt.steps = int(opt.get("step_count", self.step_count))

    def save(self, checkpoint_dir, iteration=None):
        """Write step-N.pdparams and step-N.pdopt (N = iteration or the completed steps) and record it in checkpoint_dir/checkpoint."""
        from .. import checkpoint
        it = self.step_count if iteration is None else int(iteration)
        params, opt = self.state_dict()
        os.makedirs(checkpoint_dir, exist_ok=True)
        base = os.path.join(checkpoint_dir, f"step-{it}")
        checkpoint.save(params, base + ".pdparams")
        checkpoint.save(opt, base + ".pdopt")
        with open(os.path.join(checkpoint_dir, "checkpoint"), "w") as fh:
            fh.write(f"model_checkpoint_path: step-{it}")
        return base

    def load(self, checkpoint_dir, iteration=None):
        from .. import checkpoint
        if iteration is None:
            with open(os.path.join(checkpoint_dir, "checkpoint")) as fh:
                iteration = int(fh.read().strip().rsplit("-", 1)[-1])
        base = os.path.join(checkpoint_dir, f"step-{iteration}")
        self.set_state_dict(checkpoint.load(base + ".pdparams"), checkpoint.load(base + ".pdopt"))
        return int(iteration)
