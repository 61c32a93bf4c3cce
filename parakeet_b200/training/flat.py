"""Flat parameter / gradient buffers for the data-parallel training step, and what every training step shares around them.

The reference wraps the model in `paddle.DataParallel` (examples/fastspeech2/*/train.py:117-119), which all-reduces
gradients bucket by bucket.  Here every trainable tensor is a view into ONE flat fp32 buffer (and its gradient into a second
one), so the exchange step of the path is a single `all_reduce(SUM)` of the flat gradient and the optimiser (`FlatAdam`, the
one every training step uses) is a single kernel over the flat buffers; it also applies the 1/world scale of the DataParallel
mean.
Device-agnostic on purpose: the CPU tests run the buffers over gloo (tests/test_dist_cpu.py), the optimiser's checkpoint
entries (tests/test_flat_adam_cpu.py) and the graph / zero-plane owner `StepGraphs` (tests/test_graph_cpu.py) on the CPU; only
`FlatAdam.update` needs the library.
`TrainStep` is the base of the FastSpeech2, SpeedySpeech, TransformerTTS, WaveFlow and GE2E steps: set-up (FlatAdam, rank 0's
broadcast), the CUDA graphs of the forward + backward with their zero planes, and the three entry points `forward_backward`,
`forward_backward_graphed` and `step`.  `UpdaterSnapshot` (the `StandardUpdater` container) and `PdCheckpoint` (the old-style
pair) are the two snapshot formats.
"""
import os
from collections import OrderedDict

import torch
import torch.distributed as dist

from .. import _lib
from ..graph import GraphRunner
from ..ops import _ptr, _stream
from .conv import ConvOps
from .wgrad import ZeroPlanes

BUFFERS = ("_mean", "_variance")      # BatchNorm running statistics: state-dict entries that are not trained


def _train_graphs_on(use_graphs):
    return os.environ.get("PK_TRAIN_GRAPH", "1") != "0" if use_graphs is None else bool(use_graphs)


def step_graphs(max_graphs, use_graphs=None):
    """The GraphRunner that replays a training step's forward + backward: on when `use_graphs` says so, else unless
    PK_TRAIN_GRAPH=0 (PK_CUDA_GRAPHS=0 turns every graph off).  PWGTrainStep's; the other steps own a StepGraphs."""
    return GraphRunner(max_graphs=max_graphs, enabled=_train_graphs_on(use_graphs))


class StepGraphs(GraphRunner):
    """The CUDA graphs of a training step's forward + backward, one per batch shape, and the zero planes baked into them
    (`planes`, wgrad.ZeroPlanes), filed under the same key.  `run` makes the key's planes current (most recently used) before it
    runs the function eagerly or through its graph; evicting a key's planes beyond `max_graphs` drops the graph of that key,
    whose kernels hold the planes' addresses.  Switched like step_graphs."""

    def __init__(self, max_graphs, use_graphs=None):
        super().__init__(max_graphs=max_graphs, enabled=_train_graphs_on(use_graphs))
        self.planes = ZeroPlanes(max_geoms=max_graphs, on_evict=self.drop)

    def run(self, key, fn, inputs, graph=True):
        self.planes.begin(key)
        return super().run(key, fn, inputs) if graph else fn(*inputs)


def need_cuda(model):
    if model.device.type != "cuda":
        raise _lib.PkError("training needs a CUDA device (no CPU fallback)")


def broadcast_from_rank0(flat, params, group=None):
    """paddle.DataParallel broadcasts rank 0's parameters and buffers at construction (examples/fastspeech2/*/train.py:117-119):
    the flat parameter buffer, then every BUFFERS entry of `params`."""
    dist.broadcast(flat, src=0, group=group)
    for k, v in params.items():
        if k.endswith(BUFFERS):
            dist.broadcast(v, src=0, group=group)


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
    """The old-style `step-N.pdparams` / `step-N.pdopt` pair of ExperimentBase (utils/checkpoint.py:61-138) for a TrainStep: the
    model's state dict, and the Adam state under Paddle's accumulator suffixes (`<name>_moment1_0`, `<name>_moment2_0`, `<name>_beta1_pow_acc_0`, `<name>_beta2_pow_acc_0`)."""

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


class UpdaterSnapshot:
    """StandardUpdater.state_dict's container {"main_params", "main_optimizer", "epoch", "iteration"} (training/updaters/
    standard_updater.py; the Snapshot extension writes it with paddle.save as snapshot_iter_<n>.pdz) for a training step that
    holds self.m, self.opt (a FlatAdam) and self.lr: the Adam moments per parameter under Paddle's accumulator suffixes
    (FlatAdam.moments) plus the step count the bias correction needs.  train.py resumes by constructing the updater first and
    loading afterwards, which is why Layer.set_state_dict copies IN PLACE into the flat buffer."""

    def state_dict(self, epoch=0):
        o = self.opt.moments()
        o["step_count"] = self.opt.steps
        o["LR_Scheduler"] = {"last_lr": self.lr}
        return {"main_params": self.m.state_dict(), "main_optimizer": o, "epoch": int(epoch), "iteration": int(self.opt.steps)}

    def set_state_dict(self, state):
        self.m.set_state_dict(state["main_params"])
        o = state.get("main_optimizer", {})
        self.opt.load_moments(o)
        self.opt.steps = int(o.get("step_count", state.get("iteration", self.opt.steps)))
        if hasattr(self, "step_dev"):
            self.step_dev.fill_(self.opt.steps)      # the dropout masks continue from the restored step

    def save(self, path, epoch=0):
        from .. import checkpoint
        checkpoint.save(self.state_dict(epoch), path)

    def load(self, path):
        from .. import checkpoint
        self.set_state_dict(checkpoint.load(path))


class TrainStep:
    """The base of a training step.  A subclass runs its own refusals, then this constructor, and provides
    `_prepare(batch) -> (tensors, key)` (host-side checks and the device tensors of the batch; `key` names its shape) and
    `_forward_backward(*tensors)` (losses on the device, every gradient in gflat; a step that runs ConvOps and accumulates into
    gflat calls `_prologue()` first).

    Construction refuses a non-CUDA model, turns the model's trainable tensors (every state-dict entry but the BatchNorm running
    statistics) into views of FlatAdam's flat buffer and broadcasts rank 0's parameters under data parallelism.
    `max_graphs`: the CUDA graphs kept (a graph pins every saved activation of its batch shape); `use_graphs`: None -> env
    PK_TRAIN_GRAPH (default on).  A graph replays forward + backward as one launch per batch shape: eager the first time a shape
    is seen, captured the second, replayed afterwards."""

    def __init__(self, model, learning_rate, process_group, max_graphs, use_graphs=None, **adam):
        need_cuda(model)
        self.m, self.dev, self.lr, self.group = model, model.device, learning_rate, process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.opt = FlatAdam(model._params, [k for k in model._params if not k.endswith(BUFFERS)], self.dev, **adam)
        opt = self.opt
        self.buffers, self.flat, self.gflat, self.grads, self.adam_m, self.adam_v = opt.buffers, opt.flat, opt.gflat, opt.grads, opt.m, opt.v
        self._graphs = StepGraphs(max_graphs, use_graphs)
        self._zp = self._graphs.planes
        self.conv = ConvOps(self._zp)
        model._packed = None
        if self.world > 1:
            broadcast_from_rank0(self.flat, model._params, process_group)

    step_count = property(lambda self: self.opt.steps)

    def _prologue(self):
        """Every forward + backward packs the weights of its own step (inside a captured graph the pack kernels are part of the
        graph) and accumulates into a zeroed gradient."""
        self.conv.reset()
        self.gflat.zero_()

    def _named(self, out):
        """The result of forward_backward and step, from the outputs of _forward_backward."""
        return out

    def _run(self, batch, graph):
        tensors, key = self._prepare(batch)
        return self._graphs.run(key, self._forward_backward, tensors, graph=graph)

    def forward_backward(self, batch):
        """Forward + backward, eager and without an update: the losses, and every gradient in self.grads."""
        return self._named(self._run(batch, graph=False))

    def forward_backward_graphed(self, batch):
        """Forward + backward through the CUDA graph of the batch's shape, without an update: the outputs of _forward_backward,
        the graph's own tensors (valid until its next replay)."""
        return self._run(batch, graph=True)

    def step(self, batch):
        """One update: forward + backward through the graph of the batch's shape, the flat all-reduce when data-parallel, Adam.
        Returns the losses as device tensors, the values before the update."""
        out = self._run(batch, graph=True).clone()
        self._update()
        return self._named(out)

    def _update(self):
        """The update after a forward + backward: the one exchange step of the path, then Adam with the 1/world mean folded in."""
        self.opt.update(self.lr, self.world, self.group)
        if hasattr(self, "step_dev"):
            self.step_dev += 1           # the next step's dropout masks
        self.m._packed = None            # inference re-packs the updated weights and running statistics
