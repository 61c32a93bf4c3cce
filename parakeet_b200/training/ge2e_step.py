"""GE2E speaker-encoder training step on H100 (reference: examples/ge2e/train.py:62-75 `Ge2eExperiment.train_batch`):
`loss, eer = model(specs, speakers_per_batch)`, `loss.backward()`, `model.do_gradient_ops()` (similarity w / b gradients times
0.01), `Adam(1e-4, grad_clip=ClipGradByGlobalNorm(3))`.

Forward: per layer one `pk_conv_gemm` (input half of the gates over all steps) and one persistent `pk_lstm_fwd` that keeps the
post-activation gates and every c_t; Linear + ReLU, normalisation, then `pk_ge2e_loss` with its backward (the 0.01 applied in
the kernel).  Backward: `pk_ge2e_embed_bwd`, the Linear's data / weight gradients, then per layer (top down) one persistent
`pk_lstm_bwd` and the weight gradients of W_hh / W_ih as split-K GEMMs over the time-major operands (K = B * T; h_{t-1} for all
t is slabs 0 .. T-1 of the layer's h buffer), the data gradient into the layer below as one `pk_conv_gemm`.  None of these
kernels uses atomics, so loss and gradients are bit-reproducible; the clip's global norm is FlatAdam's shared `pk_sq_sum`, whose
per-block double atomics can move its last bit when the clip is active.  Parameters, gradients and Adam moments are `FlatAdam`'s
flat buffers.
"""

import torch
import torch.distributed as dist

from .. import _lib, ops
from ..models.lstm_speaker_encoder import lstm_key, start_states
from ..ops import Split
from .conv import ConvOps
from .flat import FlatAdam, PdCheckpoint, broadcast_from_rank0, step_graphs
from .wgrad import ZeroPlanes


class GE2ETrainStep(PdCheckpoint):
    def __init__(self, model, learning_rate=1e-4, max_grad_norm=3.0, num_speakers=64, beta1=0.9, beta2=0.999, epsilon=1e-8,
                 process_group=None):
        if model.device.type != "cuda":
            raise _lib.PkError("training needs a CUDA device (no CPU fallback)")
        self.m, self.lr, self.num_speakers = model, learning_rate, num_speakers
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.opt = FlatAdam(model._params, list(model._params), model.device, beta1, beta2, epsilon, clip_norm=max_grad_norm)
        self.flat, self.gflat, self.grads = self.opt.flat, self.opt.gflat, self.opt.grads
        self._graphs = step_graphs(2)
        self._zp = ZeroPlanes(max_geoms=2, on_evict=self._graphs.drop)
        self.conv = ConvOps(self._zp)
        self._perm = ops.lstm_gate_perm(model.hidden_size, model.device)
        model._packed = None
        if self.world > 1:
            broadcast_from_rank0(self.flat, model._params, process_group)

    def _n(self, specs):
        m = self.m
        if not specs.is_cuda:
            raise _lib.PkError("GE2ETrainStep needs CUDA tensors (no CPU fallback)")
        if specs.dim() != 3 or specs.shape[2] != m.n_mels or specs.shape[1] < 1:
            raise ValueError(f"expected specs (B, T, {m.n_mels}), got {tuple(specs.shape)}")
        n = self.num_speakers
        if n is None:
            raise ValueError("num_speakers (the recipe's speakers_per_batch) is needed for the forward's reshape")
        return n, m.grouping(specs.shape[0], m.output_size, n)

    def forward_backward(self, specs):
        """-> (loss (1,), similarity matrix (N*M', N)); the gradients (after do_gradient_ops) are left in self.grads."""
        N, Mg = self._n(specs)
        m, P, G = self.m, self.m._params, self.grads
        B, T, _ = specs.shape
        H, dev = m.hidden_size, specs.device
        self.conv.reset()
        self._zp.begin((B, T))
        self.gflat.zero_()
        inp = specs.float().transpose(0, 1).contiguous().reshape(1, T * B, m.n_mels)          # time-major
        counters = ops.lstm_counters(B, T, dev)
        perm = self._perm
        saved = []
        for l in range(m.num_layers):
            xs = Split.from_f32(inp)
            w_ih = P[lstm_key(l, "weight_ih")].unsqueeze(-1)
            g_in = self.conv.fwd(xs, ("ih", l), w_ih, bias=P[lstm_key(l, "bias_ih")])[0]
            h_all, h_split, c_all = start_states(T, B, H, dev, keep_c=True)
            gates = torch.empty(T, B, 4 * H, dtype=torch.float32, device=dev)
            ops.lstm_fwd(g_in.reshape(T, B, 4 * H), P[lstm_key(l, "bias_hh")], ops.lstm_pack_fwd(P[lstm_key(l, "weight_hh")], perm), h_all,
                         h_split, c_all, gates, counters)
            saved.append((xs, h_all, h_split, c_all, gates))
            inp = h_all[1:].reshape(1, T * B, H)
        hs = Split.from_f32(h_all[T].reshape(1, B, H))
        e = self.conv.fwd(hs, "lin", P["linear.weight"], linear=True, bias=P["linear.bias"], act="relu")[0].reshape(B, m.output_size)
        y = ops.l2_normalize_axis1(e)
        loss, sim, dy, dw, db = ops.ge2e_loss(y, N, Mg, N, P["similarity_weight"], P["similarity_bias"], want_grads=True)
        G["similarity_weight"].copy_(dw)
        G["similarity_bias"].copy_(db)
        dz = ops.ge2e_embed_bwd(e, dy)
        dzs = Split.from_f32(dz.reshape(1, B, m.output_size))
        self.conv.wgrad(hs, dzs, P["linear.weight"], linear=True, out=G["linear.weight"])
        ops.sum_slices(dz, G["linear.bias"])          # bias gradients: fixed-order row sums (pk_colsum accumulates with atomics)
        dh_last = self.conv.dgrad(dzs, "lin", P["linear.weight"], linear=True).reshape(B, H)
        dh_in = None
        dc = torch.empty(B, H, dtype=torch.float32, device=dev)
        per_row = torch.empty(B, 4 * H, dtype=torch.float32, device=dev)
        for l in reversed(range(m.num_layers)):
            xs, h_all, h_split, c_all, gates = saved[l]
            dgates = torch.empty(T, B, 4 * H, dtype=torch.float32, device=dev)
            dgs = Split.empty((1, T * B, 4 * H), dev)
            ops.lstm_bwd(ops.lstm_pack_bwd(P[lstm_key(l, "weight_hh")]), gates, c_all, dh_in, dh_last if dh_in is None else None, dgates,
                         dgs, dc, counters)
            h_prev = Split(h_split.hi[:T].reshape(1, T * B, H), h_split.lo[:T].reshape(1, T * B, H))     # h_{t-1} for every t
            self.conv.wgrad(h_prev, dgs, P[lstm_key(l, "weight_hh")].unsqueeze(-1), out=G[lstm_key(l, "weight_hh")].unsqueeze(-1))
            w_ih = P[lstm_key(l, "weight_ih")].unsqueeze(-1)
            self.conv.wgrad(xs, dgs, w_ih, out=G[lstm_key(l, "weight_ih")].unsqueeze(-1))
            ops.sum_slices(ops.sum_slices(dgates, per_row), G[lstm_key(l, "bias_ih")])      # over t, then over rows
            G[lstm_key(l, "bias_hh")].copy_(G[lstm_key(l, "bias_ih")])
            if l > 0:
                dh_in = self.conv.dgrad(dgs, ("ih", l), w_ih).reshape(T, B, H)
        return loss, sim

    def forward_backward_graphed(self, specs):
        return self._graphs.run(tuple(specs.shape), lambda s: self.forward_backward(s), [specs])

    def step(self, specs, eer=False):
        """One train_batch: forward, GE2E loss, backward, do_gradient_ops, clipped Adam.  Returns the loss (device tensor (1,),
        the value before the update), and with eer=True also the batch's EER (one device -> host copy)."""
        N, Mg = self._n(specs)
        loss, sim = self.forward_backward_graphed(specs.contiguous().float())
        out_eer = None
        if eer:
            from ..models.lstm_speaker_encoder import equal_error_rate
            out_eer = equal_error_rate(sim.cpu().numpy(), N, Mg)
        self.opt.update(self.lr, self.world, self.group)
        self.m._packed = None
        return (loss.clone(), out_eer) if eer else loss.clone()
