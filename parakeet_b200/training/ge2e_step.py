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

from .. import _lib, ops
from ..models.lstm_speaker_encoder import lstm_key, start_states
from ..ops import Split
from .flat import PdCheckpoint, TrainStep


class GE2ETrainStep(PdCheckpoint, TrainStep):
    def __init__(self, model, learning_rate=1e-4, max_grad_norm=3.0, num_speakers=64, beta1=0.9, beta2=0.999, epsilon=1e-8,
                 process_group=None):
        super().__init__(model, learning_rate, process_group, max_graphs=2, beta1=beta1, beta2=beta2, epsilon=epsilon,
                         clip_norm=max_grad_norm)
        self.num_speakers = num_speakers
        self._perm = ops.lstm_gate_perm(model.hidden_size, model.device)

    def _groups(self, B):
        """(N, M'): the speakers of the batch and the utterances per speaker."""
        return self.num_speakers, self.m.grouping(B, self.m.output_size, self.num_speakers)

    def _prepare(self, specs):
        m = self.m
        if not specs.is_cuda:
            raise _lib.PkError("GE2ETrainStep needs CUDA tensors (no CPU fallback)")
        if specs.dim() != 3 or specs.shape[2] != m.n_mels or specs.shape[1] < 1:
            raise ValueError(f"expected specs (B, T, {m.n_mels}), got {tuple(specs.shape)}")
        if self.num_speakers is None:
            raise ValueError("num_speakers (the recipe's speakers_per_batch) is needed for the forward's reshape")
        self._groups(specs.shape[0])                # raises for a batch the reference's reshape cannot group
        return [specs.contiguous().float()], tuple(specs.shape)

    def _forward_backward(self, specs):
        """-> (loss (1,), similarity matrix (N*M', N)); the gradients (after do_gradient_ops) are left in self.grads."""
        m, P, G = self.m, self.m._params, self.grads
        B, T, _ = specs.shape
        N, Mg = self._groups(B)
        H, dev = m.hidden_size, specs.device
        self._prologue()
        inp = specs.transpose(0, 1).contiguous().reshape(1, T * B, m.n_mels)          # time-major
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

    def step(self, specs, eer=False):
        """One train_batch: forward, GE2E loss, backward, do_gradient_ops, clipped Adam.  Returns the loss (device tensor (1,),
        the value before the update), and with eer=True also the batch's EER (one device -> host copy)."""
        loss, sim = self.forward_backward_graphed(specs)
        out_eer = None
        if eer:
            from ..models.lstm_speaker_encoder import equal_error_rate
            out_eer = equal_error_rate(sim.cpu().numpy(), *self._groups(specs.shape[0]))
        self._update()
        return (loss.clone(), out_eer) if eer else loss.clone()
