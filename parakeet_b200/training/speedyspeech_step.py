"""SpeedySpeech training step on H100 (reference: SpeedySpeechUpdater.update_core / SpeedySpeechEvaluator.evaluate_core,
parakeet/models/speedyspeech/speedyspeech_updater.py:48-85, :110-157; baker recipe examples/speedyspeech/baker/conf/default.yaml).

    forward in train mode (every BatchNorm1D takes its batch statistics over ALL B*T or B*L rows: nothing is masked, padded
    tokens and frames are live; the duration predictor reads encodings.detach())
    -> masked L1 + SSIM + Huber-on-log-durations -> backward -> mean all-reduce of the flat gradient over ranks
    -> paddle.optimizer.Adam with ClipGradByGlobalNorm (training/flat.py: FlatAdam).

The model's own forward / inference keep refusing training mode; the train-mode forward lives here, and the step neither reads
nor changes `model.training`.  Parameters, gradients and Adam moments are flat buffers (FlatAdam); the BatchNorm running
statistics stay the model's own tensors and are updated in place by pk_ss_bn_train_fwd.

Every Conv1D -> ReLU -> BatchNorm1D unit is pk_conv_gemm (bias + ReLU in its epilogue) followed by pk_ss_bn_train_fwd (statistics,
normalisation, the block's residual add, fp32 + split planes); its backward is pk_ss_bn_relu_bwd (dgamma, dbeta, the conv's bias
gradient, and the gradient at the conv's output as split planes), then the data gradient (pk_conv_gemm with flipped taps, the
block's residual gradient added in its epilogue) and the split-K weight gradient (training/wgrad.py: splitk_wgrad).  The losses and
their gradients are pk_ss_loss; the embedding tables' dense gradients are pk_spk_table_grad over the B*T tokens.
"""
import torch

from .. import _lib, ops
from ..models.speedyspeech import CHANNELS, SpeedySpeech, _i32, paddle_same_conv
from ..ops import Split, _ptr, _stream
from .flat import TrainStep, UpdaterSnapshot

_KEYS = ("phones", "tones", "num_phones", "num_frames", "feats", "durations")


class SpeedySpeechTrainStep(UpdaterSnapshot, TrainStep):
    def __init__(self, model: SpeedySpeech, learning_rate=2e-3, max_grad_norm=1.0, beta1=0.9, beta2=0.999, epsilon=1e-8,
                 process_group=None, check_durations=True):
        """check_durations: compare the longest row sum of batch["durations"] with feats.shape[1] on every call and raise PkError
        when they differ.  It is the step's only device->host copy; pass False once the data pipeline is trusted (a longer sum
        is then cut at feats.shape[1] frames and a shorter one leaves zero rows, as pk_length_regulate defines)."""
        if not isinstance(model, SpeedySpeech):
            raise _lib.PkError("SpeedySpeechTrainStep needs a parakeet_b200.models.SpeedySpeech")
        self.check_durations = check_durations
        # a falsy max_grad_norm never clips; a graph pins every saved activation of its batch shape
        super().__init__(model, learning_rate, process_group, max_graphs=4, beta1=beta1, beta2=beta2, epsilon=epsilon,
                         clip_norm=max_grad_norm or 0.0)
        self.one = torch.ones(1, device=self.dev)

    # ------------------------------------------------------------------------------------------------------------
    # batch checks (host side; nothing here can fault on the device)
    # ------------------------------------------------------------------------------------------------------------
    def _prepare(self, batch):
        missing = [k for k in _KEYS if k not in batch and k != "tones"]
        if missing:
            raise _lib.PkError(f"batch lacks {missing}")
        tones = batch.get("tones")
        if tones is not None and not self.m.tone_size:
            raise _lib.PkError("tones given to a SpeedySpeech built without tone_size")
        if tones is None and self.m.tone_size:
            raise _lib.PkError("this SpeedySpeech has a tone embedding: the batch needs tones")
        ts = {k: batch[k] for k in _KEYS if batch.get(k) is not None}
        for k, v in ts.items():
            if not torch.is_tensor(v) or not v.is_cuda:
                raise _lib.PkError(f"batch[{k!r}] must be a CUDA tensor (no CPU fallback)")
        phones, feats = ts["phones"], ts["feats"]
        if phones.dim() != 2 or feats.dim() != 3 or feats.shape[2] != self.m.odim or feats.shape[1] == 0 or phones.shape[1] == 0:
            raise _lib.PkError(f"phones must be (B, T) and feats (B, L, {self.m.odim}) (got {tuple(phones.shape)}, {tuple(feats.shape)})")
        B, T = phones.shape
        want = dict(durations=(B, T), num_phones=(B,), num_frames=(B,), feats=(B,) + tuple(feats.shape[1:]))
        if tones is not None:
            want["tones"] = (B, T)
        for k, shape in want.items():
            if tuple(ts[k].shape) != shape:
                raise _lib.PkError(f"batch[{k!r}] has shape {tuple(ts[k].shape)}, expected {shape}")
        L = feats.shape[1]
        dur = ts["durations"].to(torch.int64).contiguous()
        if self.check_durations:
            longest = int(dur.clamp(min=0).sum(1).max().item())
            if longest != L:
                raise _lib.PkError(f"the longest utterance's durations add up to {longest} frames but feats has {L}")
        out = [phones.to(torch.int64).contiguous(), dur, feats.float().contiguous(), _i32(ts["num_frames"]), _i32(ts["num_phones"])]
        if tones is not None:
            out.append(tones.to(torch.int64).contiguous())
        return out, (B, T, L, tones is not None)

    # ------------------------------------------------------------------------------------------------------------
    # GEMM-shaped pieces
    # ------------------------------------------------------------------------------------------------------------
    def P(self, name):
        return self.m._params[name]

    def workspace(self, rows, batch=0, l=0):
        """The kernels' fp32 workspace for one call.  Allocated by the call that uses it, never kept across calls: inside a graph
        capture it then belongs to that graph's memory pool and lives as long as the graph whose kernels hold its address."""
        return torch.empty(ops.ss_scratch_elems(rows, batch, l, self.m.odim), dtype=torch.float32, device=self.dev)

    def lin_fwd(self, xs, name, **kw):
        return self.conv.fwd(xs, name, self.P(name + ".weight"), linear=True, bias=self.P(name + ".bias"), **kw)

    def lin_bwd(self, dy, x_saved, name, need_dx=True):
        """dy fp32 (B, T, out) or its Split; x_saved Split (B, T, in): writes the weight / bias gradients, returns dx fp32."""
        w = self.P(name + ".weight")
        dys = dy if isinstance(dy, Split) else ops.split_pad8(dy)
        ops.colsum_split_(dys, w.shape[1], self.grads[name + ".bias"])
        self.conv.wgrad(x_saved, dys, w, linear=True, out=self.grads[name + ".weight"])
        return self.conv.dgrad(dys, name, w, linear=True) if need_dx else None

    # ------------------------------------------------------------------------------------------------------------
    # ResidualBlock (speedyspeech.py:21-39) in training mode
    # ------------------------------------------------------------------------------------------------------------
    def block_fwd(self, x, xs, pre, k, n):
        """x fp32 / xs Split (B, T, 128) -> (y fp32, y Split, saved context): n units, the input added to the last one."""
        _, left, _ = paddle_same_conv(k, 1)
        sc = self._ws
        units, hs = [], xs
        for j in range(n):
            q = f"{pre}blocks.{j}."
            r, _ = self.conv.fwd(hs, q, self.P(q + "0.weight"), bias=self.P(q + "0.bias"), pad=left, act="relu")
            last = j == n - 1
            y, ys, mean, rstd = ops.ss_bn_train_fwd(r, self.P(q + "2.weight"), self.P(q + "2.bias"), self.P(q + "2._mean"),
                                                    self.P(q + "2._variance"), sc, residual=x if last else None, want_f32=last)
            units.append(dict(q=q, x=hs, r=r, mean=mean, rstd=rstd))
            hs = ys
        return y, hs, dict(units=units, left=left)

    def block_bwd(self, dy, ctx, need_dx=True):
        """dy fp32: gradient at the block's output -> gradient at its input (the residual path included)."""
        left = ctx["left"]
        sc = self._ws
        g = dy
        for j in reversed(range(len(ctx["units"]))):
            u = ctx["units"][j]
            q = u["q"]
            _, drs = ops.ss_bn_relu_bwd(g, u["r"], u["mean"], u["rstd"], self.P(q + "2.weight"), sc, self.grads[q + "2.weight"],
                                        self.grads[q + "2.bias"], dbias=self.grads[q + "0.bias"])
            # tap pairs dY[t] with X[t + tap - left]: the 4-tap kernel pads one more row on the right
            w = self.P(q + "0.weight")
            self.conv.wgrad(u["x"], drs, w, pad=left, out=self.grads[q + "0.weight"])
            if j == 0 and not need_dx:
                return None
            g = self.conv.dgrad(drs, q, w, pad=left, residual=dy if j == 0 else None)
        return g

    # ------------------------------------------------------------------------------------------------------------
    # forward + losses + backward
    # ------------------------------------------------------------------------------------------------------------
    def _forward_backward(self, phones, dur, feats, num_frames, num_phones, tones=None):
        m, L_ = self.m, _lib.lib()
        st = _stream()
        B, T = phones.shape
        L = feats.shape[1]
        C = CHANNELS
        self._prologue()
        self._ws = sc = self.workspace(max(B * T, B * L), B, L)
        ek, dk = m.encoder_kernel_size, m.decoder_kernel_size
        # ---- encoder (:100-106) ----
        text_w = self.P("encoder.embedding.text_embedding.weight")
        emb = m._embed_ids(text_w, phones)
        if tones is not None:
            tone_w = self.P("encoder.embedding.tone_embedding.weight")
            ops.axpy_(1.0, m._embed_ids(tone_w, tones), emb)
        emb_s = Split.from_f32(emb)
        pre, pre_s = self.lin_fwd(emb_s, "encoder.prenet.0", act="relu", out_split=True)
        x, xs, enc_ctx = pre, pre_s, []
        for i in range(len(m.encoder_dilations)):
            x, xs, c = self.block_fwd(x, xs, f"encoder.res_blocks.{i}.", ek, 2)
            enc_ctx.append(c)
        enc_out_s = xs
        x1, _ = self.lin_fwd(xs, "encoder.postnet1.0", residual=pre)
        r1 = torch.empty_like(x1)
        _lib.check(L_.pk_leaky_relu(_ptr(x1), x1.numel(), 0.0, _ptr(r1), None, None, st), "pk_leaky_relu")
        q = "encoder.postnet2.1"
        _, bn_s, mean1, rstd1 = ops.ss_bn_train_fwd(r1, self.P(q + ".weight"), self.P(q + ".bias"), self.P(q + "._mean"),
                                                    self.P(q + "._variance"), sc, want_f32=False)
        enc, enc_s = self.lin_fwd(bn_s, "encoder.postnet2.2", out_split=True)
        # ---- duration predictor on encodings.detach() (:109-118, :178) ----
        h, hs, dur_ctx = enc, enc_s, []
        for i, k in enumerate((4, 3, 1)):
            h, hs, c = self.block_fwd(h, hs, f"duration_predictor.layers.{i}.", k, 1)
            dur_ctx.append(c)
        pred = self.lin_fwd(hs, "duration_predictor.layers.3")[0].reshape(B, T)
        dur_hs = hs
        # ---- expand, position encoding, decoder (:134-138, :180-184) ----
        x0, _ = ops.length_regulate(enc, dur, L)
        x0 = ops.embed_pe(None, None, x0, self.one, None)
        x, xs, dec_ctx = x0, Split.from_f32(x0), []
        for i in range(len(m.decoder_dilations)):
            x, xs, c = self.block_fwd(x, xs, f"decoder.res_blocks.{i}.", dk, 2)
            dec_ctx.append(c)
        x2, x2s = self.lin_fwd(xs, "decoder.postnet1.0", residual=x0, out_split=True)
        _, hs2, post_ctx = self.block_fwd(x2, x2s, "decoder.postnet2.0.", dk, 2)
        decoded, _ = self.lin_fwd(hs2, "decoder.postnet2.1")
        # ---- losses and their gradients (update_core :57-80) ----
        losses, g_dec, g_dur = ops.ss_loss(decoded, feats, num_frames, pred, dur, num_phones, sc)
        # ---- backward: decoder ----
        g = self.lin_bwd(g_dec, hs2, "decoder.postnet2.1")
        dx2 = self.block_bwd(g, post_ctx)
        g = self.lin_bwd(dx2, xs, "decoder.postnet1.0")
        for c in reversed(dec_ctx):
            g = self.block_bwd(g, c)
        ops.axpy_(1.0, dx2, g)                                # x0 feeds the blocks and postnet1's residual; the encoding add is identity
        denc = torch.empty(B, T, C, dtype=torch.float32, device=self.dev)
        _lib.check(L_.pk_length_regulate_bwd(_ptr(g), _ptr(dur), B, T, C, L, _ptr(denc), st), "pk_length_regulate_bwd")
        # ---- duration predictor: its input is detached, so nothing flows into the encoder from here ----
        g = self.lin_bwd(g_dur.reshape(B, T, 1), dur_hs, "duration_predictor.layers.3")
        for i in reversed(range(3)):
            g = self.block_bwd(g, dur_ctx[i], need_dx=i > 0)
        # ---- encoder ----
        g = self.lin_bwd(denc, bn_s, "encoder.postnet2.2")
        dx1, dx1s = ops.ss_bn_relu_bwd(g, r1, mean1, rstd1, self.P(q + ".weight"), sc, self.grads[q + ".weight"], self.grads[q + ".bias"],
                                       want_f32=True)
        g = self.lin_bwd(dx1s, enc_out_s, "encoder.postnet1.0")
        for c in reversed(enc_ctx):
            g = self.block_bwd(g, c)
        ops.axpy_(1.0, dx1, g)                                # prenet output feeds the blocks and postnet1's residual
        _, dpre_s = ops.relu_bwd(g, pre_s)
        demb = self.lin_bwd(dpre_s, emb_s, "encoder.prenet.0")
        ops.spk_table_grad(demb.reshape(B * T, C), phones.reshape(-1), self.grads["encoder.embedding.text_embedding.weight"], 0)
        if tones is not None:
            ops.spk_table_grad(demb.reshape(B * T, C), tones.reshape(-1), self.grads["encoder.embedding.tone_embedding.weight"], 0)
        self._ws = None
        return losses

    @staticmethod
    def _named(losses):
        return dict(loss=losses[0], l1_loss=losses[1], duration_loss=losses[2], ssim_loss=losses[3])

    def evaluate(self, batch):
        """SpeedySpeechEvaluator.evaluate_core (:110-157): the eval-mode forward (running statistics) and the same four numbers.
        Reads the current parameters; changes nothing, the model's `training` flag included."""
        (phones, dur, feats, num_frames, num_phones, *tones), (B, T, L, _) = self._prepare(batch)
        enc, pred = self.m._stage_a(phones, tones[0] if tones else None, None)
        decoded = self.m._stage_b(enc, dur, L, None)
        sc = self.workspace(0, B, L)
        losses, _, _ = ops.ss_loss(decoded.contiguous(), feats, num_frames, pred.contiguous(), dur, num_phones, sc, want_grads=False)
        return self._named(losses)
