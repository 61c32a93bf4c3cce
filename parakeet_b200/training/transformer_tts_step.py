"""TransformerTTS training step on H100 for the ljspeech recipe (reference: TransformerTTSUpdater.update_core /
TransformerTTSEvaluator.evaluate_core, parakeet/models/transformer_tts/transformer_tts_updater.py:73-170, :222; recipe
examples/transformer_tts/ljspeech/conf/default.yaml).

    forward in train mode (Dropout at every site with Philox masks that the backward regenerates - pk_dropout, keyed by the
    device step counter so that every graph replay draws fresh masks, the decoder prenet's always-on p = 0.5 included; postnet
    BatchNorm on the batch statistics of all B x Lmax rows)
    -> TransformerTTSLoss (masked L1 / L2, pos-weighted BCE on the stop logits) + GuidedMultiHeadAttentionLoss on the source
    attention of the last decoder layers -> backward -> mean all-reduce of the flat gradient over ranks -> paddle.optimizer.Adam.

The encoder is the FFT-block stack of training/transformer.py; each decoder layer (pre-LN causal self-attention, source attention
over the fused K | V memory of all layers, Linear feed-forward) calls its mha_fwd / mha_bwd.  The guided loss is folded into the
softmax backward of the guided layers (pk_softmax_bwd): dP of the selected heads gains lambda / N * G, and the loss's row
partials come out of the same pass.  The model's own `train()` keeps refusing; this class is the training entry point and
neither reads nor changes `model.training`.

Dropout sites (TransformerTrainOps.site; oracle/transformer_tts_train.py: dropout_site restates this numbering): stack 0 encoder,
1 decoder, 2 decoder prenet, 5 postnet; kind 0 positional encoding, 1 self-attention probabilities, 2 self-attention sub-layer
output, 3 feed-forward hidden, 4 feed-forward sub-layer output, 5 source-attention probabilities, 6 source-attention sub-layer
output (decoder) or postnet layer (stack 5), 7 prenet layer.
"""
import os

import torch
import torch.distributed as dist

from .. import _lib, ops
from ..models.transformer_tts import TransformerTTS
from ..ops import Split, _ptr, _stream
from . import wgrad
from .conv import ConvOps
from .flat import BUFFERS, FlatAdam, broadcast_from_rank0, load_updater_state, step_graphs, updater_state
from .transformer import TransformerTrainOps

_KEYS = ("text", "text_lengths", "speech", "speech_lengths")
P_PRENET = 0.5            # DecoderPrenet's F.dropout: always on, Paddle's default p, whatever dprenet_dropout_rate says
LOSS_NAMES = ("loss", "l1_loss", "l2_loss", "bce_loss", "enc_dec_attn_loss")


class TransformerTTSTrainStep(TransformerTrainOps):
    def __init__(self, model: TransformerTTS, learning_rate=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-8, use_masking=True,
                 use_weighted_masking=False, bce_pos_weight=5.0, loss_type="L1", use_guided_attn_loss=True,
                 modules_applied_guided_attn=("encoder-decoder",), guided_attn_loss_sigma=0.4, guided_attn_loss_lambda=1.0, dropout=True,
                 seed=0, process_group=None, use_graphs=None):
        """dropout: True -> the model's constructor rates, a dict of the reference's rate keywords to override some, False / None ->
        every transformer and postnet rate 0 (the decoder prenet's dropout stays on: the reference never turns it off).
        seed: base seed of the Philox masks; every rank should pass its own.  use_graphs: replay forward + backward as one CUDA
        graph per batch shape; None -> env PK_TRAIN_GRAPH (default on)."""
        if not isinstance(model, TransformerTTS):
            raise _lib.PkError("TransformerTTSTrainStep needs a parakeet_b200.models.TransformerTTS")
        if model.r != 1:
            raise NotImplementedError("reduction_factor != 1: the reference's guided attention loss is shape-inconsistent there "
                                      "(its olens are cut to a multiple of r, the attention has L / r query rows)")
        if use_weighted_masking:
            raise NotImplementedError("use_weighted_masking: the recipe masks (use_masking=True)")
        if not use_masking:
            raise NotImplementedError("use_masking=False: the losses are taken over the non-pad frames only")
        if loss_type not in ops.TTS_LOSS_TYPES:
            raise ValueError(f"unknown loss_type {loss_type!r} (L1, L2 or L1+L2)")
        mods = tuple(modules_applied_guided_attn or ()) if use_guided_attn_loss else ()
        other = [x for x in mods if x != "encoder-decoder"]
        if other:
            raise NotImplementedError(f"guided attention loss on {other}: only the source attention ('encoder-decoder') is covered; "
                                      "no recipe guides the encoder or decoder self-attention")
        if model.adim > 512:
            raise NotImplementedError("pk_layer_norm_bwd supports rows of at most 512 channels (adim)")
        if model.device.type != "cuda":
            raise _lib.PkError("training needs a CUDA device (no CPU fallback)")
        self.m, self.dev, self.group = model, model.device, process_group
        self.lr = learning_rate
        self.pos_weight, self.loss_type = float(bce_pos_weight), loss_type
        self.guided = bool(mods)
        self.sigma, self.lam = float(guided_attn_loss_sigma), float(guided_attn_loss_lambda)
        self.g_heads = min(model.num_heads_applied_guided_attn, model.aheads)
        self.g_layers = min(model.num_layers_applied_guided_attn, model.dlayers)
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        self.overlap = os.environ.get("PK_TRAIN_OVERLAP", "1") != "0"      # parameter gradients on a side stream (on_side)
        self._side, self._side_used, self._keep = None, False, []
        names = [k for k in model._params if not k.endswith(BUFFERS)]
        self.opt = opt = FlatAdam(model._params, names, self.dev, beta1, beta2, epsilon)
        self.buffers, self.flat, self.gflat, self.grads, self.adam_m, self.adam_v = opt.buffers, opt.flat, opt.gflat, opt.grads, opt.m, opt.v
        model._packed = None
        rates = dict(model.dropout_rates)
        if dropout is True:
            self.rates = rates
        elif isinstance(dropout, dict):
            self.rates = {**rates, **dropout}
        else:
            self.rates = {k: 0.0 for k in rates}
        self.seed = int(seed)
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self._graphs = step_graphs(4, use_graphs)          # a graph pins every saved activation of its batch shape
        self._zp = wgrad.ZeroPlanes(max_geoms=4, on_evict=self._graphs.drop)
        self.conv = ConvOps(self._zp)
        widest = max([model.odim, model.adim] + [int(v.shape[0]) for k, v in model._params.items() if k.startswith("postnet.")])
        self.sums = torch.zeros(max(4096, 2 * widest), dtype=torch.float32, device=self.dev)
        if self.world > 1:
            broadcast_from_rank0(self.flat, model._params, process_group)

    step_count = property(lambda self: self.opt.steps)

    # ------------------------------------------------------------------------------------------------------------
    # batch checks (host side)
    # ------------------------------------------------------------------------------------------------------------
    def _prepare(self, batch):
        if batch.get("spembs") is not None:
            raise NotImplementedError("spembs: TransformerTTS here has no speaker embedding")
        missing = [k for k in _KEYS if k not in batch]
        if missing:
            raise _lib.PkError(f"batch lacks {missing}")
        text, speech = batch["text"], batch["speech"]
        for k in _KEYS:
            if not torch.is_tensor(batch[k]) or not batch[k].is_cuda:
                raise _lib.PkError(f"batch[{k!r}] must be a CUDA tensor (no CPU fallback)")
        if text.dim() != 2 or speech.dim() != 3 or speech.shape[0] != text.shape[0] or speech.shape[2] != self.m.odim or speech.shape[1] < 1:
            raise _lib.PkError(f"text must be (B, T) and speech (B, L, {self.m.odim}) (got {tuple(text.shape)}, {tuple(speech.shape)})")
        B = text.shape[0]
        if tuple(batch["text_lengths"].shape) != (B,) or tuple(batch["speech_lengths"].shape) != (B,):
            raise _lib.PkError("text_lengths and speech_lengths must be (B,)")
        ts = [text.to(torch.int64).contiguous(), batch["text_lengths"].to(torch.int32).contiguous(), speech.float().contiguous(),
              batch["speech_lengths"].to(torch.int32).contiguous()]
        return ts, tuple(tuple(t.shape) for t in ts)

    # ------------------------------------------------------------------------------------------------------------
    # pieces
    # ------------------------------------------------------------------------------------------------------------
    def sub_fwd(self, ctx, name, x, rate, site):
        """x + dropout(Linear `name`(ctx)): the residual add rides in the GEMM epilogue when there is no dropout."""
        if rate > 0:
            y, _ = self.layer_fwd(ctx, name + ".weight", name + ".bias", "lin")
            self.drop(y, rate, site, inplace=True)
            ops.axpy_(1.0, x, y)
            return y
        return self.layer_fwd(ctx, name + ".weight", name + ".bias", "lin", residual=x)[0]

    def sub_bwd(self, dx, ctx, name, rate, site):
        """The gradient at the ctx input of sub_fwd (its weight / bias gradients written)."""
        dsub = self.drop(dx, rate, site)[0] if rate > 0 else dx
        return self.layer_bwd(dsub, ctx, name + ".weight", name + ".bias", "lin")

    def dec_layer_fwd(self, l, x, mem, olens, ilens):
        """DecoderLayer.forward (decoder_layer.py, pre-LN, concat_after=False) in train mode: x fp32 (B, L, A) -> (x', context)."""
        m, R = self.m, self.rates
        A, H = m.adim, m.aheads
        r_layer, r_self, r_src = R["transformer_dec_dropout_rate"], R["transformer_dec_attn_dropout_rate"], R["transformer_enc_dec_attn_dropout_rate"]
        q = f"decoder.decoders.{l}."
        c = dict(x0=x)
        _, c["h1"] = ops.layer_norm(x, self.P(q + "norm1.weight"), self.P(q + "norm1.bias"))
        bqkv = torch.cat([self.P(q + "self_attn.linear_q.bias"), self.P(q + "self_attn.linear_k.bias"), self.P(q + "self_attn.linear_v.bias")])
        _, qkv = self.conv.fwd(c["h1"], q + "qkv", self.wqkv(q), linear=True, bias=bqkv, out_f32=False, out_split=True)
        c["ctx1"], c["a1"] = self.mha_fwd(qkv, qkv, heads=H, dk=A // H, q_col0=0, k_col0=A, v_col0=2 * A, key_lens=olens, causal=True,
                                          rate=r_self, site=self.site(1, l, 1))
        c["x1"] = x1 = self.sub_fwd(c["ctx1"], q + "self_attn.linear_out", x, r_layer, self.site(1, l, 2))
        _, c["h2"] = ops.layer_norm(x1, self.P(q + "norm2.weight"), self.P(q + "norm2.bias"))
        _, qs = self.layer_fwd(c["h2"], q + "src_attn.linear_q.weight", q + "src_attn.linear_q.bias", "lin", out_f32=False, out_split=True)
        c["ctx2"], c["a2"] = self.mha_fwd(qs, mem, heads=H, dk=A // H, q_col0=0, k_col0=2 * A * l, v_col0=2 * A * l + A, key_lens=ilens,
                                          rate=r_src, site=self.site(1, l, 5))
        c["x2"] = x2 = self.sub_fwd(c["ctx2"], q + "src_attn.linear_out", x1, r_layer, self.site(1, l, 6))
        _, c["h3"] = ops.layer_norm(x2, self.P(q + "norm3.weight"), self.P(q + "norm3.bias"))
        _, c["u"] = self.layer_fwd(c["h3"], q + "feed_forward.w_1.weight", q + "feed_forward.w_1.bias", "lin", act="relu", out_f32=False,
                                   out_split=True)
        c["ud"] = self.drop(c["u"], r_layer, self.site(1, l, 3), out_f32=False, out_split=True)[1] if r_layer > 0 else c["u"]
        return self.sub_fwd(c["ud"], q + "feed_forward.w_2", x2, r_layer, self.site(1, l, 4)), c

    def dec_layer_bwd(self, l, dx, c, dmem, guided):
        """dx: gradient at the layer's output, updated in place to the gradient at its input; dmem (B, Tk, layers 2A) gains the
        layer's source-attention K / V gradient in its own columns."""
        m, R = self.m, self.rates
        A = m.adim
        r_layer = R["transformer_dec_dropout_rate"]
        q = f"decoder.decoders.{l}."
        B, L, _ = dx.shape
        du = self.sub_bwd(dx, c["ud"], q + "feed_forward.w_2", r_layer, self.site(1, l, 4))
        if r_layer > 0:
            self.drop(du, r_layer, self.site(1, l, 3), inplace=True)
        du_f, _ = ops.relu_bwd(du, c["u"], want_f32=True)
        dh3 = self.layer_bwd(du_f, c["h3"], q + "feed_forward.w_1.weight", q + "feed_forward.w_1.bias", "lin")
        ops.layer_norm_bwd(c["x2"], self.P(q + "norm3.weight"), dh3, dx, True, self.grads[q + "norm3.weight"], self.grads[q + "norm3.bias"])
        # source attention
        dctx = self.sub_bwd(dx, c["ctx2"], q + "src_attn.linear_out", r_layer, self.site(1, l, 6))
        dq = torch.zeros(B, L, A, dtype=torch.float32, device=self.dev)
        self.mha_bwd(Split.from_f32(dctx), c["a2"], dq, dmem, guided=guided)
        dh2 = self.layer_bwd(dq, c["h2"], q + "src_attn.linear_q.weight", q + "src_attn.linear_q.bias", "lin")
        ops.layer_norm_bwd(c["x1"], self.P(q + "norm2.weight"), dh2, dx, True, self.grads[q + "norm2.weight"], self.grads[q + "norm2.bias"])
        # causal self-attention
        dctx = self.sub_bwd(dx, c["ctx1"], q + "self_attn.linear_out", r_layer, self.site(1, l, 2))
        dqkv = torch.zeros(B, L, 3 * A, dtype=torch.float32, device=self.dev)
        self.mha_bwd(Split.from_f32(dctx), c["a1"], dqkv, dqkv)
        dh1 = self.qkv_bwd(q, dqkv, c["h1"], self.dev)
        ops.layer_norm_bwd(c["x0"], self.P(q + "norm1.weight"), dh1, dx, True, self.grads[q + "norm1.weight"], self.grads[q + "norm1.bias"])

    def wkv(self):
        """The source-attention K | V projections of every decoder layer as one Paddle Linear weight [A, layers 2A] and its bias."""
        src = [f"decoder.decoders.{l}.src_attn." for l in range(self.m.dlayers)]
        w = torch.cat([torch.cat([self.P(s + "linear_k.weight"), self.P(s + "linear_v.weight")], 1) for s in src], 1)
        b = torch.cat([torch.cat([self.P(s + "linear_k.bias"), self.P(s + "linear_v.bias")]) for s in src])
        return w, b

    def mem_bwd(self, dmem, hs_split):
        """Backward of the fused K | V projection: the per-layer weight / bias gradients on the side stream, returns d hs fp32."""
        m = self.m
        A, Lyr = m.adim, m.dlayers
        B, Tk, n = dmem.shape
        dms = Split.from_f32(dmem)
        w, _ = self.wkv()

        def param_grads(dmem=dmem, dms=dms, w=w):
            bsum = torch.zeros(n, dtype=torch.float32, device=self.dev)
            ops.colsum_(dmem.reshape(B * Tk, n), bsum)
            gw = self.conv.wgrad(hs_split, dms, w, linear=True)
            for l in range(Lyr):
                s = f"decoder.decoders.{l}.src_attn."
                for j, nm in enumerate(("linear_k", "linear_v")):
                    c0 = 2 * A * l + j * A
                    self.grads[s + nm + ".bias"].copy_(bsum[c0:c0 + A])
                    self.grads[s + nm + ".weight"].copy_(gw[:, c0:c0 + A])

        self.on_side(param_grads, dmem, dms, hs_split)
        return self.conv.dgrad(dms, "mem_kv", w, linear=True)

    # ------------------------------------------------------------------------------------------------------------
    # forward + losses + backward
    # ------------------------------------------------------------------------------------------------------------
    def _forward_backward(self, text, text_lens, ys, olens):
        m, R = self.m, self.rates
        L_ = _lib.lib()
        st = _stream()
        dev = self.dev
        A, H, odim = m.adim, m.aheads, m.odim
        self.conv.reset()
        self._zp.begin(tuple(tuple(t.shape) for t in (text, text_lens, ys, olens)))       # the graph key of step()
        self.gflat.zero_()
        B, Lm = ys.shape[0], ys.shape[1]
        # ---- encoder: Embedding + ScaledPositionalEncoding (+ dropout), the FFT blocks ----
        xs, ilens = ops.tts_text_eos(text, text_lens, m.eos)
        Tk = xs.shape[1]
        x = ops.embed_pe(xs, self.P("encoder.embed.0.weight"), None, self.P("encoder.embed.1.alpha"), None, m.padding_idx)
        if R["transformer_enc_positional_dropout_rate"] > 0:
            self.drop(x, R["transformer_enc_positional_dropout_rate"], self.site(0, 0, 0), inplace=True)
        _, hs_split, S_enc = self.stack_fwd(x, "encoder.", m.elayers, ilens, heads=H, ffn="conv", sid=0,
                                            r_layer=R["transformer_enc_dropout_rate"], r_attn=R["transformer_enc_attn_dropout_rate"])
        wkv, bkv = self.wkv()
        _, mem = self.conv.fwd(hs_split, "mem_kv", wkv, linear=True, bias=bkv, out_f32=False, out_split=True)
        # ---- decoder input: shifted frames -> prenet (always-on dropout) -> Linear -> + alpha pe (+ dropout) ----
        h = Split.from_f32(ops.tts_shift_frames(ys, 1))
        pre = []
        for i in range(m.dprenet_layers):
            q = f"decoder.embed.0.0.prenet.{i}.0."
            y, ysp = self.layer_fwd(h, q + "weight", q + "bias", "lin", act="relu", out_split=True)
            pre.append(dict(x=h, y=ysp))
            h = self.drop(y, P_PRENET, self.site(2, i, 7), out_f32=False, out_split=True)[1]
        pre_out = h
        xd, _ = self.layer_fwd(h, "decoder.embed.0.1.weight", "decoder.embed.0.1.bias", "lin")
        xd = ops.embed_pe(None, None, xd, self.P("decoder.embed.1.alpha"), None)
        if R["transformer_dec_positional_dropout_rate"] > 0:
            self.drop(xd, R["transformer_dec_positional_dropout_rate"], self.site(1, 0, 0), inplace=True)
        dec = []
        for l in range(m.dlayers):
            xd, c = self.dec_layer_fwd(l, xd, mem, olens, ilens)
            dec.append(c)
        _, zs = ops.layer_norm(xd, self.P("decoder.after_norm.weight"), self.P("decoder.after_norm.bias"))
        before, before_split = self.layer_fwd(zs, "feat_out.weight", "feat_out.bias", "lin", out_split=True)
        logits, _ = self.layer_fwd(zs, "prob_out.weight", "prob_out.bias", "lin")
        logits = logits.reshape(B, Lm)
        # ---- postnet: Conv1D -> train-mode BatchNorm1D (-> tanh) -> Dropout, over all B x Lmax rows ----
        post, hp, rows = [], before_split, B * Lm
        for i in range(m.postnet_layers):
            last = i == m.postnet_layers - 1
            q = f"postnet.postnet.{i}.1."
            conv_out, _ = self.layer_fwd(hp, f"postnet.postnet.{i}.0.weight", None, "conv")
            cdim = conv_out.shape[-1]
            y = torch.empty_like(conv_out)
            ysplit = Split.empty(tuple(conv_out.shape), dev) if not last else None
            mean, rstd = torch.empty(cdim, device=dev), torch.empty(cdim, device=dev)
            _lib.check(L_.pk_batch_norm_train(_ptr(conv_out), rows, cdim, _ptr(self.P(q + "weight")), _ptr(self.P(q + "bias")), 1e-5,
                                              0 if last else 2, 0.9, _ptr(m._params[q + "_mean"]), _ptr(m._params[q + "_variance"]),
                                              _ptr(self.sums), _ptr(y), _ptr(ysplit.hi) if ysplit else None,
                                              _ptr(ysplit.lo) if ysplit else None, _ptr(mean), _ptr(rstd), st), "pk_batch_norm_train")
            yd = y
            if R["postnet_dropout_rate"] > 0:
                yd, ysplit = self.drop(y, R["postnet_dropout_rate"], self.site(5, i, 6), out_f32=True, out_split=not last)
            post.append(dict(x=hp, conv=conv_out, y=y, yd=yd, mean=mean, rstd=rstd))
            hp = ysplit
        after = before.clone()
        if post:
            ops.axpy_(1.0, post[-1]["yd"], after)
        # ---- losses and their gradients ----
        labels = ops.tts_stop_labels(olens, Lm)
        losses = ops.tts_loss(before, after, ys, logits, labels, olens, self.pos_weight, self.loss_type)
        g_before, g_after, g_logits = ops.tts_loss_bwd(before, after, ys, logits, labels, olens, self.pos_weight, self.loss_type)
        # ---- backward: postnet ----
        g = g_after
        for i in reversed(range(m.postnet_layers)):
            last = i == m.postnet_layers - 1
            c = post[i]
            q = f"postnet.postnet.{i}.1."
            cdim = c["conv"].shape[-1]
            dconv = torch.empty_like(c["conv"])
            if R["postnet_dropout_rate"] > 0:
                g = self.drop(g, R["postnet_dropout_rate"], self.site(5, i, 6))[0]
            _lib.check(L_.pk_batch_norm_bwd(_ptr(c["conv"]), _ptr(g), _ptr(c["y"]), _ptr(c["mean"]), _ptr(c["rstd"]), _ptr(self.P(q + "weight")),
                                            0 if last else 2, rows, cdim, _ptr(self.sums), _ptr(dconv), st), "pk_batch_norm_bwd")
            self.grads[q + "bias"].copy_(self.sums[:cdim])
            self.grads[q + "weight"].copy_(self.sums[cdim:2 * cdim])
            g = self.layer_bwd(dconv, c["x"], f"postnet.postnet.{i}.0.weight", None, "conv")
        if post:
            ops.axpy_(1.0, g_after, g)                          # after = before + postnet(before)
            ops.axpy_(1.0, g_before, g)
        else:
            g = g_before.clone()
            ops.axpy_(1.0, g_after, g)
        dzs = self.layer_bwd(g, zs, "feat_out.weight", "feat_out.bias", "lin")
        ops.axpy_(1.0, self.layer_bwd(g_logits.reshape(B, Lm, 1), zs, "prob_out.weight", "prob_out.bias", "lin"), dzs)
        # ---- decoder ----
        dx = torch.empty_like(dzs)
        ops.layer_norm_bwd(xd, self.P("decoder.after_norm.weight"), dzs, dx, False, self.grads["decoder.after_norm.weight"],
                           self.grads["decoder.after_norm.bias"])
        dmem = torch.zeros(B, Tk, 2 * A * m.dlayers, dtype=torch.float32, device=dev)
        partials = torch.zeros(max(self.g_layers, 1), B, max(self.g_heads, 1), Lm, dtype=torch.float32, device=dev)
        for l in reversed(range(m.dlayers)):
            j = m.dlayers - 1 - l                    # the reference concatenates the guided layers from the last one down
            guided = None
            if self.guided and j < self.g_layers and self.g_heads > 0:
                guided = dict(heads=self.g_heads, layers=self.g_layers, ilens=ilens, olens=olens, sigma=self.sigma, lam=self.lam,
                              partials=partials[j])
            self.dec_layer_bwd(l, dx, dec[l], dmem, guided)
        if self.guided and self.g_heads > 0:
            ops.tts_guided_loss(partials, ilens, olens, Lm, Tk, self.g_heads * self.g_layers, self.lam, losses)
        if R["transformer_dec_positional_dropout_rate"] > 0:
            self.drop(dx, R["transformer_dec_positional_dropout_rate"], self.site(1, 0, 0), inplace=True)
        _lib.check(L_.pk_embed_pe_bwd(None, _ptr(dx), 0, 0, B, Lm, A, None, _ptr(self.grads["decoder.embed.1.alpha"]), st), "pk_embed_pe_bwd")
        g = self.layer_bwd(dx, pre_out, "decoder.embed.0.1.weight", "decoder.embed.0.1.bias", "lin")
        for i in reversed(range(m.dprenet_layers)):
            q = f"decoder.embed.0.0.prenet.{i}.0."
            self.drop(g, P_PRENET, self.site(2, i, 7), inplace=True)
            g, _ = ops.relu_bwd(g, pre[i]["y"], want_f32=True)
            g = self.layer_bwd(g, pre[i]["x"], q + "weight", q + "bias", "lin", need_dx=i > 0)
        # ---- encoder ----
        dhs = self.mem_bwd(dmem, hs_split)
        dxe = self.stack_bwd(dhs, S_enc)
        if R["transformer_enc_positional_dropout_rate"] > 0:
            self.drop(dxe, R["transformer_enc_positional_dropout_rate"], self.site(0, 0, 0), inplace=True)
        _lib.check(L_.pk_embed_pe_bwd(_ptr(xs), _ptr(dxe), m.idim, m.padding_idx, B, Tk, A, _ptr(self.grads["encoder.embed.0.weight"]),
                                      _ptr(self.grads["encoder.embed.1.alpha"]), st), "pk_embed_pe_bwd")
        self.join_side()
        return losses

    def _named(self, losses):
        out = {k: losses[i] for i, k in enumerate(LOSS_NAMES)}
        if not self.guided:
            del out["enc_dec_attn_loss"]
        out["encoder_alpha"] = self.P("encoder.embed.1.alpha")[0].clone()
        out["decoder_alpha"] = self.P("decoder.embed.1.alpha")[0].clone()
        return out

    def forward_backward(self, batch):
        """Losses and the flat gradient (self.grads: name -> view), no update and no graph; the running statistics move."""
        ts, _ = self._prepare(batch)
        return self._named(self._forward_backward(*ts))

    def evaluate(self, batch):
        """TransformerTTSEvaluator.evaluate_core: the eval-mode forward (running statistics, the prenet's position-keyed masks
        drawn from `seed`) and the same losses.  Changes nothing."""
        (text, text_lens, ys, olens), _ = self._prepare(batch)
        m = self.m
        B, Lm = ys.shape[0], ys.shape[1]
        after, before, logits, att = m._forward(text, text_lens, ys, olens, self.seed, want_att=self.guided)
        labels = ops.tts_stop_labels(olens, Lm)
        losses = ops.tts_loss(before.contiguous(), after.contiguous(), ys, logits.contiguous(), labels, olens, self.pos_weight, self.loss_type)
        if self.guided and self.g_heads > 0:
            Tk = att.shape[-1]
            partials = torch.zeros(self.g_layers, B, self.g_heads, Lm, dtype=torch.float32, device=self.dev)
            ilens = text_lens + 1
            zero = torch.zeros(B * m.aheads, Lm, Tk, dtype=torch.float32, device=self.dev)
            for j in range(self.g_layers):          # the loss's partial sums from the guided softmax backward on dP = 0
                p = Split.from_f32(att[:, m.dlayers - 1 - j].reshape(B * m.aheads, Lm, Tk))
                ops.softmax_bwd(p, zero, Tk, 1.0, dict(heads=self.g_heads, layers=self.g_layers, ilens=ilens, olens=olens, sigma=self.sigma,
                                                       lam=self.lam, partials=partials[j]))
            ops.tts_guided_loss(partials, ilens, olens, Lm, Tk, self.g_heads * self.g_layers, self.lam, losses)
        return self._named(losses)

    def step(self, batch):
        """One update: forward + backward (one CUDA graph per batch shape: eager the first time a shape is seen, captured the
        second, replayed afterwards), the flat all-reduce when data-parallel, Adam.  Returns the losses as device scalars."""
        ts, key = self._prepare(batch)
        self._zp.touch(key)                      # a replay does not pass through _forward_backward: keep the LRU order honest
        losses = self._graphs.run(key, self._forward_backward, ts).clone()
        self.opt.update(self.lr, self.world, self.group)
        self.step_dev += 1
        self.m._packed = None            # inference re-packs the updated weights and running statistics
        return self._named(losses)

    # ------------------------------------------------------------------------------------------------------------
    # snapshot / resume: the container of StandardUpdater.state_dict, as the other steps write it
    # ------------------------------------------------------------------------------------------------------------
    def state_dict(self, epoch=0):
        return updater_state(self.m, self.opt, self.lr, epoch)

    def set_state_dict(self, state):
        load_updater_state(self.m, self.opt, state)
        self.step_dev.fill_(self.step_count)
        self.conv.reset()

    def save(self, path, epoch=0):
        from .. import checkpoint
        checkpoint.save(self.state_dict(epoch), path)

    def load(self, path):
        from .. import checkpoint
        self.set_state_dict(checkpoint.load(path))
