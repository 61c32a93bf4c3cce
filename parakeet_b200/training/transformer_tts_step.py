"""TransformerTTS training step on H100 for the ljspeech recipe (reference: TransformerTTSUpdater.update_core /
TransformerTTSEvaluator.evaluate_core, parakeet/models/transformer_tts/transformer_tts_updater.py:73-170, :222; recipe
examples/transformer_tts/ljspeech/conf/default.yaml).

    forward in train mode (Dropout at every site with Philox masks that the backward regenerates - pk_dropout, keyed by the
    device step counter so that every graph replay draws fresh masks, the decoder prenet's always-on p = 0.5 included; postnet
    BatchNorm on the batch statistics of all B x Lmax rows)
    -> TransformerTTSLoss (masked L1 / L2, pos-weighted BCE on the stop logits) + GuidedMultiHeadAttentionLoss on the source
    attention of the last decoder layers -> backward -> mean all-reduce of the flat gradient over ranks -> paddle.optimizer.Adam.

The encoder is the FFT-block stack of training/transformer.py; each decoder layer is that stack's pre-LN self-attention block
(causal) and feed-forward block (Linear) around a source attention over the fused K | V memory of all layers (mha_fwd / mha_bwd);
the postnet is training/transformer.py's as well.  The guided loss is folded into the
softmax backward of the guided layers (pk_softmax_bwd): dP of the selected heads gains lambda / N * G, and the loss's row
partials come out of the same pass.  The model's own `train()` keeps refusing; this class is the training entry point and
neither reads nor changes `model.training`.

Dropout sites (TransformerTrainOps.site; oracle/transformer_tts_train.py: dropout_site restates this numbering): stack 0 encoder,
1 decoder, 2 decoder prenet, 5 postnet; kind 0 positional encoding, 1 self-attention probabilities, 2 self-attention sub-layer
output, 3 feed-forward hidden, 4 feed-forward sub-layer output, 5 source-attention probabilities, 6 source-attention sub-layer
output (decoder) or postnet layer (stack 5), 7 prenet layer.
"""
import torch

from .. import _lib, ops
from ..models.transformer_tts import TransformerTTS
from ..ops import Split, _ptr, _stream
from .flat import UpdaterSnapshot
from .transformer import TransformerTrainOps

_KEYS = ("text", "text_lengths", "speech", "speech_lengths")
P_PRENET = 0.5            # DecoderPrenet's F.dropout: always on, Paddle's default p, whatever dprenet_dropout_rate says
LOSS_NAMES = ("loss", "l1_loss", "l2_loss", "bce_loss", "enc_dec_attn_loss")


class TransformerTTSTrainStep(UpdaterSnapshot, TransformerTrainOps):
    def __init__(self, model: TransformerTTS, learning_rate=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-8, use_masking=True,
                 use_weighted_masking=False, bce_pos_weight=5.0, loss_type="L1", use_guided_attn_loss=True,
                 modules_applied_guided_attn=("encoder-decoder",), guided_attn_loss_sigma=0.4, guided_attn_loss_lambda=1.0, dropout=True,
                 seed=0, process_group=None, use_graphs=None):
        """dropout, seed: TransformerTrainOps (False / None leaves the decoder prenet's dropout on: the reference never turns it
        off).  use_graphs: replay forward + backward as one CUDA graph per batch shape (TrainStep); None -> env PK_TRAIN_GRAPH
        (default on)."""
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
        self.pos_weight, self.loss_type = float(bce_pos_weight), loss_type
        self.guided = bool(mods)
        self.sigma, self.lam = float(guided_attn_loss_sigma), float(guided_attn_loss_lambda)
        self.g_heads = min(model.num_heads_applied_guided_attn, model.aheads)
        self.g_layers = min(model.num_layers_applied_guided_attn, model.dlayers)
        super().__init__(model, dropout, seed, learning_rate=learning_rate, process_group=process_group, max_graphs=4,
                         use_graphs=use_graphs, beta1=beta1, beta2=beta2, epsilon=epsilon)

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
    def dec_layer_fwd(self, l, x, mem, olens, ilens):
        """DecoderLayer.forward (decoder_layer.py, pre-LN, concat_after=False) in train mode: x fp32 (B, L, A) -> (x', context)."""
        m, R = self.m, self.rates
        A, H = m.adim, m.aheads
        r_layer, r_self, r_src = R["transformer_dec_dropout_rate"], R["transformer_dec_attn_dropout_rate"], R["transformer_enc_dec_attn_dropout_rate"]
        q, c = f"decoder.decoders.{l}.", {}
        c["x1"] = x1 = self.attn_fwd(x, q, olens, c, heads=H, causal=True, r_attn=r_self, r_layer=r_layer, sid=1, l=l)
        _, c["h2"] = ops.layer_norm(x1, self.P(q + "norm2.weight"), self.P(q + "norm2.bias"))
        _, qs = self.layer_fwd(c["h2"], q + "src_attn.linear_q.weight", q + "src_attn.linear_q.bias", "lin", out_f32=False, out_split=True)
        c["ctx2"], c["a2"] = self.mha_fwd(qs, mem, heads=H, dk=A // H, q_col0=0, k_col0=2 * A * l, v_col0=2 * A * l + A, key_lens=ilens,
                                          rate=r_src, site=self.site(1, l, 5))
        x2 = self.sub_fwd(c["ctx2"], q + "src_attn.linear_out", x1, r_layer, self.site(1, l, 6))
        return self.ffn_fwd(x2, q, "norm3", c, kind="lin", r_layer=r_layer, sid=1, l=l), c

    def dec_layer_bwd(self, l, dx, c, dmem, guided):
        """dx: gradient at the layer's output, updated in place to the gradient at its input; dmem (B, Tk, layers 2A) gains the
        layer's source-attention K / V gradient in its own columns."""
        m, R = self.m, self.rates
        A = m.adim
        r_layer = R["transformer_dec_dropout_rate"]
        q = f"decoder.decoders.{l}."
        B, L, _ = dx.shape
        self.ffn_bwd(dx, c, q, "norm3", kind="lin", r_layer=r_layer, sid=1, l=l)
        # source attention
        dctx = self.sub_bwd(dx, c["ctx2"], q + "src_attn.linear_out", r_layer, self.site(1, l, 6))
        dq = torch.zeros(B, L, A, dtype=torch.float32, device=self.dev)
        self.mha_bwd(Split.from_f32(dctx), c["a2"], dq, dmem, guided=guided)
        dh2 = self.layer_bwd(dq, c["h2"], q + "src_attn.linear_q.weight", q + "src_attn.linear_q.bias", "lin")
        ops.layer_norm_bwd(c["x1"], self.P(q + "norm2.weight"), dh2, dx, True, self.grads[q + "norm2.weight"], self.grads[q + "norm2.bias"])
        self.attn_bwd(dx, c, q, r_layer=r_layer, sid=1, l=l)

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
        self._prologue()
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
        after, post = self.postnet_fwd(before, before_split)
        # ---- losses and their gradients ----
        labels = ops.tts_stop_labels(olens, Lm)
        losses = ops.tts_loss(before, after, ys, logits, labels, olens, self.pos_weight, self.loss_type)
        g_before, g_after, g_logits = ops.tts_loss_bwd(before, after, ys, logits, labels, olens, self.pos_weight, self.loss_type)
        g = self.postnet_bwd(g_after, g_before, post)
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
