"""FastSpeech2 training step on H100 (reference: FastSpeech2Updater.update_core, parakeet/models/fastspeech2/
fastspeech2_updater.py:51-99; data-parallel set-up examples/fastspeech2/train.py:51-56,135-139).

    forward (train mode: BatchNorm uses batch statistics; Dropout at the reference's sites with Philox masks that the backward
    pass regenerates from (seed, step, site) - pk_dropout - so no mask is ever stored)
    -> FastSpeech2Loss (use_masking=True) -> backward -> mean all-reduce of the gradients over ranks (DataParallel)
    -> paddle.optimizer.Adam step.

All parameters live in ONE flat fp32 buffer (the model's state-dict entries are views into it), all gradients in a second
flat buffer: the data-parallel exchange is a single NCCL all-reduce of that buffer per step over NVLink, the 1/world
scale is folded into the fused Adam kernel (pk_adam; training/flat.py: FlatAdam).  Every FLOP runs in libparakeet_b200.so:
GEMM-shaped gradients (dgrad = conv with flipped taps, wgrad = dY^T X over the flattened batch x time axis - training/wgrad.py:
splitk_wgrad -, attention dQ/dK/dV/dP) reuse pk_conv_gemm on transposed split planes (pk_transpose_planes); the rest are the
row-wise kernels of train.cu.
torch is used for buffers, views, permutes / copies (layout plumbing) and torch.distributed.
"""
import torch

from .. import _lib, ops
from ..models.fastspeech2 import FastSpeech2, _i32
from ..ops import Split, _ptr, _stream
from .flat import UpdaterSnapshot, need_cuda
from .transformer import TransformerTrainOps

_KEYS = ("text", "text_lengths", "speech", "speech_lengths", "durations", "pitch", "energy")


class FastSpeech2TrainStep(UpdaterSnapshot, TransformerTrainOps):
    """Dropout sites (TransformerTrainOps.site; oracle/fastspeech2.py: dropout_site restates this numbering): stack 0 encoder,
    1 decoder, 2 pitch, 3 energy, 4 duration predictor, 5 postnet; kind 0 positional encoding, 1 attention probabilities,
    2 attention sub-layer output, 3 feed-forward hidden, 4 feed-forward sub-layer output, 5 predictor layer, 6 postnet layer;
    (6, 0, 7) / (6, 0, 8): pitch / energy embedding."""

    def __init__(self, model: FastSpeech2, learning_rate=1e-3, beta1=0.9, beta2=0.999, epsilon=1e-8,
                 stop_gradient_from_pitch_predictor=None, stop_gradient_from_energy_predictor=None, process_group=None,
                 dropout=True, seed=0, use_graphs=None):
        """dropout, seed: TransformerTrainOps.
        use_graphs: replay forward + backward as ONE CUDA graph per batch shape (TrainStep); None -> env PK_TRAIN_GRAPH (default
        on).  The step is host-bound otherwise (~700 launches of 10-40 us); bucketing samplers repeat shapes, so do synthetic
        benchmarks."""
        need_cuda(model)
        if model.tone_embed_dim is not None:
            raise NotImplementedError("the training step does not cover tone conditioning (tone_embed_dim): no recipe trains with tones")
        # multi-speaker recipes (aishell3, vctk): batch["spk_id"] -> spk_embedding_table -> F.normalize -> spk_projection
        self.spk = model.spk_embed_dim is not None
        self.sg_pitch = model.stop_gradient_from_pitch_predictor if stop_gradient_from_pitch_predictor is None else stop_gradient_from_pitch_predictor
        self.sg_energy = model.stop_gradient_from_energy_predictor if stop_gradient_from_energy_predictor is None else stop_gradient_from_energy_predictor
        super().__init__(model, dropout, seed, learning_rate=learning_rate, process_group=process_group, max_graphs=16,
                         use_graphs=use_graphs, beta1=beta1, beta2=beta2, epsilon=epsilon)

    _fb_graphs = property(lambda self: self._graphs)         # the name this step has always given its graphs

    def _prepare(self, batch):
        """The batch's tensors on the device in _forward_backward's order (+ spk_id for speaker models: a replay reads the ids of
        the current batch), and their shapes as the graph key."""
        if batch.get("spembs") is not None:
            raise NotImplementedError("training with utterance-level speaker embeddings (spembs) is not supported: the recipes pass spk_id")
        if self.spk and batch.get("spk_id") is None:
            raise ValueError("this model has a speaker embedding table: the batch needs spk_id (int64, (B,))")
        dev = self.dev
        text = batch["text"].to(dev, torch.int64).contiguous()
        B, T = text.shape
        ts = [text, _i32(batch["text_lengths"].to(dev)), batch["speech"].to(dev, torch.float32).contiguous(), _i32(batch["speech_lengths"].to(dev)),
              batch["durations"].to(dev, torch.int64).contiguous(), batch["pitch"].to(dev, torch.float32).reshape(B, T).contiguous(),
              batch["energy"].to(dev, torch.float32).reshape(B, T).contiguous()]
        if self.spk:
            ts.append(batch["spk_id"].to(dev, torch.int64).reshape(B).contiguous())
        return ts, tuple(tuple(t.shape) for t in ts)

    # ------------------------------------------------------------------------------------------------------------
    # predictors
    # ------------------------------------------------------------------------------------------------------------
    def pred_fwd(self, pre, n_layers, hs_split):
        sid, rate = {"pitch_predictor.": (2, self.rates["pitch_predictor_dropout"]), "energy_predictor.": (3, self.rates["energy_predictor_dropout"]),
                     "duration_predictor.": (4, self.rates["duration_predictor_dropout_rate"])}[pre]
        saved, h = [], hs_split
        for i in range(n_layers):
            y, ys = self.layer_fwd(h, f"{pre}conv.{i}.0.weight", f"{pre}conv.{i}.0.bias", "conv", act="relu", out_split=True)
            _, hn = ops.layer_norm(y, self.P(f"{pre}conv.{i}.2.weight"), self.P(f"{pre}conv.{i}.2.bias"))
            if rate > 0:
                hn = self.drop(hn, rate, self.site(sid, i, 5), out_f32=False, out_split=True)[1]
            saved.append(dict(x=h, y=y, ys=ys))
            h = hn
        out, _ = self.layer_fwd(h, pre + "linear.weight", pre + "linear.bias", "lin")
        return out, dict(layers=saved, h_last=h, pre=pre, sid=sid, rate=rate)

    def pred_bwd(self, dout, S, need_dx=True):
        pre = S["pre"]
        g = self.layer_bwd(dout, S["h_last"], pre + "linear.weight", pre + "linear.bias", "lin")
        n = len(S["layers"])
        for i in reversed(range(n)):
            c = S["layers"][i]
            if S["rate"] > 0:
                self.drop(g, S["rate"], self.site(S["sid"], i, 5), inplace=True)
            dy = torch.empty_like(g)
            ops.layer_norm_bwd(c["y"], self.P(f"{pre}conv.{i}.2.weight"), g, dy, False, self.grads[f"{pre}conv.{i}.2.weight"],
                               self.grads[f"{pre}conv.{i}.2.bias"])
            dpre, _ = ops.relu_bwd(dy, c["ys"], want_f32=True)
            g = self.layer_bwd(dpre, c["x"], f"{pre}conv.{i}.0.weight", f"{pre}conv.{i}.0.bias", "conv", need_dx=(i > 0 or need_dx))
        return g

    # ------------------------------------------------------------------------------------------------------------
    # speaker conditioning (fastspeech2.py:395-401, _integrate_with_spk_embed :560-590): hs' is computed on every Tmax row -
    # the padded rows are live (bias + projected speaker), the predictors' convolutions read them and they get gradient
    # ------------------------------------------------------------------------------------------------------------
    def spk_fwd(self, hs, hs_split, spk_id):
        m = self.m
        B, T, A = hs.shape
        e, norms = ops.spk_embed_fwd(self.P("spk_embedding_table.weight"), spk_id, m.padding_idx)
        S = dict(ids=spk_id, e=e, norms=norms)
        if m.spk_embed_integration_type == "add":
            S["e_split"] = Split.from_f32(e.reshape(B, 1, -1))
            proj, _ = self.layer_fwd(S["e_split"], "spk_projection.weight", "spk_projection.bias", "lin")
            hs2 = hs.clone()
            ops.axpy_(1.0, proj.expand(B, T, A).contiguous(), hs2)
            return hs2, Split.from_f32(hs2), S
        S["cat"] = Split.from_f32(torch.cat([hs, e.unsqueeze(1).expand(B, T, e.shape[1])], dim=-1))          # layout only
        hs2, hs2_split = self.layer_fwd(S["cat"], "spk_projection.weight", "spk_projection.bias", "lin", out_split=True)
        return hs2, hs2_split, S

    def spk_bwd(self, dhs2, S):
        """dhs2: gradient w.r.t. hs' (fp32 (B, T, A)).  Writes the projection's and the table's gradients, returns d hs."""
        m = self.m
        B, T, A = dhs2.shape
        D = m.spk_embed_dim
        if m.spk_embed_integration_type == "add":
            dproj, _ = ops.spk_time_sum(dhs2, 0, A)                                  # the broadcast over time, all Tmax rows
            de = self.layer_bwd(dproj.reshape(B, 1, A), S["e_split"], "spk_projection.weight", "spk_projection.bias", "lin")
            dhs = dhs2
        else:
            dcat = self.layer_bwd(dhs2, S["cat"], "spk_projection.weight", "spk_projection.bias", "lin")
            de, dhs = ops.spk_time_sum(dcat, A, D, dhs_cols=A)                       # one pass over the (B, T, A + D) gradient
        dx = ops.spk_normalize_bwd(S["e"], S["norms"], de.reshape(B, D).contiguous(), S["ids"], m.num_speakers, m.padding_idx)
        ops.spk_table_grad(dx, S["ids"], self.grads["spk_embedding_table.weight"], m.padding_idx)
        return dhs

    # ------------------------------------------------------------------------------------------------------------
    # one training step
    # ------------------------------------------------------------------------------------------------------------
    def _forward_backward(self, text, ilens, ys, olens, ds, ps, es, spk_id=None):
        m = self.m
        L = _lib.lib()
        st = _stream()
        dev = self.dev
        self._prologue()
        B, T = text.shape
        A, odim = m.adim, m.odim
        # ---- forward (train mode) ----
        R = self.rates
        x = ops.embed_pe(text, self.P("encoder.embed.0.weight"), None, self.P("encoder.embed.1.alpha"), None, m.padding_idx)
        if R["transformer_enc_positional_dropout_rate"] > 0:
            self.drop(x, R["transformer_enc_positional_dropout_rate"], self.site(0, 0, 0), inplace=True)
        ffn = "lin" if m._linear_ffn else "conv"
        hs, hs_split, S_enc = self.stack_fwd(x, "encoder.", m.elayers, ilens, heads=m.aheads, ffn=ffn, sid=0,
                                             r_layer=R["transformer_enc_dropout_rate"], r_attn=R["transformer_enc_attn_dropout_rate"])
        if self.spk:
            hs, hs_split, S_spk = self.spk_fwd(hs, hs_split, spk_id)
        p_raw, S_p = self.pred_fwd("pitch_predictor.", m.cfg["pitch"][0], hs_split)
        e_raw, S_e = self.pred_fwd("energy_predictor.", m.cfg["energy"][0], hs_split)
        d_raw, S_d = self.pred_fwd("duration_predictor.", m.cfg["dur"][0], hs_split)
        p_outs = ops.mask_rows_(p_raw.reshape(B, T).clone(), ilens)
        e_outs = ops.mask_rows_(e_raw.reshape(B, T).clone(), ilens)
        d_outs = ops.mask_rows_(d_raw.reshape(B, T).clone(), ilens)
        pe_w, ee_w = self.P("pitch_embed.0.weight"), self.P("energy_embed.0.weight")
        r_pe, r_ee = R["pitch_embed_dropout"], R["energy_embed_dropout"]
        if r_pe > 0 or r_ee > 0:
            # Sequential(Conv1D, Dropout) (fastspeech2.py:220-247): the two embeddings one at a time (the fused kernel with the
            # other embedding's weights zeroed), each through its own mask, then hs + e_embs + p_embs
            zw_p, zw_e = torch.zeros_like(pe_w.reshape(A, -1)), torch.zeros_like(ee_w.reshape(A, -1))
            zb, z0 = torch.zeros(A, device=dev), torch.zeros_like(hs)
            p_emb = ops.variance_embed_add(z0, ps, es, pe_w.reshape(A, -1), self.P("pitch_embed.0.bias"), zw_e, zb, None)
            e_emb = ops.variance_embed_add(z0, ps, es, zw_p, zb, ee_w.reshape(A, -1), self.P("energy_embed.0.bias"), None)
            if r_pe > 0:
                self.drop(p_emb, r_pe, self.site(6, 0, 7), inplace=True)
            if r_ee > 0:
                self.drop(e_emb, r_ee, self.site(6, 0, 8), inplace=True)
            hs2 = hs.clone()
            ops.axpy_(1.0, e_emb, hs2)
            ops.axpy_(1.0, p_emb, hs2)
        else:
            hs2 = ops.variance_embed_add(hs, ps, es, pe_w.reshape(A, -1), self.P("pitch_embed.0.bias"), ee_w.reshape(A, -1),
                                         self.P("energy_embed.0.bias"), None)
        t_dec = ys.shape[1]
        hs_lr, _ = ops.length_regulate(hs2, ds, t_dec)
        xd = ops.embed_pe(None, None, hs_lr, self.P("decoder.embed.0.alpha"), None)
        if R["transformer_dec_positional_dropout_rate"] > 0:
            self.drop(xd, R["transformer_dec_positional_dropout_rate"], self.site(1, 0, 0), inplace=True)
        zs, zs_split, S_dec = self.stack_fwd(xd, "decoder.", m.dlayers, olens, heads=m.aheads, ffn=ffn, sid=1,
                                             r_layer=R["transformer_dec_dropout_rate"], r_attn=R["transformer_dec_attn_dropout_rate"])
        before, before_split = self.layer_fwd(zs_split, "feat_out.weight", "feat_out.bias", "lin", out_split=True)
        after, post = self.postnet_fwd(before, before_split)
        # ---- loss and its gradient ----
        losses = torch.empty(4, dtype=torch.float32, device=dev)
        ws = torch.empty(12, dtype=torch.float32, device=dev)
        _lib.check(L.pk_fs2_loss(_ptr(before), _ptr(after), _ptr(ys), _ptr(olens), t_dec, odim, _ptr(d_outs), _ptr(ds), _ptr(p_outs), _ptr(ps),
                                 _ptr(e_outs), _ptr(es), _ptr(ilens), T, B, _ptr(ws), _ptr(losses), st), "pk_fs2_loss")
        g_before, g_after = torch.empty_like(before), torch.empty_like(after)
        g_d, g_p, g_e = torch.empty(B, T, 1, device=dev), torch.empty(B, T, 1, device=dev), torch.empty(B, T, 1, device=dev)
        _lib.check(L.pk_fs2_loss_bwd(_ptr(before), _ptr(after), _ptr(ys), _ptr(olens), t_dec, odim, _ptr(d_outs), _ptr(ds), _ptr(p_outs),
                                     _ptr(ps), _ptr(e_outs), _ptr(es), _ptr(ilens), T, B, _ptr(g_before), _ptr(g_after), _ptr(g_d), _ptr(g_p),
                                     _ptr(g_e), st), "pk_fs2_loss_bwd")
        # ---- backward ----
        g = self.postnet_bwd(g_after, g_before, post)
        dzs = self.layer_bwd(g, zs_split, "feat_out.weight", "feat_out.bias", "lin")
        dxd = self.stack_bwd(dzs, S_dec)
        if R["transformer_dec_positional_dropout_rate"] > 0:
            self.drop(dxd, R["transformer_dec_positional_dropout_rate"], self.site(1, 0, 0), inplace=True)
        _lib.check(L.pk_embed_pe_bwd(None, _ptr(dxd), 0, 0, B, t_dec, A, None, _ptr(self.grads["decoder.embed.0.alpha"]), st), "pk_embed_pe_bwd")
        dhs = torch.empty(B, T, A, dtype=torch.float32, device=dev)
        _lib.check(L.pk_length_regulate_bwd(_ptr(dxd), _ptr(ds), B, T, A, t_dec, _ptr(dhs), st), "pk_length_regulate_bwd")
        kp, ke = pe_w.shape[-1], ee_w.shape[-1]
        d_pe = self.drop(dhs, r_pe, self.site(6, 0, 7))[0] if r_pe > 0 else dhs
        d_ee = self.drop(dhs, r_ee, self.site(6, 0, 8))[0] if r_ee > 0 else dhs
        _lib.check(L.pk_scalar_conv_wgrad(_ptr(d_pe), _ptr(ps), B, T, A, kp, _ptr(self.grads["pitch_embed.0.weight"]),
                                          _ptr(self.grads["pitch_embed.0.bias"]), st), "pk_scalar_conv_wgrad")
        _lib.check(L.pk_scalar_conv_wgrad(_ptr(d_ee), _ptr(es), B, T, A, ke, _ptr(self.grads["energy_embed.0.weight"]),
                                          _ptr(self.grads["energy_embed.0.bias"]), st), "pk_scalar_conv_wgrad")
        gd = self.pred_bwd(g_d, S_d)
        ops.axpy_(1.0, gd, dhs)
        ge = self.pred_bwd(g_e, S_e, need_dx=not self.sg_energy)
        if not self.sg_energy:
            ops.axpy_(1.0, ge, dhs)
        gp = self.pred_bwd(g_p, S_p, need_dx=not self.sg_pitch)
        if not self.sg_pitch:
            ops.axpy_(1.0, gp, dhs)
        if self.spk:
            dhs = self.spk_bwd(dhs, S_spk)
        dx = self.stack_bwd(dhs, S_enc)
        if R["transformer_enc_positional_dropout_rate"] > 0:
            self.drop(dx, R["transformer_enc_positional_dropout_rate"], self.site(0, 0, 0), inplace=True)
        _lib.check(L.pk_embed_pe_bwd(_ptr(text), _ptr(dx), m.idim, m.padding_idx, B, T, A, _ptr(self.grads["encoder.embed.0.weight"]),
                                     _ptr(self.grads["encoder.embed.1.alpha"]), st), "pk_embed_pe_bwd")
        self.join_side()
        return losses
