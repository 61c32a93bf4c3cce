"""TransformerTTS (reference: parakeet/models/transformer_tts/transformer_tts.py `TransformerTTS`, `TransformerTTSInference`; recipe
examples/transformer_tts/ljspeech).

`inference` is the synthesis loop of the recipe's synthesize scripts: the encoder (Embedding + ScaledPositionalEncoding, the FFT
blocks FastSpeech2 shares, `pk_conv_gemm` / `pk_fused_attention`), one `pk_conv_gemm` for the source-attention K / V of every decoder
layer, the whole autoregressive decoder loop as one persistent `pk_tts_decode` launch (csrc/transformer_tts.cu) with the stop rule
on the device, and the postnet over the frames it produced.  The host reads the frame count once, after the decoder launch.

The decoder prenet's dropout is always on with p = 0.5, as in the reference (its `F.dropout` ignores `dprenet_dropout_rate`); the
masks are Philox masks keyed by frame position (oracle/transformer_tts.py), drawn from `seed`.

The eval-mode `forward` and `inference(use_teacher_forcing=True)` run the teacher-forced decoder on tensor cores: `pk_conv_gemm`,
`pk_layer_norm`, and `pk_fused_attention_ex` for the causal self-attention and the source attention; the source-attention weights
are computed (`batched_matmul_nt` + `pk_masked_softmax`) only where they are returned.

The training step of the ljspeech recipe is `training.TransformerTTSTrainStep` (update_core: the train-mode forward with dropout,
TransformerTTSLoss, the guided source-attention loss, backward and Adam); `train()` keeps raising, as the step is the training entry
point.

Not implemented, and refused before any launch: GST, speaker embeddings, the encoder prenet, concat_after, post-LN and non-conv1d
position-wise layers.
"""
import math

import torch

from .. import _lib, ops
from ..layer import Layer
from ..ops import Split
from ._transformer import fft_stack, pack_fft_blocks

MAX_STEPS = 16384          # decoder steps whose attention scores fit pk_tts_decode's shared-memory buffer


class TransformerTTS(Layer):
    def __init__(self, idim, odim, embed_dim=512, eprenet_conv_layers=3, eprenet_conv_chans=256, eprenet_conv_filts=5, dprenet_layers=2,
                 dprenet_units=256, elayers=6, eunits=1024, adim=512, aheads=4, dlayers=6, dunits=1024, postnet_layers=5,
                 postnet_chans=256, postnet_filts=5, positionwise_layer_type="conv1d", positionwise_conv_kernel_size=1,
                 use_scaled_pos_enc=True, use_batch_norm=True, encoder_normalize_before=True, decoder_normalize_before=True,
                 encoder_concat_after=False, decoder_concat_after=False, reduction_factor=1, spk_embed_dim=None,
                 spk_embed_integration_type="add", use_gst=False, gst_tokens=10, gst_heads=4, gst_conv_layers=6,
                 gst_conv_chans_list=(32, 32, 64, 64, 128, 128), gst_conv_kernel_size=3, gst_conv_stride=2, gst_gru_layers=1,
                 gst_gru_units=128, transformer_enc_dropout_rate=0.1, transformer_enc_positional_dropout_rate=0.1,
                 transformer_enc_attn_dropout_rate=0.1, transformer_dec_dropout_rate=0.1, transformer_dec_positional_dropout_rate=0.1,
                 transformer_dec_attn_dropout_rate=0.1, transformer_enc_dec_attn_dropout_rate=0.1, eprenet_dropout_rate=0.5,
                 dprenet_dropout_rate=0.5, postnet_dropout_rate=0.5, init_type="xavier_uniform", init_enc_alpha=1.0, init_dec_alpha=1.0,
                 use_guided_attn_loss=True, num_heads_applied_guided_attn=2, num_layers_applied_guided_attn=2, device=None):
        super().__init__(device)
        bad = []
        if eprenet_conv_layers != 0:
            bad.append("the encoder prenet (eprenet_conv_layers > 0)")
        if spk_embed_dim is not None:
            bad.append("speaker embeddings (spk_embed_dim)")
        if use_gst:
            bad.append("GST (use_gst)")
        if encoder_concat_after or decoder_concat_after:
            bad.append("concat_after")
        if not (encoder_normalize_before and decoder_normalize_before):
            bad.append("post-LN (normalize_before=False)")
        if positionwise_layer_type != "conv1d":
            bad.append(f"positionwise_layer_type={positionwise_layer_type}")
        if dprenet_layers == 0:
            bad.append("no decoder prenet (dprenet_layers = 0)")
        if not use_scaled_pos_enc:
            bad.append("unscaled positional encoding")
        if not use_batch_norm and postnet_layers:
            bad.append("postnet without batch norm")
        if adim % aheads or (adim // aheads) % 64:
            bad.append(f"attention head width adim / aheads = {adim / aheads:g} (must be a multiple of 64)")
        elif adim // aheads > 192:
            bad.append(f"attention head width adim / aheads = {adim // aheads} (the teacher-forced decoder's pk_fused_attention_ex "
                       "takes 64, 128 or 192)")
        if odim % 4 or dprenet_units % 4 or dunits % 4 or reduction_factor < 1 or reduction_factor > 16:
            bad.append("odim, dprenet_units and dunits must be multiples of 4 and 1 <= reduction_factor <= 16")
        if postnet_layers and postnet_filts % 2 == 0:
            bad.append("an even postnet kernel")
        if bad:
            raise ValueError("TransformerTTS: not supported: " + ", ".join(bad))
        self.idim, self.odim, self.adim, self.aheads, self.r = idim, odim, adim, aheads, reduction_factor
        self.eos, self.padding_idx = idim - 1, 0
        self.elayers, self.dlayers, self.dprenet_layers, self.dprenet_units = elayers, dlayers, dprenet_layers, dprenet_units
        self.ffn_k, self.postnet_layers = positionwise_conv_kernel_size, postnet_layers
        # eval-mode scalars of the reference's forward need_dict
        self.num_heads_applied_guided_attn = aheads if num_heads_applied_guided_attn == -1 else num_heads_applied_guided_attn
        self.num_layers_applied_guided_attn = elayers if num_layers_applied_guided_attn == -1 else num_layers_applied_guided_attn
        self.use_scaled_pos_enc = use_scaled_pos_enc
        # the train-mode rates, read by training/transformer_tts_step.py (the decoder prenet's p = 0.5 is not among them: its
        # F.dropout ignores dprenet_dropout_rate)
        self.dropout_rates = dict(transformer_enc_dropout_rate=transformer_enc_dropout_rate,
                                  transformer_enc_positional_dropout_rate=transformer_enc_positional_dropout_rate,
                                  transformer_enc_attn_dropout_rate=transformer_enc_attn_dropout_rate,
                                  transformer_dec_dropout_rate=transformer_dec_dropout_rate,
                                  transformer_dec_positional_dropout_rate=transformer_dec_positional_dropout_rate,
                                  transformer_dec_attn_dropout_rate=transformer_dec_attn_dropout_rate,
                                  transformer_enc_dec_attn_dropout_rate=transformer_enc_dec_attn_dropout_rate,
                                  postnet_dropout_rate=postnet_dropout_rate)
        self.training = False
        g = torch.Generator().manual_seed(0)
        A, k = adim, positionwise_conv_kernel_size

        def xavier(*shape, fan_in, fan_out):
            return (torch.rand(*shape, generator=g) * 2 - 1) * math.sqrt(6.0 / (fan_in + fan_out))

        def lin(name, i, o):
            self._register(name + ".weight", xavier(i, o, fan_in=i, fan_out=o))      # Paddle Linear: [in, out]
            self._register(name + ".bias", torch.zeros(o))

        def ln(name):
            self._register(name + ".weight", torch.ones(A))
            self._register(name + ".bias", torch.zeros(A))

        def attn(pre):
            for n in ("linear_q", "linear_k", "linear_v", "linear_out"):
                lin(pre + n, A, A)

        emb = xavier(idim, A, fan_in=idim, fan_out=A)
        emb[self.padding_idx] = 0
        self._register("encoder.embed.0.weight", emb)
        self._register("encoder.embed.1.alpha", torch.tensor([float(init_enc_alpha)]))
        for i in range(elayers):
            q = f"encoder.encoders.{i}."
            attn(q + "self_attn.")
            for n, o, c in (("w_1", eunits, A), ("w_2", A, eunits)):
                self._register(f"{q}feed_forward.{n}.weight", xavier(o, c, k, fan_in=c * k, fan_out=o * k))
                self._register(f"{q}feed_forward.{n}.bias", torch.zeros(o))
            ln(q + "norm1")
            ln(q + "norm2")
        ln("encoder.after_norm")
        for i in range(dprenet_layers):
            lin(f"decoder.embed.0.0.prenet.{i}.0", odim if i == 0 else dprenet_units, dprenet_units)
        lin("decoder.embed.0.1", dprenet_units, A)
        self._register("decoder.embed.1.alpha", torch.tensor([float(init_dec_alpha)]))
        for i in range(dlayers):
            q = f"decoder.decoders.{i}."
            attn(q + "self_attn.")
            attn(q + "src_attn.")
            lin(q + "feed_forward.w_1", A, dunits)                # the decoder's PositionwiseFeedForward is Linear
            lin(q + "feed_forward.w_2", dunits, A)
            for n in ("norm1", "norm2", "norm3"):
                ln(q + n)
        ln("decoder.after_norm")
        lin("feat_out", A, odim * reduction_factor)
        lin("prob_out", A, reduction_factor)
        for i in range(postnet_layers):
            ci = odim if i == 0 else postnet_chans
            co = odim if i == postnet_layers - 1 else postnet_chans
            self._register(f"postnet.postnet.{i}.0.weight", xavier(co, ci, postnet_filts, fan_in=ci * postnet_filts, fan_out=co * postnet_filts))
            q = f"postnet.postnet.{i}.1."
            self._register(q + "weight", torch.ones(co))
            self._register(q + "bias", torch.zeros(co))
            self._register(q + "_mean", torch.zeros(co))
            self._register(q + "_variance", torch.ones(co))

    def train(self):
        raise NotImplementedError("the TransformerTTS training step is not implemented; inference runs in eval mode")

    # -- packed weights ------------------------------------------------------------------------------------------
    def _pack(self):
        if self._packed is not None:
            return self._packed
        p = {k: v.detach().float().cpu() for k, v in self._params.items()}
        dev = self.device
        A, L, r = self.adim, self.dlayers, self.r
        pk = {}
        pk["enc"], pk["enc_norm"] = pack_fft_blocks(p, "encoder.", self.elayers, False, dev)
        pk["emb"] = p["encoder.embed.0.weight"].to(dev)
        pk["enc_alpha"] = p["encoder.embed.1.alpha"].reshape(1).to(dev)
        pk["dec_alpha"] = p["decoder.embed.1.alpha"].reshape(1).to(dev)
        src = [f"decoder.decoders.{l}.src_attn." for l in range(L)]
        wkv = torch.cat([torch.cat([p[s + "linear_k.weight"], p[s + "linear_v.weight"]], 1) for s in src], 1)      # [A, L 2A]
        pk["wkv"] = ops.pack_weight(wkv.t(), dev)
        pk["bkv"] = torch.cat([torch.cat([p[s + "linear_k.bias"], p[s + "linear_v.bias"]]) for s in src]).to(dev)
        t = lambda name: p[name].t().reshape(-1)              # Paddle Linear [in, out] -> [out][in] rows
        layers = []
        for l in range(L):
            q = f"decoder.decoders.{l}."
            sa, ca = q + "self_attn.", q + "src_attn."
            layers += [t(sa + "linear_q.weight"), t(sa + "linear_k.weight"), t(sa + "linear_v.weight"),
                       p[sa + "linear_q.bias"], p[sa + "linear_k.bias"], p[sa + "linear_v.bias"],
                       t(sa + "linear_out.weight"), p[sa + "linear_out.bias"], t(ca + "linear_q.weight"), p[ca + "linear_q.bias"],
                       t(ca + "linear_out.weight"), p[ca + "linear_out.bias"], t(q + "feed_forward.w_1.weight"), p[q + "feed_forward.w_1.bias"],
                       t(q + "feed_forward.w_2.weight"), p[q + "feed_forward.w_2.bias"]]
            layers += [p[f"{q}{n}.{b}"] for n in ("norm1", "norm2", "norm3") for b in ("weight", "bias")]
        lw = torch.cat(layers)
        assert lw.numel() == L * int(_lib.lib().pk_tts_layer_floats(A, p["decoder.decoders.0.feed_forward.w_1.bias"].numel()))
        pre = [f"decoder.embed.0.0.prenet.{i}.0." for i in range(self.dprenet_layers)]
        pk["dec"] = dict(
            adim=A, units=p["decoder.decoders.0.feed_forward.w_1.bias"].numel(), prenet_units=self.dprenet_units, layers=L, r=r,
            odim=self.odim, prenet_layers=self.dprenet_layers,
            pre_w=torch.cat([t(s + "weight") for s in pre]).to(dev), pre_b=torch.cat([p[s + "bias"] for s in pre]).to(dev),
            in_w=t("decoder.embed.0.1.weight").to(dev), in_b=p["decoder.embed.0.1.bias"].to(dev), layer_w=lw.to(dev),
            norm=torch.cat([p["decoder.after_norm.weight"], p["decoder.after_norm.bias"]]).to(dev),
            out_w=torch.cat([t("prob_out.weight"), t("feat_out.weight")]).to(dev),
            out_b=torch.cat([p["prob_out.bias"], p["feat_out.bias"]]).to(dev))
        post = []
        for i in range(self.postnet_layers):
            w = p[f"postnet.postnet.{i}.0.weight"]
            q = f"postnet.postnet.{i}.1."
            s = p[q + "weight"] / torch.sqrt(p[q + "_variance"] + 1e-5)      # eval BatchNorm1D folded into the conv
            post.append(dict(w=ops.pack_weight(w * s.reshape(-1, 1, 1), dev), b=(p[q + "bias"] - p[q + "_mean"] * s).to(dev),
                             n=w.shape[0], k=w.shape[1], taps=w.shape[2]))
        pk["post"] = post
        # the teacher-forced decoder: split-bf16 GEMM operands ([out, in] Linear weights)
        pw = lambda name: ops.pack_weight(p[name].t(), dev)   # noqa: E731
        dv = lambda name: p[name].contiguous().to(dev)        # noqa: E731
        tf = []
        for l in range(L):
            q = f"decoder.decoders.{l}."
            sa, ca = q + "self_attn.", q + "src_attn."
            wqkv = torch.cat([p[sa + "linear_q.weight"], p[sa + "linear_k.weight"], p[sa + "linear_v.weight"]], 1).t()
            tf.append(dict(wqkv=ops.pack_weight(wqkv, dev),
                           bqkv=torch.cat([p[sa + "linear_q.bias"], p[sa + "linear_k.bias"], p[sa + "linear_v.bias"]]).to(dev),
                           wo=pw(sa + "linear_out.weight"), bo=dv(sa + "linear_out.bias"), wq=pw(ca + "linear_q.weight"),
                           bq=dv(ca + "linear_q.bias"), wo_c=pw(ca + "linear_out.weight"), bo_c=dv(ca + "linear_out.bias"),
                           w1=pw(q + "feed_forward.w_1.weight"), b1=dv(q + "feed_forward.w_1.bias"), w2=pw(q + "feed_forward.w_2.weight"),
                           b2=dv(q + "feed_forward.w_2.bias"), units=p[q + "feed_forward.w_1.bias"].numel(),
                           n=[(dv(f"{q}{n}.weight"), dv(f"{q}{n}.bias")) for n in ("norm1", "norm2", "norm3")]))
        pk["tf"] = dict(layers=tf, pre=[(pw(s + "weight"), dv(s + "bias"), p[s + "weight"].shape[0]) for s in pre],
                        in_w=pw("decoder.embed.0.1.weight"), in_b=dv("decoder.embed.0.1.bias"),
                        norm=(dv("decoder.after_norm.weight"), dv("decoder.after_norm.bias")),
                        feat_w=pw("feat_out.weight"), feat_b=dv("feat_out.bias"), prob_w=pw("prob_out.weight"), prob_b=dv("prob_out.bias"))
        self._packed = pk
        return pk

    @staticmethod
    def _seed(seed):
        return int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None else int(seed)

    def _postnet(self, before):
        """before + Postnet(before) on (B, N, odim), the padded rows included as in the reference."""
        xs = Split.from_f32(before)
        post = self._pack()["post"]
        y = before
        for i, c in enumerate(post):
            last = i == len(post) - 1
            y, xs = ops.conv_gemm(xs, c["w"], n=c["n"], k=c["k"], taps=c["taps"], bias=c["b"], act=None if last else "tanh",
                                  residual=before if last else None, out_f32=last, out_split=not last)
        return y

    # -- public ------------------------------------------------------------------------------------------------------
    def inference(self, text, speech=None, spembs=None, threshold=0.5, minlenratio=0.0, maxlenratio=10.0, use_teacher_forcing=False, *,
                  seed=None):
        """-> (outs (L r, odim), probs (L r,), att_ws (dlayers, aheads, L, T + 1)) of TransformerTTS.inference for text (T,) int64;
        with use_teacher_forcing, (outs, None, att_ws) of the teacher-forced forward on speech (L, odim)."""
        return self._inference(text, speech, spembs, threshold, minlenratio, maxlenratio, use_teacher_forcing, seed)[:3]

    def _inference(self, text, speech, spembs, threshold, minlenratio, maxlenratio, use_teacher_forcing, seed):
        """inference's outputs and, without teacher forcing, the decoder's frames before the postnet (L r, odim)."""
        if spembs is not None:
            raise ValueError("spembs is not supported (no speaker embedding)")
        if speech is not None and not use_teacher_forcing:
            raise ValueError("speech is only used under teacher forcing (there is no GST)")
        if use_teacher_forcing and speech is None:
            raise ValueError("speech must be provided with teacher forcing")
        self._check(text, speech)
        if text.dim() != 1:
            raise ValueError(f"expected text (T,), got {tuple(text.shape)}")
        if use_teacher_forcing:
            if speech.dim() != 2 or speech.shape[1] != self.odim or speech.shape[0] < self.r:
                raise ValueError(f"expected speech (L >= {self.r}, {self.odim}), got {tuple(speech.shape)}")
            lens = torch.full((1,), text.numel(), dtype=torch.int32, device=text.device)
            olens = torch.full((1,), speech.shape[0], dtype=torch.int32, device=text.device)
            after, _, _, att = self._forward(text.reshape(1, -1), lens, speech.unsqueeze(0), olens, seed, want_att=True)
            return after[0], None, att[0], None
        T = text.numel() + 1
        maxlen, minlen = int(T * maxlenratio / self.r), int(T * minlenratio / self.r)
        steps = max(maxlen, minlen, 1)
        if steps > MAX_STEPS or T > MAX_STEPS:
            raise ValueError(f"{steps} decoder steps over {T} encoder rows exceed the decoder's {MAX_STEPS}-entry attention buffer")
        pk = self._pack()
        A, dev = self.adim, self.device
        x = torch.cat([text.long(), torch.full((1,), self.eos, dtype=torch.int64, device=dev)]).unsqueeze(0)
        xe = ops.embed_pe(x, pk["emb"], None, pk["enc_alpha"], None, self.padding_idx)
        _, hs = fft_stack(xe, pk["enc"], pk["enc_norm"], self.aheads, self.ffn_k, None, None, want_split_out=True)
        mem_kv = ops.conv_gemm(hs, pk["wkv"], n=self.dlayers * 2 * A, k=A, bias=pk["bkv"])[0][0]
        pe = ops.embed_pe(None, None, torch.zeros(1, steps, A, device=dev), pk["dec_alpha"], None)[0]
        outs, probs, att, frames = ops.tts_decode(pk["dec"], mem_kv, pe, heads=self.aheads, steps=steps, minlen=minlen, maxlen=maxlen,
                                                  threshold=threshold, seed=self._seed(seed))
        n = int(frames.item())            # the one host read of the call, after the decoder launch
        before = outs[:n].reshape(1, n * self.r, self.odim)
        after = self._postnet(before) if self.postnet_layers else before
        return after[0], probs[:n].reshape(-1), att[:, :, :n], before[0]

    def _check(self, text, *extra):
        for x in (text,) + extra:
            if x is not None and (not x.is_cuda or x.device != self._params["encoder.embed.0.weight"].device):
                raise _lib.PkError(f"TransformerTTS inputs must be CUDA tensors on the model's device {self.device} (no CPU fallback)")
        if text.numel():
            lo, hi = torch.aminmax(text)
            if int(lo) < 0 or int(hi) >= self.idim:
                raise ValueError(f"text ids must be in [0, {self.idim})")

    def _forward(self, text, lens, ys, olens, seed, want_att=False):
        """_forward of the reference (eval): text int64 (B, T) without eos, lens int32 (B,), ys (B, L, odim), olens int32 (B,) ->
        (after (B, L // r * r, odim), before, logits (B, L // r * r), source attention weights (B, dlayers, heads, L // r, T + 1) or
        None).  Padded rows are computed as in the reference: every query row is live, only keys are masked."""
        pk, tf = self._pack(), self._pack()["tf"]
        A, H, r, L = self.adim, self.aheads, self.r, self.dlayers
        B = text.shape[0]
        dk = A // H
        seed = self._seed(seed)
        xs, ilens = ops.tts_text_eos(text.long().contiguous(), lens, self.eos)
        Tk = xs.shape[1]
        xe = ops.embed_pe(xs, pk["emb"], None, pk["enc_alpha"], None, self.padding_idx)
        _, hs = fft_stack(xe, pk["enc"], pk["enc_norm"], H, self.ffn_k, None, ilens, want_split_out=True)      # x_masks = non_pad(ilens)
        mem = ops.conv_gemm(hs, pk["wkv"], n=L * 2 * A, k=A, bias=pk["bkv"], out_f32=False, out_split=True)[1]
        h = ops.tts_shift_frames(ys.float().contiguous(), r)                   # ys[:, r-1::r], zero first frame, last dropped
        Tq = h.shape[1]
        olens_in = torch.div(olens, r, rounding_mode="floor").to(torch.int32)
        for i, (w, b, kin) in enumerate(tf["pre"]):
            h = ops.conv_gemm(Split.from_f32(h), w, n=self.dprenet_units, k=kin, bias=b, act="relu")[0]
            ops.tts_prenet_dropout_(h, 0.5, seed, i)                             # F.dropout's default p, keyed by frame position
        x = ops.conv_gemm(Split.from_f32(h), tf["in_w"], n=A, k=self.dprenet_units, bias=tf["in_b"])[0]
        x = ops.embed_pe(None, None, x, pk["dec_alpha"], None)                 # + alpha pe
        ctx = Split.empty((B, Tq, A), x.device)
        atts = []
        for l, lay in enumerate(tf["layers"]):
            _, hn = ops.layer_norm(x, *lay["n"][0])
            _, qkv = ops.conv_gemm(hn, lay["wqkv"], n=3 * A, k=A, bias=lay["bqkv"], out_f32=False, out_split=True)
            ops.fused_attention_ex(qkv, qkv, heads=H, q_col0=0, k_col0=A, v_col0=2 * A, key_lens=olens_in, causal=True, ctx=ctx)
            x, _ = ops.conv_gemm(ctx, lay["wo"], n=A, k=A, bias=lay["bo"], residual=x)
            _, hn = ops.layer_norm(x, *lay["n"][1])
            _, q = ops.conv_gemm(hn, lay["wq"], n=A, k=A, bias=lay["bq"], out_f32=False, out_split=True)
            ops.fused_attention_ex(q, mem, heads=H, q_col0=0, k_col0=2 * A * l, v_col0=2 * A * l + A, key_lens=ilens, ctx=ctx)
            if want_att:
                # the weights only where they are returned: Q K^T of the source attention, then the key-masked softmax
                Tkp = (Tk + 63) // 64 * 64
                s_buf = torch.empty(B * H, Tq, Tkp, dtype=torch.float32, device=x.device)
                ops.batched_matmul_nt(q, mem, batch=B, heads=H, m=Tq, n=Tk, k=dk,
                                      a_spec=dict(rows=Tq, cols=A, ld=A, batch_stride=Tq * A, batches=B, bmul=1, hmul=0, col0=0, colh=dk),
                                      b_spec=dict(rows=Tk, cols=2 * A * L, ld=2 * A * L, batch_stride=Tk * 2 * A * L, batches=B, bmul=1, hmul=0,
                                                  col0=2 * A * l, colh=dk),
                                      scale=1.0 / math.sqrt(dk), y_f32=s_buf, y_batch_stride=H * Tq * Tkp, y_head_stride=Tq * Tkp, y_ld=Tkp)
                atts.append(ops.masked_softmax(s_buf, ilens, B, H, Tq, Tk).float()[..., :Tk].reshape(B, H, Tq, Tk))
            x, _ = ops.conv_gemm(ctx, lay["wo_c"], n=A, k=A, bias=lay["bo_c"], residual=x)
            _, hn = ops.layer_norm(x, *lay["n"][2])
            _, u = ops.conv_gemm(hn, lay["w1"], n=lay["units"], k=A, bias=lay["b1"], act="relu", out_f32=False, out_split=True)
            x, _ = ops.conv_gemm(u, lay["w2"], n=A, k=lay["units"], bias=lay["b2"], residual=x)
        _, zs = ops.layer_norm(x, *tf["norm"])
        before = ops.conv_gemm(zs, tf["feat_w"], n=self.odim * r, k=A, bias=tf["feat_b"])[0].reshape(B, Tq * r, self.odim)
        logits = ops.conv_gemm(zs, tf["prob_w"], n=r, k=A, bias=tf["prob_b"])[0].reshape(B, Tq * r)
        after = self._postnet(before) if self.postnet_layers else before
        return after, before, logits, (torch.stack(atts, 1) if want_att else None)

    def forward(self, text, text_lengths, speech, speech_lengths, spembs=None, *, seed=None):
        """The reference's eval-mode forward -> (after_outs, before_outs, logits, ys, labels, olens, ilens, need_dict).  need_dict holds
        the reference's scalar entries (num_heads_applied_guided_attn, num_layers_applied_guided_attn, use_scaled_pos_enc); its
        'encoder' / 'decoder' module objects, which only the training loss reads, are not included."""
        if spembs is not None:
            raise ValueError("spembs is not supported (no speaker embedding)")
        self._check(text, speech)
        if text.dim() != 2 or speech.dim() != 3 or speech.shape[0] != text.shape[0] or speech.shape[2] != self.odim:
            raise ValueError(f"expected text (B, T) and speech (B, L, {self.odim}), got {tuple(text.shape)}, {tuple(speech.shape)}")
        B = text.shape[0]
        if tuple(text_lengths.shape) != (B,) or tuple(speech_lengths.shape) != (B,):
            raise ValueError("text_lengths and speech_lengths must be (B,)")
        tl, sl = text_lengths.long().cpu(), speech_lengths.long().cpu()     # the reference reads both on the host as well
        if int(tl.min()) < 0 or int(tl.max()) > text.shape[1] or int(sl.min()) < self.r or int(sl.max()) > speech.shape[1]:
            raise ValueError(f"text_lengths must be in [0, T] and speech_lengths in [{self.r}, L]")
        if speech.shape[1] < self.r:
            raise ValueError(f"speech needs at least reduction_factor = {self.r} frames")
        dev = text.device
        lens, olens = tl.to(dev, torch.int32), sl.to(dev, torch.int32)
        after, before, logits, _ = self._forward(text, lens, speech, olens, seed)
        if self.r > 1:
            olens_out = sl - sl % self.r
            width = int(olens_out.max())
        else:
            olens_out, width = sl, int(sl.max())
        labels = ops.tts_stop_labels(olens, width)
        need = {"num_heads_applied_guided_attn": self.num_heads_applied_guided_attn,
                "num_layers_applied_guided_attn": self.num_layers_applied_guided_attn, "use_scaled_pos_enc": self.use_scaled_pos_enc}
        ys = speech if self.r == 1 else speech[:, :width]
        return after, before, logits, ys, labels, olens_out.to(dev), (tl + 1).to(dev), need


class TransformerTTSInference(Layer):
    """reference transformer_tts.py:758-768: normalizer.inverse(inference(text)[0])."""

    def __init__(self, normalizer, model):
        super().__init__(model.device)
        self.normalizer = normalizer
        self.acoustic_model = model

    def forward(self, text, spk_id=None):
        return self.normalizer.inverse(self.acoustic_model.inference(text)[0])
