"""FastSpeech2 on H100 - host side.

Mirrors parakeet/models/fastspeech2/fastspeech2.py of the reference: `FastSpeech2` (:37-659) with the same constructor
keywords, `forward(text, text_lengths, speech, speech_lengths, durations, pitch, energy, ...)` -> the reference's 7-tuple,
`inference(text, ..., alpha)` -> (L, odim), the reference's state-dict key names and Paddle layouts (Linear [in, out],
Conv1D [out, in, k], BatchNorm `_mean` / `_variance`), and `FastSpeech2Inference` (:662-671).

Every FLOP runs in libparakeet_b200.so: GEMM-shaped work (QKV / output projections, QK^T, PV, Conv1D feed-forward,
predictor convs, feat_out, postnet) through pk_conv_gemm on wgmma; row-wise work (embedding + positional encoding,
LayerNorm, masked softmax, duration rounding, length regulator) through the pk_* kernels of fs2.cu / elementwise.cu.
There is one device->host copy per call: the B output lengths (sum of durations), needed to size the decoder buffers
(the reference syncs twice per utterance, nets_utils.py:80 `.tolist()` and length_regulator.py:53 `.numpy()`).

Scope: inference-mode arithmetic (dropout = identity, BatchNorm uses its running statistics) for `inference()`,
`batch_inference()` and `forward()`, including the multi-speaker / tone conditioning of the aishell3 / vctk recipes
(`spk_id` / `spembs` / `tone_id`, "add" and "concat" integration); the training step lives in training/fs2_step.py
(single-speaker).  `reduction_factor > 1` and `concat_after` are not implemented and raise NotImplementedError.
"""
import math
from typing import Dict, Optional, Sequence, Tuple  # noqa: F401

import torch

from .. import _lib, ops
from ..layer import Layer
from ..ops import Split
from ._transformer import fft_stack, pack_fft_blocks


def _i32(t):
    return t.to(dtype=torch.int32).contiguous()


class FastSpeech2(Layer):
    def __init__(
            self,
            # network structure related
            idim: int,
            odim: int,
            adim: int = 384,
            aheads: int = 4,
            elayers: int = 6,
            eunits: int = 1536,
            dlayers: int = 6,
            dunits: int = 1536,
            postnet_layers: int = 5,
            postnet_chans: int = 512,
            postnet_filts: int = 5,
            positionwise_layer_type: str = "conv1d",
            positionwise_conv_kernel_size: int = 1,
            use_scaled_pos_enc: bool = True,
            use_batch_norm: bool = True,
            encoder_normalize_before: bool = True,
            decoder_normalize_before: bool = True,
            encoder_concat_after: bool = False,
            decoder_concat_after: bool = False,
            reduction_factor: int = 1,
            encoder_type: str = "transformer",
            decoder_type: str = "transformer",
            # duration predictor
            duration_predictor_layers: int = 2,
            duration_predictor_chans: int = 384,
            duration_predictor_kernel_size: int = 3,
            # energy predictor
            energy_predictor_layers: int = 2,
            energy_predictor_chans: int = 384,
            energy_predictor_kernel_size: int = 3,
            energy_predictor_dropout: float = 0.5,
            energy_embed_kernel_size: int = 9,
            energy_embed_dropout: float = 0.5,
            stop_gradient_from_energy_predictor: bool = False,
            # pitch predictor
            pitch_predictor_layers: int = 2,
            pitch_predictor_chans: int = 384,
            pitch_predictor_kernel_size: int = 3,
            pitch_predictor_dropout: float = 0.5,
            pitch_embed_kernel_size: int = 9,
            pitch_embed_dropout: float = 0.5,
            stop_gradient_from_pitch_predictor: bool = False,
            # spk emb
            num_speakers: int = None,
            spk_embed_dim: int = None,
            spk_embed_integration_type: str = "add",
            #  tone emb
            num_tones: int = None,
            tone_embed_dim: int = None,
            tone_embed_integration_type: str = "add",
            # training related
            transformer_enc_dropout_rate: float = 0.1,
            transformer_enc_positional_dropout_rate: float = 0.1,
            transformer_enc_attn_dropout_rate: float = 0.1,
            transformer_dec_dropout_rate: float = 0.1,
            transformer_dec_positional_dropout_rate: float = 0.1,
            transformer_dec_attn_dropout_rate: float = 0.1,
            duration_predictor_dropout_rate: float = 0.1,
            postnet_dropout_rate: float = 0.5,
            init_type: str = "xavier_uniform",
            init_enc_alpha: float = 1.0,
            init_dec_alpha: float = 1.0,
            use_masking: bool = False,
            use_weighted_masking: bool = False,
            device=None,
            seed: int = 0):
        super().__init__(device)
        unsupported = []
        if spk_embed_dim is not None and spk_embed_integration_type not in ("add", "concat"):
            unsupported.append(f"spk_embed_integration_type={spk_embed_integration_type}")
        if tone_embed_dim is not None and tone_embed_integration_type not in ("add", "concat"):
            unsupported.append(f"tone_embed_integration_type={tone_embed_integration_type}")
        if reduction_factor != 1:
            unsupported.append("reduction_factor > 1")
        if encoder_concat_after or decoder_concat_after:
            unsupported.append("concat_after")
        if not (encoder_normalize_before and decoder_normalize_before):
            unsupported.append("post-LN (normalize_before=False)")
        if encoder_type != "transformer" or decoder_type != "transformer":
            unsupported.append("non-transformer encoder/decoder")
        if positionwise_layer_type not in ("conv1d", "linear"):
            unsupported.append(f"positionwise_layer_type={positionwise_layer_type}")
        if not use_scaled_pos_enc:
            unsupported.append("unscaled positional encoding")
        if not use_batch_norm:
            unsupported.append("postnet without batch norm")
        if adim % 64 != 0 or adim % aheads != 0:
            unsupported.append("adim must be a multiple of 64 and of aheads")
        elif (adim // aheads) % 64 != 0:
            # the non-fused attention and the training step slice Q / K / V per head out of one (B, T, 3 adim) buffer, and the
            # GEMM reads K in 64-column chunks: a head width that is not a multiple of 64 would read the next head's columns
            unsupported.append(f"attention head width adim / aheads = {adim // aheads} (must be a multiple of 64)")
        if unsupported:
            raise NotImplementedError("not in this round's hot-path scope: " + ", ".join(unsupported))
        self.idim, self.odim, self.adim, self.aheads = idim, odim, adim, aheads
        # dropout is a training-time operation (identity in inference / eval forward): the rates are kept for
        # training/fs2_step.py, which applies Philox masks at the reference's sites
        self.dropout_rates = dict(
            transformer_enc_dropout_rate=transformer_enc_dropout_rate,
            transformer_enc_positional_dropout_rate=transformer_enc_positional_dropout_rate,
            transformer_enc_attn_dropout_rate=transformer_enc_attn_dropout_rate,
            transformer_dec_dropout_rate=transformer_dec_dropout_rate,
            transformer_dec_positional_dropout_rate=transformer_dec_positional_dropout_rate,
            transformer_dec_attn_dropout_rate=transformer_dec_attn_dropout_rate,
            duration_predictor_dropout_rate=duration_predictor_dropout_rate, pitch_predictor_dropout=pitch_predictor_dropout,
            energy_predictor_dropout=energy_predictor_dropout, postnet_dropout_rate=postnet_dropout_rate,
            pitch_embed_dropout=pitch_embed_dropout, energy_embed_dropout=energy_embed_dropout)
        self.eos = idim - 1
        self.reduction_factor = reduction_factor
        self.padding_idx = 0
        self.elayers, self.dlayers = elayers, dlayers
        self.ffn_k = positionwise_conv_kernel_size if positionwise_layer_type == "conv1d" else 1
        self._linear_ffn = positionwise_layer_type == "linear"
        self.postnet_layers = postnet_layers
        self.cfg = dict(dur=(duration_predictor_layers, duration_predictor_chans, duration_predictor_kernel_size),
                        pitch=(pitch_predictor_layers, pitch_predictor_chans, pitch_predictor_kernel_size),
                        energy=(energy_predictor_layers, energy_predictor_chans, energy_predictor_kernel_size))
        self.stop_gradient_from_pitch_predictor = stop_gradient_from_pitch_predictor
        self.stop_gradient_from_energy_predictor = stop_gradient_from_energy_predictor
        # multi-speaker / tone conditioning (fastspeech2.py:127-158,190-203): embedding tables + projections
        self.spk_embed_dim, self.num_speakers, self.spk_embed_integration_type = spk_embed_dim, num_speakers, spk_embed_integration_type
        self.tone_embed_dim, self.num_tones, self.tone_embed_integration_type = tone_embed_dim, num_tones, tone_embed_integration_type

        g = torch.Generator().manual_seed(seed)
        A = adim

        def xavier(*shape, fan_in, fan_out):
            bound = math.sqrt(6.0 / (fan_in + fan_out))
            return (torch.rand(*shape, generator=g) * 2 - 1) * bound

        def lin(name, i, o):
            self._register(name + ".weight", xavier(i, o, fan_in=i, fan_out=o))   # Paddle Linear: [in, out]
            self._register(name + ".bias", torch.zeros(o))

        def conv(name, o, i, k, bias=True):
            self._register(name + ".weight", xavier(o, i, k, fan_in=i * k, fan_out=o * k))
            if bias:
                self._register(name + ".bias", torch.zeros(o))

        def ln(name, c):
            self._register(name + ".weight", torch.ones(c))
            self._register(name + ".bias", torch.zeros(c))

        def enc(pre, layers, units):
            for i in range(layers):
                q = f"{pre}encoders.{i}."
                for nm in ("linear_q", "linear_k", "linear_v", "linear_out"):
                    lin(q + "self_attn." + nm, A, A)
                if self._linear_ffn:
                    lin(q + "feed_forward.w_1", A, units)
                    lin(q + "feed_forward.w_2", units, A)
                else:
                    conv(q + "feed_forward.w_1", units, A, self.ffn_k)
                    conv(q + "feed_forward.w_2", A, units, self.ffn_k)
                ln(q + "norm1", A)
                ln(q + "norm2", A)
            ln(pre + "after_norm", A)

        emb = xavier(idim, A, fan_in=idim, fan_out=A)
        emb[self.padding_idx] = 0
        self._register("encoder.embed.0.weight", emb)
        self._register("encoder.embed.1.alpha", torch.tensor([float(init_enc_alpha)]))
        enc("encoder.", elayers, eunits)

        def pred(pre, layers, chans, k):
            for i in range(layers):
                conv(f"{pre}conv.{i}.0", chans, A if i == 0 else chans, k)
                ln(f"{pre}conv.{i}.2", chans)
            lin(pre + "linear", chans, 1)

        if spk_embed_dim is not None:
            lin("spk_projection", spk_embed_dim if spk_embed_integration_type == "add" else A + spk_embed_dim, A)
        if tone_embed_dim is not None:
            lin("tone_projection", tone_embed_dim if tone_embed_integration_type == "add" else A + tone_embed_dim, A)
        pred("duration_predictor.", *self.cfg["dur"])
        pred("pitch_predictor.", *self.cfg["pitch"])
        conv("pitch_embed.0", A, 1, pitch_embed_kernel_size)
        pred("energy_predictor.", *self.cfg["energy"])
        conv("energy_embed.0", A, 1, energy_embed_kernel_size)
        self._register("decoder.embed.0.alpha", torch.tensor([float(init_dec_alpha)]))
        enc("decoder.", dlayers, dunits)
        lin("feat_out", A, odim * reduction_factor)
        for i in range(postnet_layers):
            ic = odim if i == 0 else postnet_chans
            oc = odim if i == postnet_layers - 1 else postnet_chans
            conv(f"postnet.postnet.{i}.0", oc, ic, postnet_filts, bias=False)
            q = f"postnet.postnet.{i}.1."
            self._register(q + "weight", torch.ones(oc))
            self._register(q + "bias", torch.zeros(oc))
            self._register(q + "_mean", torch.zeros(oc))
            self._register(q + "_variance", torch.ones(oc))
        if spk_embed_dim is not None:
            assert num_speakers, "num_speakers is required with spk_embed_dim"
            self._register("spk_embedding_table.weight", torch.randn(num_speakers, spk_embed_dim, generator=g))
        if tone_embed_dim is not None:
            assert num_tones, "num_tones is required with tone_embed_dim"
            self._register("tone_embedding_table.weight", torch.randn(num_tones, tone_embed_dim, generator=g))

    # ------------------------------------------------------------------------------------------------------------
    # kernel-ready weights (once per weight change)
    # ------------------------------------------------------------------------------------------------------------
    def _pack(self):
        if self._packed is not None:
            return self._packed
        p = {k: v.detach().float().cpu() for k, v in self._params.items()}
        dev = self.device
        pk = {}
        for tag in ("spk", "tone"):
            if getattr(self, tag + "_embed_dim") is not None:
                w = p[tag + "_projection.weight"]                          # Paddle Linear [in, out]
                pk[tag + "_proj"] = dict(w=ops.pack_weight(w.t().contiguous(), dev), b=p[tag + "_projection.bias"].contiguous().to(dev),
                                         k=w.shape[0])

        def dv(t):
            return t.contiguous().to(dev)

        pk["enc"], pk["enc_norm"] = pack_fft_blocks(p, "encoder.", self.elayers, self._linear_ffn, dev)
        pk["dec"], pk["dec_norm"] = pack_fft_blocks(p, "decoder.", self.dlayers, self._linear_ffn, dev)
        pk["emb"] = dv(p["encoder.embed.0.weight"])
        pk["enc_alpha"] = dv(p["encoder.embed.1.alpha"].reshape(1))
        pk["dec_alpha"] = dv(p["decoder.embed.0.alpha"].reshape(1))

        def pred(pre, layers):
            convs = []
            for i in range(layers):
                w = p[f"{pre}conv.{i}.0.weight"]
                convs.append(dict(w=ops.pack_weight(w, dev), b=dv(p[f"{pre}conv.{i}.0.bias"]), n=w.shape[0], k=w.shape[1],
                                  taps=w.shape[2], g=dv(p[f"{pre}conv.{i}.2.weight"]), be=dv(p[f"{pre}conv.{i}.2.bias"])))
            lw = p[pre + "linear.weight"]  # [chans, 1]
            return dict(convs=convs, lw=ops.pack_weight(lw.t(), dev), lb=dv(p[pre + "linear.bias"]), chans=lw.shape[0])

        pk["dur"] = pred("duration_predictor.", self.cfg["dur"][0])
        pk["pitch"] = pred("pitch_predictor.", self.cfg["pitch"][0])
        pk["energy"] = pred("energy_predictor.", self.cfg["energy"][0])
        pk["pe_w"] = dv(p["pitch_embed.0.weight"].reshape(self.adim, -1))
        pk["pe_b"] = dv(p["pitch_embed.0.bias"])
        pk["ee_w"] = dv(p["energy_embed.0.weight"].reshape(self.adim, -1))
        pk["ee_b"] = dv(p["energy_embed.0.bias"])
        pk["feat_w"] = ops.pack_weight(p["feat_out.weight"].t(), dev)
        pk["feat_b"] = dv(p["feat_out.bias"])
        post = []
        for i in range(self.postnet_layers):
            w = p[f"postnet.postnet.{i}.0.weight"]
            q = f"postnet.postnet.{i}.1."
            # eval-mode BatchNorm1D folded into the conv: y = (conv - mean) * gamma / sqrt(var + eps) + beta
            s = p[q + "weight"] / torch.sqrt(p[q + "_variance"] + 1e-5)
            post.append(dict(w=ops.pack_weight(w * s.reshape(-1, 1, 1), dev), b=dv(p[q + "bias"] - p[q + "_mean"] * s),
                             n=w.shape[0], k=w.shape[1], taps=w.shape[2]))
        pk["post"] = post
        self._packed = pk
        return pk

    # ------------------------------------------------------------------------------------------------------------
    # building blocks
    # ------------------------------------------------------------------------------------------------------------
    def _predictor(self, pk, hs_split, row_lens):
        """Conv1D -> ReLU -> LayerNorm(channel) stacks + Linear(chans -> 1) (duration_predictor.py:85-92,
        variance_predictor.py:94-100); returns fp32 (B, T, 1) before any masking / rounding."""
        h = hs_split
        for c in pk["convs"]:
            y, _ = ops.conv_gemm(h, c["w"], n=c["n"], k=c["k"], taps=c["taps"], bias=c["b"], act="relu", lens=row_lens)
            _, h = ops.layer_norm(y, c["g"], c["be"], lens=row_lens)
        out, _ = ops.conv_gemm(h, pk["lw"], n=1, k=pk["chans"], bias=pk["lb"], lens=row_lens)
        return out

    def _postnet(self, before, before_split, row_lens):
        """after = before + Postnet(before) (tacotron2/decoder.py:182-198, fastspeech2.py:460-464), BN folded."""
        pk = self._pack()["post"]
        h = before_split
        n = len(pk)
        for i, c in enumerate(pk):
            last = i == n - 1
            y, hs = ops.conv_gemm(h, c["w"], n=c["n"], k=c["k"], taps=c["taps"], bias=c["b"], act=None if last else "tanh",
                                  residual=before if last else None, lens=row_lens, out_f32=last, out_split=not last)
            h = hs
        return y

    # ------------------------------------------------------------------------------------------------------------
    # _forward (reference fastspeech2.py:377-466)
    # ------------------------------------------------------------------------------------------------------------
    def _embed_ids(self, table_name, ids):
        """nn.Embedding(padding_idx=0): rows of the table, zeros for id 0 (a gather and a fill: no arithmetic)."""
        table = self._params[table_name]
        e = table.index_select(0, ids.reshape(-1)).reshape(tuple(ids.shape) + (table.shape[1],))
        return e.masked_fill((ids == self.padding_idx).unsqueeze(-1), 0.0)

    def _integrate(self, tag, hs, emb_n, row_lens):
        """_integrate_with_spk_embed / _integrate_with_tone_embed (fastspeech2.py:560-616) after F.normalize:
        "add": hs + projection(emb); "concat": projection(concat([hs, emb broadcast over time])).
        emb_n: (B, D) (speaker) or (B, T, D) / (T, D) (tone).  Returns (hs fp32, hs split planes)."""
        pk = self._pack()[tag + "_proj"]
        B, T, A = hs.shape
        itype = getattr(self, tag + "_embed_integration_type")
        if emb_n.dim() == 2 and tag == "spk":
            emb_bt = emb_n.unsqueeze(1)                                     # (B, 1, D)
        else:
            emb_bt = emb_n.reshape(-1, T, emb_n.shape[-1])                  # (B or 1, T, D)
        if itype == "add":
            proj, _ = ops.conv_gemm(Split.from_f32(emb_bt.contiguous()), pk["w"], n=A, k=pk["k"], bias=pk["b"])
            out = hs.clone()
            ops.axpy_(1.0, proj.expand(B, T, A).contiguous(), out)
            if row_lens is not None:
                ops.mask_rows_(out, row_lens)
            return out, Split.from_f32(out)
        cat = torch.cat([hs, emb_bt.expand(B, T, emb_bt.shape[-1])], dim=-1).contiguous()      # layout only
        return ops.conv_gemm(Split.from_f32(cat), pk["w"], n=A, k=pk["k"], bias=pk["b"], lens=row_lens, out_f32=True, out_split=True)

    def _stage_a(self, xs, ilens32, ds=None, ps=None, es=None, is_inference=False, alpha=1.0, independent=False,
                 spk_emb=None, tone_emb=None):
        """Encoder, (speaker / tone integration,) variance predictors, duration rounding, variance embeddings, frame counts:
        everything whose shapes depend on (B, T) only.  No host synchronisation (CUDA-graph capturable).
        spk_emb / tone_emb: already normalised embeddings (see _conditioning)."""
        pk = self._pack()
        B, T = xs.shape
        row_lens = ilens32 if independent else None
        # encoder: Embedding(padding_idx=0) + ScaledPositionalEncoding, FFT blocks, after_norm; keys masked by ilens
        x = ops.embed_pe(xs, pk["emb"], None, pk["enc_alpha"], row_lens, self.padding_idx)
        hs, hs_split = fft_stack(x, pk["enc"], pk["enc_norm"], self.aheads, self.ffn_k, row_lens, ilens32, want_split_out=True)
        if spk_emb is not None:                                             # fastspeech2.py:395-401
            hs, hs_split = self._integrate("spk", hs, spk_emb, row_lens)
        if tone_emb is not None:                                            # :403-407
            hs, hs_split = self._integrate("tone", hs, tone_emb, row_lens)
        # variance predictors (masked_fill with the pad mask, variance_predictor.py:101-103)
        p_outs = ops.mask_rows_(self._predictor(pk["pitch"], hs_split, row_lens), ilens32)
        e_outs = ops.mask_rows_(self._predictor(pk["energy"], hs_split, row_lens), ilens32)
        d_raw = self._predictor(pk["dur"], hs_split, row_lens).reshape(B, T)
        if is_inference:
            d_outs, d_int = ops.duration_post(d_raw, ilens32)
            hs2 = ops.variance_embed_add(hs, p_outs.reshape(B, T), e_outs.reshape(B, T), pk["pe_w"], pk["pe_b"], pk["ee_w"],
                                         pk["ee_b"], row_lens)
            if alpha != 1.0:
                assert alpha > 0
                d_int = ops.duration_scale(d_int, float(alpha))
        else:
            d_outs = ops.mask_rows_(d_raw, ilens32)
            hs2 = ops.variance_embed_add(hs, ps.reshape(B, T).float(), es.reshape(B, T).float(), pk["pe_w"], pk["pe_b"],
                                         pk["ee_w"], pk["ee_b"], row_lens)
            d_int = ds.to(torch.int64)
        # length regulator: device-side frame counts
        lr_lens = ops.length_regulator_lens(d_int)
        return hs2, d_int, lr_lens, d_outs, p_outs, e_outs

    def _stage_b(self, hs2, d_int, t_dec, dec_rows, dec_keys):
        """Length regulator, decoder, feat_out, postnet for a decoder length t_dec known on the host (capturable)."""
        pk = self._pack()
        hs_lr, _ = ops.length_regulate(hs2, d_int, t_dec)
        x = ops.embed_pe(None, None, hs_lr, pk["dec_alpha"], dec_rows)
        _, zs = fft_stack(x, pk["dec"], pk["dec_norm"], self.aheads, self.ffn_k, dec_rows, dec_keys, want_split_out=True)
        zs_split = zs if isinstance(zs, Split) else None
        before, before_split = ops.conv_gemm(zs_split, pk["feat_w"], n=self.odim, k=self.adim, bias=pk["feat_b"], lens=dec_rows,
                                             out_f32=True, out_split=True)
        after = before if self.postnet_layers == 0 else self._postnet(before, before_split, dec_rows)
        return before, after

    def _conditioning(self, B, T, spembs=None, spk_id=None, tone_id=None, per_utterance=False):
        """Speaker / tone embeddings, looked up and L2-normalised as the reference does (F.normalize, axis 1).
        per_utterance: the single-utterance `inference` path, where tone embeddings are (T, D) and axis 1 is the feature axis;
        in the batched forward axis 1 of the (B, T, D) tone tensor is TIME (the reference's own behaviour, kept)."""
        spk_emb = tone_emb = None
        if self.spk_embed_dim is not None:
            if spembs is not None:
                spk_emb = ops.l2_normalize_axis1(spembs.reshape(B, -1).to(self.device))
            elif spk_id is not None:
                spk_emb = ops.l2_normalize_axis1(self._embed_ids("spk_embedding_table.weight", spk_id.to(self.device, torch.int64).reshape(B)))
        if self.tone_embed_dim is not None and tone_id is not None:
            e = self._embed_ids("tone_embedding_table.weight", tone_id.to(self.device, torch.int64).reshape(B, T))
            if per_utterance:
                tone_emb = ops.l2_normalize_axis1(e.reshape(B * T, -1)).reshape(B, T, -1)
            else:
                tone_emb = ops.l2_normalize_axis1(e)
        return spk_emb, tone_emb

    def _forward(self, xs, ilens, olens=None, ds=None, ps=None, es=None, is_inference=False, alpha=1.0, independent=False,
                 spk_emb=None, tone_emb=None):
        if not xs.is_cuda:
            raise _lib.PkError("FastSpeech2 needs CUDA tensors (no CPU fallback)")
        B = xs.shape[0]
        ilens32 = _i32(ilens.to(xs.device))
        hs2, d_int, lr_lens, d_outs, p_outs, e_outs = self._stage_a(xs.to(torch.int64), ilens32, ds, ps, es, is_inference, alpha,
                                                                    independent, spk_emb, tone_emb)
        t_dec = int(lr_lens.max().item())        # the one D2H copy (B integers) that sizes the decoder
        if t_dec == 0:
            empty = torch.zeros(B, 0, self.odim, device=xs.device)
            return empty, empty, d_outs, p_outs, e_outs, lr_lens
        if independent:
            dec_rows, dec_keys = lr_lens, lr_lens
        elif olens is not None and not is_inference:
            dec_rows, dec_keys = None, _i32(olens.to(xs.device))   # h_masks = _source_mask(olens)  (:451)
        else:
            dec_rows, dec_keys = None, None                        # h_masks = None                 (:453)
        before, after = self._stage_b(hs2, d_int, t_dec, dec_rows, dec_keys)
        return before, after, d_outs, p_outs, e_outs, lr_lens

    def _infer(self, xs, ilens, alpha=1.0, spk_emb=None, tone_emb=None):
        """Inference through CUDA graphs (parakeet_b200/graph.py): every utterance is computed as if alone (utterance-local
        padding and key masks), so the decoder length can be rounded up to a bucket of 32 frames - padded rows are inert
        and are sliced off - and the two shape-static halves replay as graphs.  Returns (after, d_outs, frame counts)."""
        if not xs.is_cuda:
            raise _lib.PkError("FastSpeech2 needs CUDA tensors (no CPU fallback)")
        B, T = xs.shape
        xs = xs.to(torch.int64).contiguous()
        ilens32 = _i32(ilens.to(xs.device))
        alpha = float(alpha)
        cond = [t for t in (spk_emb, tone_emb) if t is not None]
        def fa(x_, l_, *c_):
            c_ = list(c_)
            se = c_.pop(0) if spk_emb is not None else None
            te = c_.pop(0) if tone_emb is not None else None
            return self._stage_a(x_, l_, is_inference=True, alpha=alpha, independent=True, spk_emb=se, tone_emb=te)
        hs2, d_int, lr_lens, d_outs, _, _ = self._graphs.run(("a", B, T, alpha, spk_emb is not None, tone_emb is not None), fa,
                                                              [xs, ilens32] + cond)
        t_dec = int(lr_lens.max().item())
        if t_dec == 0:
            return torch.zeros(B, 0, self.odim, device=xs.device), d_outs.clone(), lr_lens.clone()
        bucket = (t_dec + 31) // 32 * 32
        fb = lambda h_, d_, l_: self._stage_b(h_, d_, bucket, l_, l_)
        _, after = self._graphs.run(("b", B, T, bucket), fb, [hs2, d_int, lr_lens])
        return after[:, :t_dec].clone(), d_outs.clone(), lr_lens.clone()

    # ------------------------------------------------------------------------------------------------------------
    # public API (reference :289-375, :468-558)
    # ------------------------------------------------------------------------------------------------------------
    def forward(self, text, text_lengths, speech, speech_lengths, durations, pitch, energy, tone_id=None, spembs=None,
                spk_id=None):
        spk_emb, tone_emb = self._conditioning(text.shape[0], text.shape[1], spembs, spk_id, tone_id)
        before, after, d_outs, p_outs, e_outs, _ = self._forward(
            text.to(torch.int64), text_lengths.to(torch.int64), speech_lengths.to(torch.int64), durations.to(torch.int64), pitch,
            energy, is_inference=False, spk_emb=spk_emb, tone_emb=tone_emb)
        return before, after, d_outs, p_outs, e_outs, speech, speech_lengths.to(torch.int64)

    def inference(self, text, speech=None, durations=None, pitch=None, energy=None, alpha: float = 1.0,
                  use_teacher_forcing: bool = False, spembs=None, spk_id=None, tone_id=None):
        xs = text.to(torch.int64).unsqueeze(0)
        ilens = torch.tensor([xs.shape[1]], dtype=torch.int64, device=xs.device)
        spk_emb, tone_emb = self._conditioning(1, xs.shape[1], spembs, spk_id, tone_id, per_utterance=True)
        if use_teacher_forcing:
            _, outs, *_ = self._forward(xs, ilens, None, durations.to(torch.int64).unsqueeze(0), pitch.unsqueeze(0),
                                        energy.unsqueeze(0), is_inference=False, spk_emb=spk_emb, tone_emb=tone_emb)
        else:
            outs, _, _ = self._infer(xs, ilens, alpha, spk_emb, tone_emb)
        return outs[0]

    def batch_inference(self, text, text_lengths, alpha: float = 1.0, spembs=None, spk_id=None, tone_id=None):
        """Batched form of `inference`: padded ids (B, Tmax) + lengths -> (mel (B, Lmax, odim), frame counts (B,) int32,
        durations (B, Tmax)).  Each utterance is computed exactly as if it had been passed to `inference` alone
        (utterance-local zero padding and key masking, per-utterance normalisation of tone embeddings); rows past an
        utterance's own length are zero.  spk_id (B,) / spembs (B, D) / tone_id (B, Tmax) as in `forward`."""
        spk_emb, tone_emb = self._conditioning(text.shape[0], text.shape[1], spembs, spk_id, tone_id, per_utterance=True)
        after, d_outs, olens = self._infer(text, text_lengths, alpha, spk_emb, tone_emb)
        return after, olens, d_outs


class FastSpeech2Inference(Layer):
    """reference fastspeech2.py:662-671."""

    def __init__(self, normalizer, model):
        super().__init__(model.device)
        self.normalizer = normalizer
        self.acoustic_model = model

    def forward(self, text, spk_id=None):
        normalized_mel = self.acoustic_model.inference(text, spk_id=spk_id)
        return self.normalizer.inverse(normalized_mel)


class FastSpeech2Loss(Layer):
    """Loss function module for FastSpeech2 (reference fastspeech2.py:674-812), forward value, use_masking=True."""

    def __init__(self, use_masking: bool = True, use_weighted_masking: bool = False, device=None):
        super().__init__(device)
        if not use_masking or use_weighted_masking:
            raise NotImplementedError("only use_masking=True / use_weighted_masking=False (the shipped yaml) is implemented")
        self.use_masking, self.use_weighted_masking = use_masking, use_weighted_masking

    def forward(self, after_outs, before_outs, d_outs, p_outs, e_outs, ys, ds, ps, es, ilens, olens):
        """-> (l1_loss, duration_loss, pitch_loss, energy_loss) as 0-d CUDA tensors (argument order of the reference)."""
        B, L, odim = ys.shape
        T = ds.shape[1]
        dev = ys.device
        ws = torch.empty(12, dtype=torch.float32, device=dev)
        out = torch.empty(4, dtype=torch.float32, device=dev)
        # every converted operand is bound to a local so that it outlives the (asynchronous) launch call: a temporary
        # freed inside the argument list can be handed out again by the allocator before the kernel is even enqueued
        f = lambda t: t.contiguous().float()  # noqa: E731
        bo, ao, yy, do_ = f(before_outs), f(after_outs), f(ys), f(d_outs)
        po, pp = f(p_outs).reshape(B, T), f(ps).reshape(B, T)
        eo, ee = f(e_outs).reshape(B, T), f(es).reshape(B, T)
        dsi = ds.to(torch.int64).contiguous()
        ol, il = _i32(olens.to(dev)), _i32(ilens.to(dev))
        _lib.check(_lib.lib().pk_fs2_loss(ops._ptr(bo), ops._ptr(ao), ops._ptr(yy), ops._ptr(ol), L, odim, ops._ptr(do_),
                                          ops._ptr(dsi), ops._ptr(po), ops._ptr(pp), ops._ptr(eo), ops._ptr(ee), ops._ptr(il), T, B,
                                          ops._ptr(ws), ops._ptr(out), ops._stream()), "pk_fs2_loss")
        return out[0], out[1], out[2], out[3]
