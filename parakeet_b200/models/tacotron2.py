"""Tacotron2 (reference: parakeet/models/tacotron2.py `Tacotron2`, `Tacotron2Loss`; recipes examples/tacotron2 (ljspeech) and
examples/tacotron2_aishell3 (tones + a 256-wide speaker embedding as global condition)).

Eval semantics: `forward` is the teacher-forced forward of the recipes' `valid()` loops, `infer` the synthesis loop.  The encoder,
attention, decoder and postnet dropouts are identity; the prenet dropout is always on, as in the reference, drawn from `seed`.
The training step is not implemented, so `train()` raises.

Encoder: `pk_taco2_embed`, three Conv1D + BatchNorm (folded at load) + ReLU through `pk_conv_gemm`, and the bidirectional
LSTM as two `pk_lstm_fwd` recurrences (H = 256), the backward one on each sequence reversed within its own length.  The decoder
is one persistent `pk_taco2_decode` launch (csrc/tacotron2.cu); the postnet is five `pk_conv_gemm` layers with the residual add
in the last one's epilogue.

State-dict keys are Paddle 2.1's (`encoder.lstm.0.cell_fw.weight_ih`, ...); the flat keys of later Paddle releases
(`encoder.lstm.weight_ih_l0`, `..._l0_reverse`) are accepted on load.
"""
import math
import re

import torch

from .. import _lib, checkpoint, ops
from ..layer import Layer
from ..ops import Split
from .lstm_speaker_encoder import start_states

_FLAT_KEY = re.compile(r"^encoder\.lstm\.(weight_ih|weight_hh|bias_ih|bias_hh)_l0(_reverse)?$")
MAX_BATCH = 32


def canonical_keys(state):
    """Paddle >= 2.2's flat bidirectional-LSTM keys -> the 2.1 BiRNN form; other keys unchanged."""
    out = {}
    for k, v in state.items():
        m = _FLAT_KEY.match(k)
        out[f"encoder.lstm.0.{'cell_bw' if m.group(2) else 'cell_fw'}.{m.group(1)}" if m else k] = v
    return out


class Tacotron2(Layer):
    def __init__(self, vocab_size, n_tones=None, d_mels=80, d_encoder=512, encoder_conv_layers=3, encoder_kernel_size=5, d_prenet=256,
                 d_attention_rnn=1024, d_decoder_rnn=1024, attention_filters=32, attention_kernel_size=31, d_attention=128, d_postnet=512,
                 postnet_kernel_size=5, postnet_conv_layers=5, reduction_factor=1, p_encoder_dropout=0.5, p_prenet_dropout=0.5,
                 p_attention_dropout=0.1, p_decoder_dropout=0.1, p_postnet_dropout=0.5, d_global_condition=None, use_stop_token=False,
                 device=None):
        super().__init__(device)
        dk = d_encoder + (d_global_condition or 0)
        dm = d_mels * reduction_factor
        if (d_attention_rnn, d_decoder_rnn, d_prenet, d_attention) != (1024, 1024, 256, 128):
            raise ValueError("the decoder kernel is built for d_attention_rnn = d_decoder_rnn = 1024, d_prenet 256, d_attention 128")
        if d_encoder != 512 or dk not in (512, 768):
            raise ValueError(f"supported: d_encoder 512 with no or a 256-wide global condition (got {d_encoder}, {d_global_condition})")
        if dm % 4 or attention_kernel_size % 2 == 0 or attention_kernel_size > 63 or encoder_kernel_size % 2 == 0 or \
                postnet_kernel_size % 2 == 0 or postnet_conv_layers < 2:
            raise ValueError("supported: d_mels * reduction_factor a multiple of 4, odd kernel sizes (location <= 63), >= 2 postnet layers")
        if not 0.0 <= p_prenet_dropout < 1.0:
            raise ValueError("p_prenet_dropout must be in [0, 1)")
        self.vocab_size, self.n_tones, self.d_mels, self.d_encoder, self.r = vocab_size, n_tones, d_mels, d_encoder, reduction_factor
        self.encoder_conv_layers, self.encoder_kernel_size = encoder_conv_layers, encoder_kernel_size
        self.postnet_conv_layers, self.postnet_kernel_size, self.d_postnet = postnet_conv_layers, postnet_kernel_size, d_postnet
        self.p_prenet_dropout, self.d_global_condition, self.use_stop_token = p_prenet_dropout, d_global_condition, use_stop_token
        self.training = False
        g = torch.Generator().manual_seed(0)

        def u(shape, fan):
            return (torch.rand(shape, generator=g) * 2 - 1) / math.sqrt(fan)

        def conv_bn(prefix, cin, cout, k):
            self._register(prefix + "conv.weight", u((cout, cin, k), cin * k))
            self._register(prefix + "conv.bias", u((cout,), cin * k))
            self._register(prefix + "bn.weight", torch.ones(cout))
            self._register(prefix + "bn.bias", torch.zeros(cout))
            self._register(prefix + "bn._mean", torch.zeros(cout))
            self._register(prefix + "bn._variance", torch.ones(cout))

        self._register("embedding.weight", u((vocab_size, d_encoder), vocab_size + d_encoder))
        if n_tones:
            tw = u((n_tones, d_encoder), 10 * (vocab_size + d_encoder))
            tw[0] = 0.0
            self._register("embedding_tones.weight", tw)
        for i in range(encoder_conv_layers):
            conv_bn(f"encoder.conv_batchnorms.{i}.", d_encoder, d_encoder, encoder_kernel_size)
        h = d_encoder // 2
        for d in ("cell_fw", "cell_bw"):
            for part, shape in (("weight_ih", (4 * h, d_encoder)), ("weight_hh", (4 * h, h)), ("bias_ih", (4 * h,)), ("bias_hh", (4 * h,))):
                self._register(f"encoder.lstm.0.{d}.{part}", u(shape, h))
        self._register("decoder.prenet.linear1.weight", u((dm, d_prenet), dm))
        self._register("decoder.prenet.linear2.weight", u((d_prenet, d_prenet), d_prenet))
        for name, k_in in (("attention_rnn", d_prenet + dk), ("decoder_rnn", d_attention_rnn + dk)):
            for part, shape in (("weight_ih", (4096, k_in)), ("weight_hh", (4096, 1024)), ("bias_ih", (4096,)), ("bias_hh", (4096,))):
                self._register(f"decoder.{name}.{part}", u(shape, 1024))
        a = "decoder.attention_layer."
        self._register(a + "query_layer.weight", u((d_attention_rnn, d_attention), d_attention_rnn))
        self._register(a + "key_layer.weight", u((dk, d_attention), dk))
        self._register(a + "value.weight", u((d_attention, 1), d_attention))
        self._register(a + "location_conv.weight", u((attention_filters, 2, attention_kernel_size), 2 * attention_kernel_size))
        self._register(a + "location_layer.weight", u((attention_filters, d_attention), attention_filters))
        self._register("decoder.linear_projection.weight", u((d_decoder_rnn + dk, dm), d_decoder_rnn + dk))
        self._register("decoder.linear_projection.bias", u((dm,), d_decoder_rnn + dk))
        if use_stop_token:
            self._register("decoder.stop_layer.weight", u((d_decoder_rnn + dk, 1), d_decoder_rnn + dk))
            self._register("decoder.stop_layer.bias", u((1,), d_decoder_rnn + dk))
        for i in range(postnet_conv_layers):
            conv_bn(f"postnet.conv_batchnorms.{i}.", dm if i == 0 else d_postnet, dm if i == postnet_conv_layers - 1 else d_postnet,
                    postnet_kernel_size)

    @classmethod
    def from_pretrained(cls, config, checkpoint_path, device=None):
        """The recipe's config (config.model.*, config.data.n_mels) and a `step-N` checkpoint (with or without `.pdparams`)."""
        m = config.model
        names = ("vocab_size", "n_tones", "d_encoder", "encoder_conv_layers", "encoder_kernel_size", "d_prenet", "d_attention_rnn",
                 "d_decoder_rnn", "attention_filters", "attention_kernel_size", "d_attention", "d_postnet", "postnet_kernel_size",
                 "postnet_conv_layers", "reduction_factor", "p_encoder_dropout", "p_prenet_dropout", "p_attention_dropout",
                 "p_decoder_dropout", "p_postnet_dropout", "d_global_condition", "use_stop_token")
        model = cls(d_mels=config.data.n_mels, device=device, **{n: getattr(m, n) for n in names})
        path = str(checkpoint_path)
        model.set_state_dict(checkpoint.load(path if path.endswith(".pdparams") else path + ".pdparams"))
        return model

    def set_state_dict(self, state):
        super().set_state_dict(canonical_keys(state))

    load_dict = set_state_dict

    def train(self):
        raise NotImplementedError("the Tacotron2 training step is not implemented; forward and infer run in eval mode")

    # -- packed weights ------------------------------------------------------------------------------------------
    def _fold_conv(self, prefix):
        P = self._params
        s = P[prefix + "bn.weight"].double() / torch.sqrt(P[prefix + "bn._variance"].double() + 1e-5)
        w = (P[prefix + "conv.weight"].double() * s.reshape(-1, 1, 1)).float()
        b = ((P[prefix + "conv.bias"].double() - P[prefix + "bn._mean"].double()) * s + P[prefix + "bn.bias"].double()).float()
        return dict(w=ops.pack_dev(w), b=b.contiguous(), n=w.shape[0], k=w.shape[1])

    def _packs(self):
        if self._packed is None:
            P = self._params
            t = lambda x: x.t().contiguous()
            perm = ops.lstm_gate_perm(self.d_encoder // 2, self.device)
            a = "decoder.attention_layer."
            loc = torch.einsum("fd,fck->dck", P[a + "location_layer.weight"].double(), P[a + "location_conv.weight"].double())
            dec = {"pre_w1": t(P["decoder.prenet.linear1.weight"]), "pre_w2": t(P["decoder.prenet.linear2.weight"]),
                   "q_w": t(P[a + "query_layer.weight"]), "loc_w": loc.float().contiguous(), "v_w": P[a + "value.weight"][:, 0].contiguous(),
                   "proj_w": t(P["decoder.linear_projection.weight"]), "proj_b": P["decoder.linear_projection.bias"]}
            for name, key in (("att", "attention_rnn"), ("dec", "decoder_rnn")):
                dec[name + "_w"] = torch.cat([P[f"decoder.{key}.weight_ih"], P[f"decoder.{key}.weight_hh"]], 1).contiguous()
                dec[name + "_b_ih"], dec[name + "_b_hh"] = P[f"decoder.{key}.bias_ih"], P[f"decoder.{key}.bias_hh"]
            if self.use_stop_token:
                dec["stop_w"], dec["stop_b"] = P["decoder.stop_layer.weight"][:, 0].contiguous(), P["decoder.stop_layer.bias"]
            lstm = {d: dict(ih=ops.pack_dev(P[f"encoder.lstm.0.{d}.weight_ih"]), b_ih=P[f"encoder.lstm.0.{d}.bias_ih"],
                            hh=ops.lstm_pack_fwd(P[f"encoder.lstm.0.{d}.weight_hh"], perm), b_hh=P[f"encoder.lstm.0.{d}.bias_hh"])
                    for d in ("cell_fw", "cell_bw")}
            self._packed = {"enc": [self._fold_conv(f"encoder.conv_batchnorms.{i}.") for i in range(self.encoder_conv_layers)],
                            "lstm": lstm, "key": ops.pack_dev(t(P[a + "key_layer.weight"])), "dec": dec,
                            "post": [self._fold_conv(f"postnet.conv_batchnorms.{i}.") for i in range(self.postnet_conv_layers)]}
        return self._packed

    # -- input checks (all before any launch) ----------------------------------------------------------------------
    def _check(self, text, tones, global_condition, *extra):
        for x in (text, tones, global_condition) + extra:
            if x is not None and (not x.is_cuda or x.device != self._params["embedding.weight"].device):
                raise _lib.PkError(f"Tacotron2 inputs must be CUDA tensors on the model's device {self.device} (no CPU fallback)")
        if text.dim() != 2 or text.shape[1] < 1 or not 1 <= text.shape[0] <= MAX_BATCH:
            raise ValueError(f"expected text_inputs (B <= {MAX_BATCH}, T >= 1), got {tuple(text.shape)}")
        if (tones is None) != (not self.n_tones):
            raise ValueError("tones are required exactly when the model has n_tones")
        if tones is not None and tuple(tones.shape) != tuple(text.shape):
            raise ValueError("tones must have the shape of text_inputs")
        if (global_condition is None) != (self.d_global_condition is None):
            raise ValueError("global_condition is required exactly when the model has d_global_condition")
        if global_condition is not None and tuple(global_condition.shape) != (text.shape[0], self.d_global_condition):
            raise ValueError(f"global_condition must be (B, {self.d_global_condition})")
        lo, hi = torch.aminmax(text)
        if int(lo) < 0 or int(hi) >= self.vocab_size:
            raise ValueError(f"text ids must be in [0, {self.vocab_size})")
        if tones is not None:
            lo, hi = torch.aminmax(tones)
            if int(lo) < 0 or int(hi) >= self.n_tones:
                raise ValueError(f"tone ids must be in [0, {self.n_tones})")

    @staticmethod
    def _seed(seed):
        return int(torch.randint(0, 2 ** 62, (1,)).item()) if seed is None else int(seed)

    # -- layers ----------------------------------------------------------------------------------------------------
    def _encode(self, text, tones, lens, global_condition):
        """-> (keys (B, T, dk), key_layer(keys) (B, T, 128)); with lens, the LSTM runs per sequence length and rows past it are zero."""
        P, packs = self._params, self._packs()
        B, T = text.shape
        x = ops.taco2_embed(text.long(), P["embedding.weight"], tones.long() if tones is not None else None,
                            P["embedding_tones.weight"] if tones is not None else None)
        xs = Split.from_f32(x)
        for c in packs["enc"]:
            xs = ops.conv_gemm(xs, c["w"], n=c["n"], k=c["k"], taps=self.encoder_kernel_size, bias=c["b"], act="relu", out_f32=False,
                               out_split=True)[1]
        H = self.d_encoder // 2
        h = {}
        for d, rev in (("cell_fw", False), ("cell_bw", True)):
            L = packs["lstm"][d]
            g_in = ops.conv_gemm(xs, L["ih"], n=4 * H, k=self.d_encoder, bias=L["b_ih"])[0]
            h_all, h_split, c = start_states(T, B, H, text.device)
            ops.lstm_fwd(ops.taco2_time_major(g_in, lens, reverse=rev), L["b_hh"], L["hh"], h_all, h_split, c)
            h[d] = h_all[1:]
        keys = ops.taco2_bilstm_merge(h["cell_fw"], h["cell_bw"], lens, global_condition)
        dk = keys.shape[-1]
        pkeys = ops.conv_gemm(Split.from_f32(keys), packs["key"], n=128, k=dk)[0]
        return keys, pkeys

    def _postnet(self, mel, lens=None):
        """mel + DecoderPostNet(mel), rows at and past lens zero in every layer (the reference's buffer ends there)."""
        xs = Split.from_f32(mel)
        post = self._packs()["post"]
        for i, c in enumerate(post):
            last = i == len(post) - 1
            y, xs = ops.conv_gemm(xs, c["w"], n=c["n"], k=c["k"], taps=self.postnet_kernel_size, bias=c["b"], act=None if last else "tanh",
                                  residual=mel if last else None, lens=lens, out_f32=last, out_split=not last)
        return y

    # -- public ------------------------------------------------------------------------------------------------------
    def infer(self, text_inputs, max_decoder_steps=1000, tones=None, global_condition=None, *, seed=None):
        """-> {mel_output, mel_outputs_postnet, alignments[, stop_logits]} of Tacotron2.infer (B, N, d_mels * r)."""
        self._check(text_inputs, tones, global_condition)
        if max_decoder_steps < 1:
            raise ValueError("max_decoder_steps must be >= 1")
        if self.use_stop_token and text_inputs.shape[0] != 1:
            raise ValueError("with a stop token the reference's infer loop is defined for one utterance (its `if tensor` raises for B > 1)")
        keys, pkeys = self._encode(text_inputs, tones, None, global_condition.float() if global_condition is not None else None)
        mel, align, stop, frames = ops.taco2_decode(self._packs()["dec"], keys, pkeys, int(max_decoder_steps), teacher=False,
                                                    p_prenet=self.p_prenet_dropout, seed=self._seed(seed))
        post = self._postnet(mel, frames)
        n = int(frames[0].item())          # the one host read of the call, after all launches
        out = {"mel_output": mel[:, :n], "mel_outputs_postnet": post[:, :n], "alignments": align[:, :n]}
        if stop is not None:
            out["stop_logits"] = stop[:, :n]
        return out

    def forward(self, text_inputs, text_lens, mels, output_lens=None, tones=None, global_condition=None, *, seed=None):
        """Teacher-forced Tacotron2.forward (eval): mels (B, T_mel, d_mels) with T_mel % reduction_factor == 0."""
        self._check(text_inputs, tones, global_condition, text_lens, mels, output_lens)
        B, T = text_inputs.shape
        if mels.dim() != 3 or mels.shape[0] != B or mels.shape[2] != self.d_mels or mels.shape[1] < self.r:
            raise ValueError(f"expected mels (B, T_mel >= {self.r}, {self.d_mels}), got {tuple(mels.shape)}")
        if mels.shape[1] % self.r:
            raise ValueError(f"T_mel ({mels.shape[1]}) must be a multiple of reduction_factor ({self.r})")
        if text_lens.shape != (B,) or (output_lens is not None and output_lens.shape != (B,)):
            raise ValueError("text_lens and output_lens must be (B,)")
        lo, hi = torch.aminmax(text_lens)
        if int(lo) < 1 or int(hi) > T:
            raise ValueError(f"text_lens must be in [1, {T}]")
        lens = text_lens.to(torch.int32).contiguous()
        keys, pkeys = self._encode(text_inputs, tones, lens, global_condition.float() if global_condition is not None else None)
        mel, align, stop, _ = ops.taco2_decode(self._packs()["dec"], keys, pkeys, mels.shape[1] // self.r, teacher=True,
                                               mels=mels.float().contiguous(), text_lens=lens, p_prenet=self.p_prenet_dropout,
                                               seed=self._seed(seed))
        post = self._postnet(mel)
        if output_lens is not None:
            olens = output_lens.to(torch.int32).contiguous()
            ops.mask_rows_(mel, olens)
            ops.mask_rows_(post, olens)
        out = {"mel_output": mel, "mel_outputs_postnet": post, "alignments": align}
        if stop is not None:
            out["stop_logits"] = stop
        return out


class Tacotron2Loss:
    """Tacotron2Loss.forward (validation numbers; no backward): one pk_taco2_loss block."""

    def __init__(self, use_stop_token_loss=True, use_guided_attention_loss=False, sigma=0.2):
        self.use_stop_token_loss, self.use_guided_attention_loss, self.sigma = use_stop_token_loss, use_guided_attention_loss, sigma

    def __call__(self, mel_outputs, mel_outputs_postnet, mel_targets, attention_weights=None, slens=None, plens=None, stop_logits=None):
        if mel_outputs.shape != mel_targets.shape or mel_outputs_postnet.shape != mel_targets.shape:
            raise ValueError("mel_outputs, mel_outputs_postnet and mel_targets must have one shape")
        if self.use_guided_attention_loss and (attention_weights is None or slens is None or plens is None):
            raise ValueError("the guided attention loss needs attention_weights, slens and plens")
        if self.use_stop_token_loss and (stop_logits is None or slens is None):
            raise ValueError("the stop token loss needs stop_logits and slens")
        out = ops.taco2_loss(mel_outputs, mel_outputs_postnet, mel_targets, attention_weights if self.use_guided_attention_loss else None,
                             slens, plens, self.sigma, stop_logits if self.use_stop_token_loss else None)
        losses = {"loss": out[0], "mel_loss": out[1], "post_mel_loss": out[2]}
        if self.use_guided_attention_loss:
            losses["guided_attn_loss"] = out[3]
        if self.use_stop_token_loss:
            losses["stop_loss"] = out[4]
        return losses

    forward = __call__
