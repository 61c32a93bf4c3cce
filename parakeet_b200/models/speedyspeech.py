"""SpeedySpeech on H100 - host side.

Mirrors parakeet/models/speedyspeech/speedyspeech.py of the reference: `SpeedySpeech` (:141-220) with the same constructor
arguments and state-dict key names (Linear [in, out], Conv1D [out, in, k], BatchNorm1D `_mean` / `_variance`), the eval-mode
teacher-forced `forward(text, tones, durations)`, `inference(text, tones)`, and `SpeedySpeechInference` (:223-232).
`batch_inference` is the batched form of `inference`, as FastSpeech2's.

Every FLOP runs in libparakeet_b200.so: each ResidualBlock (Conv1D -> ReLU -> BatchNorm1D, once or twice, plus the residual)
is one pk_ss_residual_block launch (csrc/speedyspeech.cu); the Linear layers run through pk_conv_gemm, the ReLU before the
encoder's last BatchNorm through pk_leaky_relu (slope 0), duration rounding through pk_duration_post (offset 0), expansion
through pk_length_regulate, the sinusoid position encoding through pk_embed_pe (alpha 1).  The embedding lookups are gathers
(no arithmetic), as in FastSpeech2.  There is one device->host copy per call: the frame counts that size the decoder.

Scope: eval-mode arithmetic only (BatchNorm uses its running statistics): a forward in training mode raises PkError.  The
train-mode forward, the losses of speedyspeech_updater.py and the update live in training/speedyspeech_step.py
(SpeedySpeechTrainStep), which does not go through this class's forward.  Every hidden size must be 128.
"""
import math

import torch

from .. import _lib, ops
from ..layer import Layer
from ..ops import Split

CHANNELS = 128
BN_EPS = 1e-5


def paddle_same_conv(kernel_size, dilation):
    """Paddle 2.1's padding="same" for a stride-1 Conv1D -> (dilation, pad_left, pad_right).

    UpdatePaddingAndDilation (paddle/fluid/operators/conv_op.h) takes the SAME branch from the UNDILATED kernel size,
    pad_sum = max(k - 1, 0), left = pad_sum // 2, right = pad_sum - left, and resets the dilation to 1.  So every SpeedySpeech
    conv runs undilated, whatever its dilation argument, and an even kernel pads one row more on the right.  The released
    checkpoints were trained under this rule; the model, the oracle and the Paddle stand-in all take it from here."""
    del dilation
    pad_sum = max(kernel_size - 1, 0)
    return 1, pad_sum // 2, pad_sum - pad_sum // 2


def _i32(t):
    return t.to(dtype=torch.int32).contiguous()


class SpeedySpeech(Layer):
    def __init__(self, vocab_size, encoder_hidden_size, encoder_kernel_size, encoder_dilations, duration_predictor_hidden_size,
                 decoder_hidden_size, decoder_output_size, decoder_kernel_size, decoder_dilations, tone_size=None, device=None,
                 seed=0):
        super().__init__(device)
        sizes = (encoder_hidden_size, duration_predictor_hidden_size, decoder_hidden_size)
        if any(s != CHANNELS for s in sizes):
            raise _lib.PkError(f"SpeedySpeech runs hidden size {CHANNELS} only (got {sizes})")
        for k in (encoder_kernel_size, decoder_kernel_size):
            if not 1 <= k <= 4:
                raise _lib.PkError(f"SpeedySpeech kernel sizes must be in [1, 4] (got {k})")
        self.vocab_size, self.tone_size = vocab_size, tone_size
        self.encoder_kernel_size, self.decoder_kernel_size = encoder_kernel_size, decoder_kernel_size
        # stored as given; under Paddle's padding="same" they do not change the computation (paddle_same_conv)
        self.encoder_dilations, self.decoder_dilations = list(encoder_dilations), list(decoder_dilations)
        self.odim = decoder_output_size
        C = CHANNELS
        g = torch.Generator().manual_seed(seed)

        def uniform(*shape, bound):
            return (torch.rand(*shape, generator=g) * 2 - 1) * bound

        def lin(name, i, o):
            self._register(name + ".weight", uniform(i, o, bound=math.sqrt(6.0 / (i + o))))       # Paddle Linear: [in, out]
            self._register(name + ".bias", torch.zeros(o))

        def res_block(pre, k, n):
            for j in range(n):
                q = f"{pre}blocks.{j}."
                self._register(q + "0.weight", uniform(C, C, k, bound=1.0 / math.sqrt(C * k)))
                self._register(q + "0.bias", torch.zeros(C))
                bn(q + "2")

        def bn(name):
            self._register(name + ".weight", torch.ones(C))
            self._register(name + ".bias", torch.zeros(C))
            self._register(name + "._mean", torch.zeros(C))
            self._register(name + "._variance", torch.ones(C))

        emb = torch.randn(vocab_size, C, generator=g)
        emb[0] = 0
        self._register("encoder.embedding.text_embedding.weight", emb)
        if tone_size:
            tone = torch.randn(tone_size, C, generator=g)
            tone[0] = 0
            self._register("encoder.embedding.tone_embedding.weight", tone)
        lin("encoder.prenet.0", C, C)
        for i in range(len(self.encoder_dilations)):
            res_block(f"encoder.res_blocks.{i}.", encoder_kernel_size, 2)
        lin("encoder.postnet1.0", C, C)
        bn("encoder.postnet2.1")
        lin("encoder.postnet2.2", C, C)
        for i, k in enumerate((4, 3, 1)):
            res_block(f"duration_predictor.layers.{i}.", k, 1)
        lin("duration_predictor.layers.3", C, 1)
        for i in range(len(self.decoder_dilations)):
            res_block(f"decoder.res_blocks.{i}.", decoder_kernel_size, 2)
        lin("decoder.postnet1.0", C, C)
        res_block("decoder.postnet2.0.", decoder_kernel_size, 2)
        lin("decoder.postnet2.1", C, decoder_output_size)

    # ------------------------------------------------------------------------------------------------------------
    # kernel-ready weights (once per weight change)
    # ------------------------------------------------------------------------------------------------------------
    def _pack(self):
        if self._packed is not None:
            return self._packed
        p = {k: v.detach().float().cpu() for k, v in self._params.items()}
        dev = self.device

        def dv(t):
            return t.contiguous().to(dev)

        def bn_affine(name):
            s = p[name + ".weight"] / torch.sqrt(p[name + "._variance"] + BN_EPS)
            return s, p[name + ".bias"] - p[name + "._mean"] * s

        def lin(name):
            w = p[name + ".weight"]                                          # [in, out]
            return dict(w=ops.pack_weight(w.t(), dev), b=dv(p[name + ".bias"]), n=w.shape[1])

        def res_block(pre, k, n):
            convs = []
            for j in range(n):
                q = f"{pre}blocks.{j}."
                s, t = bn_affine(q + "2")
                convs.append(dict(w=ops.pack_weight(p[q + "0.weight"], dev), b=dv(p[q + "0.bias"]), s=dv(s), t=dv(t)))
            _, left, _ = paddle_same_conv(k, 1)
            return dict(convs=convs, taps=k, left=left)

        pk = dict(emb=dv(p["encoder.embedding.text_embedding.weight"]))
        if self.tone_size:
            pk["tone"] = dv(p["encoder.embedding.tone_embedding.weight"])
        pk["prenet"] = lin("encoder.prenet.0")
        pk["enc_blocks"] = [res_block(f"encoder.res_blocks.{i}.", self.encoder_kernel_size, 2) for i in range(len(self.encoder_dilations))]
        pk["enc_post1"] = lin("encoder.postnet1.0")
        # ReLU -> BatchNorm1D -> Linear: the BN affine folds exactly into the Linear (no padding there)
        s, t = bn_affine("encoder.postnet2.1")
        w, b = p["encoder.postnet2.2.weight"], p["encoder.postnet2.2.bias"]
        pk["enc_post2"] = dict(w=ops.pack_weight((s[:, None] * w).t(), dev), b=dv(t @ w + b), n=w.shape[1])
        pk["dur_blocks"] = [res_block(f"duration_predictor.layers.{i}.", k, 1) for i, k in enumerate((4, 3, 1))]
        pk["dur_out"] = lin("duration_predictor.layers.3")
        pk["dec_blocks"] = [res_block(f"decoder.res_blocks.{i}.", self.decoder_kernel_size, 2) for i in range(len(self.decoder_dilations))]
        pk["dec_post1"] = lin("decoder.postnet1.0")
        pk["dec_post2_block"] = res_block("decoder.postnet2.0.", self.decoder_kernel_size, 2)
        pk["dec_out"] = lin("decoder.postnet2.1")
        pk["one"] = torch.ones(1, device=dev)
        self._packed = pk
        return pk

    # ------------------------------------------------------------------------------------------------------------
    # building blocks
    # ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def _blocks(x, xs, blocks, lens):
        for blk in blocks:
            x, xs = ops.ss_residual_block(x, xs, blk["convs"], blk["taps"], blk["left"], lens)
        return x, xs

    @staticmethod
    def _linear(xs, lin, lens, residual=None, out_split=False):
        return ops.conv_gemm(xs, lin["w"], n=lin["n"], k=CHANNELS, bias=lin["b"], residual=residual, lens=lens, out_split=out_split)

    def _embed_ids(self, table, ids):
        """nn.Embedding(padding_idx=0): rows of the table, zeros for id 0 (a gather and a fill: no arithmetic)."""
        e = table.index_select(0, ids.reshape(-1)).reshape(tuple(ids.shape) + (table.shape[1],))
        return e.masked_fill((ids == 0).unsqueeze(-1), 0.0)

    def _stage_a(self, text, tones, lens):
        """SpeedySpeechEncoder.forward (:100-106) and DurationPredictor.forward (:117-118) -> (encodings fp32 (B, T, C),
        log-durations (B, T)).  lens: int32 (B,) for utterance-local padding (rows >= lens are zero), or None."""
        pk = self._pack()
        emb = self._embed_ids(pk["emb"], text)
        if tones is not None:
            ops.axpy_(1.0, self._embed_ids(pk["tone"], tones), emb)     # TextEmbedding, concat=False: text + tone
        if lens is not None:
            ops.mask_rows_(emb, lens)
        pre, pre_s = ops.conv_gemm(Split.from_f32(emb), pk["prenet"]["w"], n=CHANNELS, k=CHANNELS, bias=pk["prenet"]["b"],
                                   act="relu", lens=lens, out_split=True)
        _, xs = self._blocks(pre, pre_s, pk["enc_blocks"], lens)
        x = self._linear(xs, pk["enc_post1"], lens, residual=pre)[0]     # embedding + postnet1(res_blocks(embedding))
        enc, enc_s = self._linear(ops.relu_split(x), pk["enc_post2"], lens, out_split=True)
        _, hs = self._blocks(enc, enc_s, pk["dur_blocks"], lens)
        d = self._linear(hs, pk["dur_out"], lens)[0]
        return enc, d.reshape(d.shape[0], d.shape[1])

    def _stage_b(self, enc, d_int, t_dec, lens):
        """expand + sinusoid_position_encoding + SpeedySpeechDecoder.forward (:134-138) for a decoder length known on the host."""
        pk = self._pack()
        x, _ = ops.length_regulate(enc, d_int, t_dec)
        x = ops.embed_pe(None, None, x, pk["one"], lens)
        xs = Split.from_f32(x)
        _, hs = self._blocks(x, xs, pk["dec_blocks"], lens)
        x2, x2s = self._linear(hs, pk["dec_post1"], lens, residual=x, out_split=True)
        _, hs = self._blocks(x2, x2s, [pk["dec_post2_block"]], lens)
        return self._linear(hs, pk["dec_out"], lens)[0]

    def _check(self, text, tones):
        if self.training:
            raise _lib.PkError("SpeedySpeech runs in eval mode only (call .eval()): train-mode BatchNorm is not implemented")
        if tones is not None and not self.tone_size:
            raise _lib.PkError("tones given to a SpeedySpeech built without tone_size")
        if not text.is_cuda or (tones is not None and not tones.is_cuda):
            raise _lib.PkError("SpeedySpeech needs CUDA tensors (no CPU fallback)")

    def _infer(self, text, lens, tones):
        """Inference through CUDA graphs: every utterance is computed as if alone (utterance-local padding), so the decoder
        length can be rounded up to a bucket of 32 frames - padded rows are inert and sliced off - and the two shape-static
        halves replay as graphs.  Returns (mel (B, L, odim), frame counts int32 (B,), durations int64 (B, T))."""
        self._check(text, tones)
        B, T = text.shape
        text = text.to(torch.int64).contiguous()
        lens = _i32(lens.to(text.device))
        inputs = [text, lens] + ([tones.to(torch.int64).contiguous()] if tones is not None else [])

        def fa(x_, l_, *t_):
            enc, d = self._stage_a(x_, t_[0] if t_ else None, l_)
            _, d_int = ops.duration_post(d, l_, offset=0.0)                 # round(exp(d)), half away from zero
            return enc, d_int, ops.length_regulator_lens(d_int)
        enc, d_int, frames = self._graphs.run(("a", B, T, tones is not None), fa, inputs)
        t_dec = int(frames.max().item())         # the one D2H copy: sizes the decoder
        if t_dec == 0:
            return torch.zeros(B, 0, self.odim, device=text.device), frames.clone(), d_int.clone()
        bucket = (t_dec + 31) // 32 * 32
        mel = self._graphs.run(("b", B, T, bucket), lambda e_, d_, f_: self._stage_b(e_, d_, bucket, f_), [enc, d_int, frames])
        return mel[:, :t_dec].clone(), frames.clone(), d_int.clone()

    # ------------------------------------------------------------------------------------------------------------
    # public API (reference :166-220)
    # ------------------------------------------------------------------------------------------------------------
    def forward(self, text, tones, durations):
        """Eval-mode teacher-forced forward (:166-184): text / tones / durations (B, T) -> (decoded (B, L, odim),
        pred_durations (B, T)), L = the longest utterance's sum of durations.  No lengths: padded tokens are live and the
        decoder sees every row, exactly as in the reference."""
        self._check(text, tones)
        text = text.to(torch.int64).contiguous()
        tones = tones.to(torch.int64).contiguous() if tones is not None else None
        enc, d_pred = self._stage_a(text, tones, None)
        d_int = durations.to(device=text.device, dtype=torch.int64).contiguous()
        t_dec = int(ops.length_regulator_lens(d_int).max().item())
        if t_dec == 0:
            return torch.zeros(text.shape[0], 0, self.odim, device=text.device), d_pred
        return self._stage_b(enc, d_int, t_dec, None), d_pred

    def inference(self, text, tones=None):
        """(T,) phone ids (and tone ids) -> mel (L, odim) (:186-220)."""
        xs = text.reshape(1, -1)
        lens = torch.full((1,), xs.shape[1], dtype=torch.int32, device=xs.device)
        mel, _, _ = self._infer(xs, lens, tones.reshape(1, -1) if tones is not None else None)
        return mel[0]

    def batch_inference(self, text, text_lengths, tones=None):
        """Batched form of `inference`: padded ids (B, Tmax) + lengths -> (mel (B, Lmax, odim), frame counts (B,) int32,
        durations (B, Tmax) int64).  Each utterance is computed exactly as if it had been passed to `inference` alone; rows
        past an utterance's own frame count are zero."""
        return self._infer(text, text_lengths, tones)


class SpeedySpeechInference(Layer):
    """reference speedyspeech.py:223-232."""

    def __init__(self, normalizer, model):
        super().__init__(model.device)
        self.normalizer = normalizer
        self.acoustic_model = model

    def forward(self, phones, tones=None):
        normalized_mel = self.acoustic_model.inference(phones, tones)
        return self.normalizer.inverse(normalized_mel)
