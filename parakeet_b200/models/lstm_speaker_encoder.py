"""GE2E speaker encoder (reference: parakeet/models/lstm_speaker_encoder.py `LSTMSpeakerEncoder`; recipe examples/ge2e).

3 LSTM layers over log-mel partials, Linear + ReLU on the last layer's final h, L2 normalisation; the GE2E softmax loss over
(speakers, utterances, dims).  Each LSTM layer is one `pk_conv_gemm` for the input half of the gates over all steps and one
persistent `pk_lstm_fwd` launch for the recurrence (csrc/lstm.cu); the loss and similarity matrix are one `pk_ge2e_loss` block.
The EER is computed on the host (numpy + scipy), as the reference does with sklearn.

State-dict keys are Paddle 2.1's (`lstm.{l}.cell.weight_ih` ...); the flat form of later Paddle releases (`lstm.weight_ih_l{l}`)
is accepted on load (DESIGN.md section 2).
"""
import re

import numpy as np
import torch

from .. import _lib, ops
from ..layer import Layer
from ..ops import Split

HIDDEN_SIZES = (64, 256)       # the hidden sizes pk_lstm_fwd / pk_lstm_bwd are instantiated for
_FLAT_KEY = re.compile(r"^lstm\.(weight_ih|weight_hh|bias_ih|bias_hh)_l(\d+)$")


def lstm_key(layer, part):
    return f"lstm.{layer}.cell.{part}"


def canonical_keys(state):
    """Paddle >= 2.2's flat LSTM keys -> the 2.1 LayerList form; other keys unchanged."""
    out = {}
    for k, v in state.items():
        m = _FLAT_KEY.match(k)
        out[lstm_key(int(m.group(2)), m.group(1)) if m else k] = v
    return out


def roc_curve(labels, scores):
    """sklearn.metrics.roc_curve(labels, scores) (drop_intermediate=True): -> (fpr, tpr)."""
    order = np.argsort(scores, kind="mergesort")[::-1]
    s, y = scores[order], labels[order].astype(np.float64)
    distinct = np.where(np.diff(s))[0]
    idx = np.r_[distinct, y.size - 1]
    tps = np.cumsum(y)[idx]
    fps = 1 + idx - tps
    if tps.size > 2:
        keep = np.where(np.r_[True, np.logical_or(np.diff(fps, 2), np.diff(tps, 2)), True])[0]
        fps, tps = fps[keep], tps[keep]
    fps, tps = np.r_[0, fps], np.r_[0, tps]
    return fps / fps[-1], tps / tps[-1]


def equal_error_rate(sim, num_speakers, utterances_per_speaker):
    """The reference's EER of a similarity matrix (N*M, N): one-hot labels of the own speaker, roc curve, brentq on 1 - x = tpr(x)."""
    from scipy.interpolate import interp1d
    from scipy.optimize import brentq
    sim = np.asarray(sim, dtype=np.float32)
    labels = np.zeros_like(sim)
    labels[np.arange(sim.shape[0]), np.arange(sim.shape[0]) // utterances_per_speaker] = 1
    fpr, tpr = roc_curve(labels.reshape(-1), sim.reshape(-1))
    return brentq(lambda x: 1. - x - interp1d(fpr, tpr)(x), 0., 1.)


def start_states(T, B, H, device, h0=None, c0=None, keep_c=False):
    """-> (h_all (T+1, B, H), its Split planes, c): h0 (zeros if None) in slab 0 of both; c is (B, H) holding c0, or with
    keep_c (T+1, B, H) with c0 in slab 0 (training keeps every c_t)."""
    h_all = torch.empty(T + 1, B, H, dtype=torch.float32, device=device)
    h_split = Split.empty((T + 1, B, H), device)
    c = torch.empty((T + 1, B, H) if keep_c else (B, H), dtype=torch.float32, device=device)
    c0_slab = c[0] if keep_c else c
    if h0 is None:
        h_all[0].zero_()
        h_split.hi[0].zero_()
        h_split.lo[0].zero_()
    else:
        h_all[0].copy_(h0)
        s0 = Split.from_f32(h_all[0])
        h_split.hi[0].copy_(s0.hi)
        h_split.lo[0].copy_(s0.lo)
    if c0 is None:
        c0_slab.zero_()
    else:
        c0_slab.copy_(c0)
    return h_all, h_split, c


class LSTMSpeakerEncoder(Layer):
    def __init__(self, n_mels, num_layers, hidden_size, output_size, device=None):
        super().__init__(device)
        if hidden_size not in HIDDEN_SIZES:
            raise ValueError(f"the LSTM kernels are built for hidden sizes {HIDDEN_SIZES} (got {hidden_size})")
        self.n_mels, self.num_layers, self.hidden_size, self.output_size = n_mels, num_layers, hidden_size, output_size
        g = torch.Generator().manual_seed(0)
        k = hidden_size ** -0.5
        u = lambda *shape: (torch.rand(*shape, generator=g) * 2 - 1) * k       # Paddle's LSTM / Linear default: uniform(+-1/sqrt(H))
        for l in range(num_layers):
            self._register(lstm_key(l, "weight_ih"), u(4 * hidden_size, n_mels if l == 0 else hidden_size))
            self._register(lstm_key(l, "weight_hh"), u(4 * hidden_size, hidden_size))
            self._register(lstm_key(l, "bias_ih"), u(4 * hidden_size))
            self._register(lstm_key(l, "bias_hh"), u(4 * hidden_size))
        self._register("linear.weight", u(hidden_size, output_size))
        self._register("linear.bias", u(output_size))
        self._register("similarity_weight", torch.tensor([10.0]))
        self._register("similarity_bias", torch.tensor([-5.0]))

    def set_state_dict(self, state):
        super().set_state_dict(canonical_keys(state))

    load_dict = set_state_dict

    def _packs(self):
        if self._packed is None:
            P = self._params
            perm = ops.lstm_gate_perm(self.hidden_size, self.device)
            self._packed = {"ih": [ops.pack_dev(P[lstm_key(l, "weight_ih")]) for l in range(self.num_layers)],
                            "hh": [ops.lstm_pack_fwd(P[lstm_key(l, "weight_hh")], perm) for l in range(self.num_layers)],
                            "lin": ops.pack_dev(P["linear.weight"].t())}
        return self._packed

    def _check(self, utterances):
        if not utterances.is_cuda:
            raise _lib.PkError("LSTMSpeakerEncoder needs CUDA tensors (no CPU fallback)")
        if utterances.dim() != 3 or utterances.shape[2] != self.n_mels or utterances.shape[1] < 1 or utterances.shape[0] < 1:
            raise ValueError(f"expected utterances (B, T >= 1, {self.n_mels}), got {tuple(utterances.shape)}")

    def _last_h(self, utterances, initial_states=None):
        """the top layer's h after the last step, (B, H)."""
        self._check(utterances)
        B, T, _ = utterances.shape
        H, P, packs = self.hidden_size, self._params, self._packs()
        inp = utterances.float().transpose(0, 1).contiguous().reshape(1, T * B, self.n_mels)     # time-major
        counters = ops.lstm_counters(B, T, utterances.device)
        for l in range(self.num_layers):
            g_in = ops.conv_gemm(Split.from_f32(inp), packs["ih"][l], n=4 * H, k=inp.shape[-1], bias=P[lstm_key(l, "bias_ih")])[0]
            h_all, h_split, c = start_states(T, B, H, utterances.device, None if initial_states is None else initial_states[0][l],
                                             None if initial_states is None else initial_states[1][l])
            ops.lstm_fwd(g_in.reshape(T, B, 4 * H), P[lstm_key(l, "bias_hh")], packs["hh"][l], h_all, h_split, c, counters=counters)
            inp = h_all[1:].reshape(1, T * B, H)
        return h_all[T]

    def _embed(self, h):
        """F.normalize(relu(linear(h)))."""
        P = self._params
        e = ops.conv_gemm(Split.from_f32(h.reshape(1, *h.shape)), self._packs()["lin"], n=self.output_size, k=self.hidden_size,
                          bias=P["linear.bias"], act="relu")[0]
        return ops.l2_normalize_axis1(e.reshape(h.shape[0], self.output_size))

    def embed_sequences(self, utterances, initial_states=None, reduce=False):
        """utterances (B, T, n_mels) -> normalised embeddings (B, output_size), or with reduce=True their normalised mean."""
        if initial_states is not None:
            h0, c0 = initial_states
            shape = (self.num_layers, utterances.shape[0], self.hidden_size)
            if tuple(h0.shape) != shape or tuple(c0.shape) != shape:
                raise ValueError(f"initial states must be two tensors of shape {shape}")
            if not (h0.is_cuda and c0.is_cuda):
                raise _lib.PkError("initial states must be CUDA tensors (no CPU fallback)")
        e = self._embed(self._last_h(utterances, initial_states))
        if reduce:
            offsets = torch.tensor([0, e.shape[0]], dtype=torch.int32, device=e.device)
            return ops.segment_mean_normalize(e, offsets)[0]
        return e

    def embed_utterance(self, utterances, initial_states=None):
        return self.embed_sequences(utterances, initial_states, reduce=True)

    def embed_utterances(self, partials):
        """A list of U utterances' partials (each (P_u, T, n_mels), the same T) -> (U, output_size), equal to per-utterance
        embed_utterance: all partials run as one recurrence, then a segmented mean and normalisation."""
        if len(partials) == 0:
            raise ValueError("no utterances")
        counts = [int(p.shape[0]) for p in partials]
        if min(counts) < 1:
            raise ValueError("every utterance needs at least one partial")
        x = torch.cat([p.to(self.device, torch.float32) for p in partials], 0)
        e = self._embed(self._last_h(x))
        offsets = torch.tensor(np.r_[0, np.cumsum(counts)], dtype=torch.int32, device=e.device)
        return ops.segment_mean_normalize(e, offsets)

    def similarity_matrix(self, embeds):
        """embeds (N, M, C) -> (N*M, N): the reference's similarity matrix (own speaker: exclusive centroid), times w plus b."""
        N, M, C = self._loss_shape(embeds)
        return ops.ge2e_loss(embeds.float().contiguous(), N, M, C, self._params["similarity_weight"], self._params["similarity_bias"])[1]

    def _loss_shape(self, embeds):
        if not embeds.is_cuda or embeds.device != self._params["similarity_weight"].device:
            raise _lib.PkError(f"embeds must be a CUDA tensor on the model's device {self.device} (no CPU fallback)")
        if embeds.dim() != 3:
            raise ValueError(f"expected embeds (N, M, C), got {tuple(embeds.shape)}")
        N, M, C = embeds.shape
        if M < 2:
            raise ValueError(f"the exclusive centroid needs at least 2 utterances per speaker (got {M})")
        return N, M, C

    def loss(self, embeds):
        """embeds (N, M, C) -> (loss (1,) on the device, eer float)."""
        N, M, C = self._loss_shape(embeds)
        loss, sim = ops.ge2e_loss(embeds.float().contiguous(), N, M, C, self._params["similarity_weight"],
                                  self._params["similarity_bias"])[:2]
        return loss, equal_error_rate(sim.cpu().numpy(), N, M)

    @staticmethod
    def grouping(batch, output_size, num_speakers):
        """The reference forward's reshape of the (batch, output_size) embeddings to [num_speakers, -1, num_speakers]: -> M'."""
        if num_speakers < 1 or (batch * output_size) % (num_speakers * num_speakers):
            raise ValueError(f"{batch} x {output_size} embeddings cannot be reshaped to [{num_speakers}, -1, {num_speakers}]")
        m = batch * output_size // (num_speakers * num_speakers)
        if m < 2:
            raise ValueError(f"the reshape [{num_speakers}, -1, {num_speakers}] leaves {m} < 2 rows per speaker")
        return m

    def forward(self, utterances, num_speakers, initial_states=None):
        """-> (loss, eer) as LSTMSpeakerEncoder.forward: the embeddings reshaped to [num_speakers, -1, num_speakers]."""
        self.grouping(utterances.shape[0], self.output_size, num_speakers)
        e = self.embed_sequences(utterances, initial_states)
        return self.loss(e.reshape(num_speakers, -1, num_speakers))
