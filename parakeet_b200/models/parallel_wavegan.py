"""Parallel WaveGAN generator on H100 - host side.

Mirrors parakeet/models/parallel_wavegan/parallel_wavegan.py of the reference: `PWGGenerator` (:318-520) with the same
constructor keywords, `forward(x, c)`, `inference(c)`, `apply_weight_norm` / `remove_weight_norm`, and the same
state-dict key names (`first_conv.*`, `upsample_net.conv_in.weight`, `upsample_net.upsample.up_layers.{1,3,5,7}.weight`,
`conv_layers.{i}.{conv,conv1x1_aux,conv1x1_out,conv1x1_skip}.*`, `last_conv_layers.{1,3}.*`; `weight_g` [out] /
`weight_v` while weight norm is applied); `PWGInference` (:766-775).

All arithmetic runs in libparakeet_b200.so (pk_pwg_* in include/parakeet_b200.h); torch only owns the buffers.
"""
import ctypes as C
import math
from typing import Any, Dict, List, Optional

import numpy as np
import torch

from .. import _lib, ops
from ..layer import Layer
from ..ops import Split, _ptr, _stream

from .._lib import PwgLayerArgs


def _declare():
    _lib.lib()


def _split_host(w, device):
    hi = w.to(torch.bfloat16)
    lo = (w - hi.float()).to(torch.bfloat16)
    return Split(hi.to(device).contiguous(), lo.to(device).contiguous())


class PWGGenerator(Layer):
    """Wave generator of Parallel WaveGAN (reference parallel_wavegan.py:318-443 for the constructor)."""

    def __init__(self,
                 in_channels: int = 1,
                 out_channels: int = 1,
                 kernel_size: int = 3,
                 layers: int = 30,
                 stacks: int = 3,
                 residual_channels: int = 64,
                 gate_channels: int = 128,
                 skip_channels: int = 64,
                 aux_channels: int = 80,
                 aux_context_window: int = 2,
                 dropout: float = 0.,
                 bias: bool = True,
                 use_weight_norm: bool = True,
                 use_causal_conv: bool = False,
                 upsample_scales: List[int] = [4, 4, 4, 4],
                 nonlinear_activation: Optional[str] = None,
                 nonlinear_activation_params: Dict[str, Any] = {},
                 interpolate_mode: str = "nearest",
                 freq_axis_kernel_size: int = 1,
                 device=None,
                 seed: int = 0):
        super().__init__(device)
        if use_causal_conv:
            raise NotImplementedError("use_causal_conv=True is out of scope (the reference's causal branch indexes "
                                      "instead of slicing, parallel_wavegan.py:305)")
        if nonlinear_activation is not None:
            raise NotImplementedError("upsample-net activations are not used by the shipped configs")
        if interpolate_mode != "nearest" or freq_axis_kernel_size != 1:
            raise NotImplementedError("only nearest interpolation / freq_axis_kernel_size=1 are supported")
        if (in_channels, out_channels, kernel_size, residual_channels, gate_channels, skip_channels) != (1, 1, 3, 64, 128, 64):
            raise NotImplementedError("the sm_90a kernels are specialised for 1/1 io channels, kernel 3, 64/128/64 channels")
        if not (64 < aux_channels <= 128 and aux_channels % 8 == 0):
            raise NotImplementedError("aux_channels must be in (64, 128] and a multiple of 8")
        if dropout != 0.0:
            raise NotImplementedError("dropout > 0 is a training-time feature (next round)")
        assert layers % stacks == 0
        self.in_channels, self.out_channels = in_channels, out_channels
        self.aux_channels, self.aux_context_window = aux_channels, aux_context_window
        self.layers, self.stacks, self.kernel_size = layers, stacks, kernel_size
        self.upsample_scales = list(upsample_scales)
        self.upsample_factor = int(np.prod(upsample_scales))
        self.use_bias = bias
        self._weight_norm = False
        self._ws = {}

        g = torch.Generator().manual_seed(seed)

        def conv(name, o, i, *k, with_bias=True):
            bound = 1.0 / math.sqrt(i * math.prod(k))
            self._register(name + ".weight", (torch.rand(o, i, *k, generator=g) * 2 - 1) * bound)
            if with_bias:
                self._register(name + ".bias", (torch.rand(o, generator=g) * 2 - 1) * bound)

        R, G, S, A = residual_channels, gate_channels, skip_channels, aux_channels
        conv("first_conv", R, in_channels, 1)
        conv("upsample_net.conv_in", A, A, 2 * aux_context_window + 1, with_bias=False)
        for i, s in enumerate(self.upsample_scales):
            conv(f"upsample_net.upsample.up_layers.{2 * i + 1}", 1, 1, 1, 2 * s + 1, with_bias=False)
        for i in range(layers):
            pre = f"conv_layers.{i}."
            conv(pre + "conv", G, R, kernel_size, with_bias=bias)
            conv(pre + "conv1x1_aux", G, A, 1, with_bias=False)
            conv(pre + "conv1x1_out", R, G // 2, 1, with_bias=bias)
            conv(pre + "conv1x1_skip", S, G // 2, 1, with_bias=bias)
        conv("last_conv_layers.1", S, S, 1)
        conv("last_conv_layers.3", out_channels, S, 1)
        if use_weight_norm:
            self.apply_weight_norm()

    # -- weight norm (reference :474-496) ---------------------------------------------------------------------
    def apply_weight_norm(self):
        """weight -> (weight_g [out], weight_v) with g = ||v|| (paddle.nn.utils.weight_norm, dim=0)."""
        if self._weight_norm:
            return
        new = type(self._params)()
        for k, v in self._params.items():
            if k.endswith(".weight"):
                new[k + "_g"] = v.reshape(v.shape[0], -1).norm(dim=1)
                new[k + "_v"] = v
            else:
                new[k] = v
        self._params = new
        self._weight_norm = True
        self._packed = None

    def remove_weight_norm(self):
        if not self._weight_norm:
            return
        self._params = type(self._params)(self._folded().items())
        self._weight_norm = False
        self._packed = None

    def _folded(self):
        """state with weight_g / weight_v folded into weight = g * v / ||v|| (done once per weight change)."""
        if not self._weight_norm:
            return self._params
        out = type(self._params)()
        for k, v in self._params.items():
            if k.endswith("weight_g"):
                continue
            if k.endswith("weight_v"):
                g = self._params[k[:-1] + "g"]
                norm = v.reshape(v.shape[0], -1).norm(dim=1)
                out[k[:-2]] = v * (g / norm).reshape([-1] + [1] * (v.dim() - 1))
            else:
                out[k] = v
        return out

    # -- kernel-ready weights ------------------------------------------------------------------------------------
    def _pack(self):
        if self._packed is not None:
            return self._packed
        p = {k: v.detach().float().cpu() for k, v in self._folded().items()}
        dev = self.device
        pk = {}
        pk["conv_in_w"] = p["upsample_net.conv_in.weight"].contiguous().to(dev)
        fir = [p[f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"].reshape(-1) for i in range(len(self.upsample_scales))]
        pk["fir_host"] = np.ascontiguousarray(torch.cat(fir).numpy(), dtype=np.float32)
        pk["scales_host"] = np.asarray(self.upsample_scales, dtype=np.int32)
        pk["first_w"] = p["first_conv.weight"].reshape(-1).contiguous().to(dev)
        pk["first_b"] = p["first_conv.bias"].contiguous().to(dev)
        A = self.aux_channels
        layers = []
        zeros64 = torch.zeros(64)
        for i in range(self.layers):
            pre = f"conv_layers.{i}."
            w = p[pre + "conv.weight"]                       # [128, 64, 3]
            w1 = torch.zeros(128, 5 * 64)
            for tap in range(3):
                w1[:, tap * 64:(tap + 1) * 64] = w[:, :, tap]
            w1[:, 192:192 + A] = p[pre + "conv1x1_aux.weight"][:, :, 0]
            w2 = torch.cat([p[pre + "conv1x1_skip.weight"][:, :, 0], p[pre + "conv1x1_out.weight"][:, :, 0]], dim=0)  # [128, 64]
            b1 = p.get(pre + "conv.bias", torch.zeros(128))
            b2 = torch.cat([p.get(pre + "conv1x1_skip.bias", zeros64), p.get(pre + "conv1x1_out.bias", zeros64)])
            # the layer biases are HOST arrays: pk_pwg_residual_layer copies them into the kernel's parameter block
            layers.append(dict(w1=_split_host(w1, dev), w2=_split_host(w2, dev),
                               b1=np.ascontiguousarray(b1.numpy(), dtype=np.float32),
                               b2=np.ascontiguousarray(b2.numpy(), dtype=np.float32), dil=2 ** (i % (self.layers // self.stacks))))
        pk["layers"] = layers
        pk["skip_bias_sum"] = torch.stack([p.get(f"conv_layers.{i}.conv1x1_skip.bias", zeros64) for i in range(self.layers)]).double().sum(0).float().contiguous().to(dev)
        pk["tail_w1"] = p["last_conv_layers.1.weight"][:, :, 0].contiguous().to(dev)
        pk["tail_b1"] = p["last_conv_layers.1.bias"].contiguous().to(dev)
        pk["tail_w2"] = p["last_conv_layers.3.weight"].reshape(-1).contiguous().to(dev)
        pk["tail_b2"] = p["last_conv_layers.3.bias"].contiguous().to(dev)
        # the ends of the frame-rate stack (pk_pwg_layer_fc_args): layer 0 computes first_conv itself, from HOST vectors of
        # first_conv and of W1_tap . w, W1_tap . b per tap (float64 here); the last layer runs the tail, on the split planes
        # of last_conv_layers.1 and HOST copies of the tail vectors
        fw, fb = p["first_conv.weight"].reshape(-1).double(), p["first_conv.bias"].double()
        w0 = p["conv_layers.0.conv.weight"].double()                                   # [128, 64, 3]
        host = lambda t: np.ascontiguousarray(t.numpy(), dtype=np.float32)  # noqa: E731
        pk["first_host"] = dict(w=host(fw), b=host(fb), u=host(torch.einsum("oik,i->ko", w0, fw)),
                                v=host(torch.einsum("oik,i->ko", w0, fb)))
        pk["tail_host"] = dict(w1=_split_host(pk["tail_w1"].cpu(), dev), b1=host(pk["tail_b1"].cpu()),
                               w2=host(pk["tail_w2"].cpu()), b2=host(pk["tail_b2"].cpu()),
                               skip_bias=host(pk["skip_bias_sum"].cpu()))
        self._packed = pk
        return pk

    def _workspace(self, B, T):
        key = (B, T)
        ws = self._ws.get(key)
        if ws is None:
            self._ws.clear()
            self._graphs.clear()          # captured forwards point into the old workspace
            dev = self.device
            ws = dict(xa=Split.zeros((B, T, 64), dev), xb=Split.zeros((B, T, 64), dev),
                      c=Split.empty((B, T, self.aux_channels), dev) if not self._uses_frame_cond() else None,   # sample-rate path only
                      skip=torch.empty(B, T, 64, dtype=torch.float32, device=dev),
                      conv_in=torch.empty(B, T // self.upsample_factor, self.aux_channels, dtype=torch.float32, device=dev))
            self._ws[key] = ws
        return ws

    @staticmethod
    def _frame_cond():
        """True.  bench.py calls this to label its roofline kernel: its workload runs the frame-rate path."""
        return True

    def _uses_frame_cond(self):
        """Whether this generator runs the frame-rate path: the compact band tables are exact for its upsample_scales (hop >= 256
        and the upsampler's padding reaches at most EDGE samples into an utterance; _pwg_frame_cond.frame_rate_exact).  Other
        configs, e.g. [2, 16, 8] or a hop of 64, run the sample-rate kernel."""
        from ._pwg_frame_cond import frame_rate_exact
        return frame_rate_exact(self.upsample_scales)

    # -- forward (reference :445-472) ------------------------------------------------------------------------------
    def forward(self, x, c, lens=None):
        """x: (B, 1, T) noise, c: (B, aux, T' + 2*aux_context_window) -> (B, 1, T).

        `lens` (optional, int32 (B,) valid samples per utterance) lets a ragged batch run as one call: every
        utterance is then generated exactly as if it were alone (zero padding at its own end).

        A repeated (B, T, lengths) replays as ONE CUDA graph (eager the first time, captured the second): the forward is ~40
        launches, each with a handful of tensor-map encodes on the host - invisible at batch 32 x 400 frames (33 ms of GPU work),
        but most of the latency of a single utterance or of a 4-utterance shard."""
        _declare()
        if not (x.is_cuda and c.is_cuda):
            raise _lib.PkError("PWGGenerator.forward needs CUDA tensors (no CPU fallback)")
        B, _, T = x.shape
        frames = c.shape[-1] - 2 * self.aux_context_window
        assert frames * self.upsample_factor == T, (c.shape, x.shape)   # reference :462
        lens_key = None
        if lens is not None:
            assert lens.dtype == torch.int32 and lens.is_cuda
            # host copy of the lengths: they select the band-table end blocks (lengths are host data in the reference's callers
            # too, synthesize.py:96-104).  An utterance is a whole number of frames: a length that is not, or one past T, would
            # give band tables and conditioning that disagree with the rows the layer kernels treat as live.
            hop = self.upsample_factor
            lens_h = lens.cpu().tolist() if lens.dim() == 1 and lens.shape[0] == B else None
            if lens_h is None or any(v < 0 or v > T or v % hop for v in lens_h):
                raise _lib.PkError(f"lens must hold {B} lengths in samples, each a multiple of hop {hop} in [0, {T}] "
                                   f"(got {lens.cpu().tolist()})")
            lens_key = tuple(v // hop for v in lens_h)
        eager = not self._uses_frame_cond() or getattr(self, "_layer_events", None) is not None
        if eager:
            return self._forward_impl(x, c, lens, lens_key)
        fn = lambda x_, c_, *l_: self._forward_impl(x_, c_, l_[0] if l_ else None, lens_key)   # noqa: E731
        out = self._graphs.run(("fwd", B, T, lens_key), fn, [x.contiguous().float(), c.contiguous().float()] + ([lens] if lens is not None else []))
        return out.clone()

    def _forward_impl(self, x, c, lens, lens_key):
        L = _lib.lib()
        pk = self._pack()
        B, _, T = x.shape
        frames = c.shape[-1] - 2 * self.aux_context_window
        fcond = self._uses_frame_cond()
        ws = self._workspace(B, T)
        st = _stream()
        x = x.contiguous().float()
        c = c.contiguous().float()
        lens_p = _ptr(lens) if lens is not None else None
        frame_lens = None
        if lens is not None:
            frame_lens = torch.div(lens, self.upsample_factor, rounding_mode="floor").to(torch.int32)
        _lib.check(L.pk_pwg_upsample(_ptr(c), _ptr(pk["conv_in_w"]), pk["fir_host"].ctypes.data_as(C.c_void_p),
                                     pk["scales_host"].ctypes.data_as(C.c_void_p), len(self.upsample_scales), B,
                                     self.aux_channels, frames, self.aux_context_window, _ptr(frame_lens), _ptr(ws["conv_in"]),
                                     None, _ptr(ws["c"].hi) if not fcond else None, _ptr(ws["c"].lo) if not fcond else None, st),
                   "pk_pwg_upsample")
        if lens is not None:
            ws["xb"].hi.zero_()
            ws["xb"].lo.zero_()
        src, dst = ws["xa"], ws["xb"]
        if fcond:
            if lens is not None:   # the layers skip tiles wholly past an utterance's end: their rows stay zero in both planes
                ws["xa"].hi.zero_()
                ws["xa"].lo.zero_()
            return self._forward_frame_cond(pk, ws, x, src, dst, B, T, frames, lens, frame_lens, st, lens_key)
        _lib.check(L.pk_pwg_first_conv(_ptr(x), _ptr(pk["first_w"]), _ptr(pk["first_b"]), lens_p, B, T, _ptr(ws["xa"].hi),
                                       _ptr(ws["xa"].lo), st), "pk_pwg_first_conv")
        args = PwgLayerArgs()
        args.batch, args.t, args.aux_channels = B, T, self.aux_channels
        args.lens = lens.data_ptr() if lens is not None else None
        args.c_hi, args.c_lo = ws["c"].hi.data_ptr(), ws["c"].lo.data_ptr()
        args.skip = ws["skip"].data_ptr()
        ev = getattr(self, "_layer_events", None)
        if ev is not None:   # bench.py: CUDA events around the 30 residual-layer launches, on the launching stream
            ev_a, ev_b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev_a.record()
        for i, lay in enumerate(pk["layers"]):
            args.dilation = lay["dil"]
            args.x_hi, args.x_lo, args.y_hi, args.y_lo = src.hi.data_ptr(), src.lo.data_ptr(), dst.hi.data_ptr(), dst.lo.data_ptr()
            args.w1_hi, args.w1_lo = lay["w1"].hi.data_ptr(), lay["w1"].lo.data_ptr()
            args.w2_hi, args.w2_lo = lay["w2"].hi.data_ptr(), lay["w2"].lo.data_ptr()
            args.bias1, args.bias2 = lay["b1"].ctypes.data, lay["b2"].ctypes.data
            args.skip_init = 1 if i == 0 else 0
            _lib.check(L.pk_pwg_residual_layer(C.byref(args), st), "pk_pwg_residual_layer")
            src, dst = dst, src
        if ev is not None:
            ev_b.record()
            ev.append((ev_a, ev_b))
        out = torch.empty(B, 1, T, dtype=torch.float32, device=self.device)
        _lib.check(L.pk_pwg_tail(_ptr(ws["skip"]), _ptr(pk["skip_bias_sum"]), _ptr(pk["tail_w1"]), _ptr(pk["tail_b1"]), _ptr(pk["tail_w2"]),
                                 _ptr(pk["tail_b2"]), math.sqrt(1.0 / self.layers), B * T, _ptr(out), st), "pk_pwg_tail")
        if lens is not None:
            ops.mask_rows_(out.reshape(B, T, 1), lens)
        self._last_x = src  # layer-30 residual stream (tests)
        return out

    def _forward_frame_cond(self, pk, ws, x, src, dst, B, T, frames, lens, frame_lens, st, lens_key=None):
        """Residual stack with frame-rate conditioning (DESIGN.md 5, csrc/pwg_fc.cu): conv1x1_aux of all 30 layers is applied
        to conv_in(mel) at frame rate by ONE GEMM per forward (P), and each layer multiplies the band table of the (linear,
        per-channel) upsampling operator with the 16-frame window of P its tile touches - no sample-rate conditioning tensor.
        Layer 0 computes first_conv(x) itself and the last layer runs the tail into `out`, so neither x0 nor the final skip
        sum goes through memory (a one-layer stack keeps pk_pwg_tail)."""
        from . import _pwg_frame_cond as fc
        L = _lib.lib()
        hop, A, NL = self.upsample_factor, self.aux_channels, self.layers
        if "aux_all" not in pk:
            # the 30 aux weights stacked as the row operand of one GEMM per forward, P[b] = W_aux_all (30*128 x aux) . m'[b]^T,
            # and the FIRs of the upsampling stages for the band tables
            fp = {k: v.detach().float().cpu() for k, v in self._folded().items()}
            aux_all = torch.cat([fp[f"conv_layers.{i}.conv1x1_aux.weight"][:, :, 0] for i in range(NL)], dim=0)
            pk["aux_all"] = Split.from_f32(aux_all.contiguous().to(self.device).unsqueeze(0))      # (1, 30*128, aux)
            firs, off = [], 0
            for s_ in self.upsample_scales:
                firs.append(torch.from_numpy(pk["fir_host"][off:off + 2 * s_ + 1].copy()))
                off += 2 * s_ + 1
            pk["firs"] = firs
            pk["band_tables"] = {}
        m1 = ws["conv_in"]                                               # (B, frames, aux) written by pk_pwg_upsample above
        if frame_lens is not None:
            ops.mask_rows_(m1, frame_lens)                               # frames past an utterance's end contribute nothing
        m1s = Split.from_f32(m1)
        Fp = max((frames + 7) // 8 * 8, 64)
        key = ("P", B, Fp)
        P = ws.get(key)
        if P is None:
            P = ws[key] = Split.zeros((B, NL * 128, Fp), self.device)    # columns [frames, Fp) stay zero
        a_spec = dict(rows=NL * 128, cols=A, ld=A, batch_stride=0, batches=1, bmul=0, hmul=0, col0=0, colh=0)
        b_spec = dict(rows=frames, cols=A, ld=A, batch_stride=frames * A, batches=B, bmul=1, hmul=0, col0=0, colh=0)
        ops.batched_matmul_nt(pk["aux_all"], m1s, batch=B, heads=1, m=NL * 128, n=frames, k=A, a_spec=a_spec, b_spec=b_spec,
                              y_split=P, y_batch_stride=NL * 128 * Fp, y_head_stride=0, y_ld=Fp)
        # compact band table (constants of the model + the utterance lengths of this batch; a few MB, cached per length tuple)
        if lens_key is None:
            lens_key = (frames,) * B
        ent = pk["band_tables"].get(lens_key)
        if ent is None:
            if len(pk["band_tables"]) >= 16:
                pk["band_tables"].pop(next(iter(pk["band_tables"])))
                self._graphs.clear()      # a captured forward may point at the evicted table
            tab, lay, pk["band_base"] = fc.compact_band_tables(pk["firs"], self.upsample_scales, lens_key, pk.get("band_base"))
            wide = torch.zeros(tab.shape[0], 64, dtype=torch.float32)
            wide[:, :fc.KWIN] = tab.float()
            ent = pk["band_tables"][lens_key] = (Split.from_f32(wide.to(self.device)), lay)
        U, lay = ent
        args = _lib.PwgLayerFcArgs()
        args.batch, args.t, args.hop = B, T, hop
        args.lens = lens.data_ptr() if lens is not None else None
        args.u_hi, args.u_lo, args.u_rows = U.hi.data_ptr(), U.lo.data_ptr(), U.hi.shape[0]
        args.u_period, args.u_start_row, args.u_end_base = lay["period"], lay["start_row"], lay["end_base"]
        args.p_hi, args.p_lo, args.p_rows, args.p_ld, args.p_frames = P.hi.data_ptr(), P.lo.data_ptr(), NL * 128, Fp, frames
        args.skip = ws["skip"].data_ptr()
        out = torch.empty(B, 1, T, dtype=torch.float32, device=self.device)
        fh, th = pk["first_host"], pk["tail_host"]
        args.first_w, args.first_b, args.first_u, args.first_v = fh["w"].ctypes.data, fh["b"].ctypes.data, fh["u"].ctypes.data, fh["v"].ctypes.data
        args.tail_w1_hi, args.tail_w1_lo = th["w1"].hi.data_ptr(), th["w1"].lo.data_ptr()
        args.tail_b1, args.tail_w2, args.tail_b2 = th["b1"].ctypes.data, th["w2"].ctypes.data, th["b2"].ctypes.data
        args.skip_bias, args.tail_scale = th["skip_bias"].ctypes.data, math.sqrt(1.0 / NL)
        ev = getattr(self, "_layer_events", None)
        if ev is not None:   # bench.py: CUDA events around the 30 residual-layer launches, on the launching stream
            ev_a, ev_b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev_a.record()
        for i, lay_ in enumerate(pk["layers"]):
            first, last = i == 0, i == NL - 1 and i > 0
            args.dilation, args.p_row0 = lay_["dil"], i * 128
            args.noise = x.data_ptr() if first else None
            args.out = out.data_ptr() if last else None
            args.x_hi, args.x_lo = (None, None) if first else (src.hi.data_ptr(), src.lo.data_ptr())
            args.y_hi, args.y_lo = dst.hi.data_ptr(), dst.lo.data_ptr()
            args.w1_hi, args.w1_lo = lay_["w1"].hi.data_ptr(), lay_["w1"].lo.data_ptr()
            args.w2_hi, args.w2_lo = lay_["w2"].hi.data_ptr(), lay_["w2"].lo.data_ptr()
            args.bias1, args.bias2 = lay_["b1"].ctypes.data, lay_["b2"].ctypes.data
            args.skip_init = 1 if first else 0
            _lib.check(L.pk_pwg_residual_layer_fc(C.byref(args), st), "pk_pwg_residual_layer_fc")
            src, dst = dst, src
        if ev is not None:
            ev_b.record()
            ev.append((ev_a, ev_b))
        if NL == 1:
            _lib.check(L.pk_pwg_tail(_ptr(ws["skip"]), _ptr(pk["skip_bias_sum"]), _ptr(pk["tail_w1"]), _ptr(pk["tail_b1"]),
                                     _ptr(pk["tail_w2"]), _ptr(pk["tail_b2"]), 1.0, B * T, _ptr(out), st), "pk_pwg_tail")
        if lens is not None:
            ops.mask_rows_(out.reshape(B, T, 1), lens)       # samples past an utterance's end: zero, not tail(bias)
        self._last_x = src
        return out

    def upsample(self, c):
        """ConvInUpsampleNet.forward (:201-216) alone: (B, aux, T'+2w) -> (B, aux, T) fp32 (used by the tests)."""
        _declare()
        pk = self._pack()
        B = c.shape[0]
        frames = c.shape[-1] - 2 * self.aux_context_window
        out = torch.empty(B, self.aux_channels, frames * self.upsample_factor, dtype=torch.float32, device=self.device)
        c = c.contiguous().float()
        cin = torch.empty(B, frames, self.aux_channels, dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib().pk_pwg_upsample(_ptr(c), _ptr(pk["conv_in_w"]),
                                              pk["fir_host"].ctypes.data_as(C.c_void_p),
                                              pk["scales_host"].ctypes.data_as(C.c_void_p), len(self.upsample_scales), B,
                                              self.aux_channels, frames, self.aux_context_window, None, _ptr(cin), _ptr(out),
                                              None, None, _stream()), "pk_pwg_upsample")
        return out

    def inference(self, c=None, x=None):
        """Single-utterance generation (reference :498-520): c (T', aux) -> (T, out_channels).
        The noise is drawn with torch.randn unless `x` (1, 1, T) is supplied (parity tests supply it)."""
        T = c.shape[0] * self.upsample_factor
        if x is None:
            x = torch.randn(1, self.in_channels, T, device=self.device)
        c = c.transpose(0, 1).unsqueeze(0)
        w = self.aux_context_window
        c = torch.cat([c[:, :, :1].expand(-1, -1, w), c, c[:, :, -1:].expand(-1, -1, w)], dim=-1)  # Pad1D 'replicate'
        return self.forward(x, c).squeeze(0).transpose(0, 1)


class PWGDiscriminator(Layer):
    """Convolutional discriminator of Parallel WaveGAN (reference parallel_wavegan.py:523-627): layers - 1 x [Conv1D(k, dilation
    d_i, 'same' zero padding) + LeakyReLU] + Conv1D(k), weight norm on every conv.  Same constructor keywords and state-dict keys
    (`conv_layers.{2 i}.{weight_g, weight_v, bias}`: the Sequential alternates convs and activations).  `forward` and the
    training step (training/pwg_step.py) run every conv through pk_conv_gemm."""

    def __init__(self, in_channels: int = 1, out_channels: int = 1, kernel_size: int = 3, layers: int = 10, conv_channels: int = 64,
                 dilation_factor: int = 1, nonlinear_activation: str = "LeakyReLU",
                 nonlinear_activation_params: Dict[str, Any] = {"negative_slope": 0.2}, bias: bool = True, use_weight_norm: bool = True,
                 device=None, seed: int = 0):
        super().__init__(device)
        assert kernel_size % 2 == 1 and dilation_factor > 0
        if nonlinear_activation != "LeakyReLU" or in_channels != 1 or out_channels != 1:
            raise NotImplementedError("LeakyReLU, 1 input / output channel (the shipped configs)")
        self.layers, self.kernel_size, self.conv_channels = layers, kernel_size, conv_channels
        self.slope = float(nonlinear_activation_params.get("negative_slope", 0.01))
        self.dilations = [1 if i == 0 else (i if dilation_factor == 1 else dilation_factor ** i) for i in range(layers - 1)] + [1]
        self._weight_norm = False
        g = torch.Generator().manual_seed(seed)
        cin = in_channels
        for i in range(layers):
            cout = out_channels if i == layers - 1 else conv_channels
            bound = 1.0 / math.sqrt(cin * kernel_size)
            self._register(f"conv_layers.{2 * i}.weight", (torch.rand(cout, cin, kernel_size, generator=g) * 2 - 1) * bound)
            if bias:
                self._register(f"conv_layers.{2 * i}.bias", (torch.rand(cout, generator=g) * 2 - 1) * bound)
            cin = conv_channels
        if use_weight_norm:
            self.apply_weight_norm()

    apply_weight_norm = PWGGenerator.apply_weight_norm
    remove_weight_norm = PWGGenerator.remove_weight_norm
    _folded = PWGGenerator._folded

    def forward(self, x):
        """(N, 1, T) audio -> (N, 1, T) logits."""
        if not x.is_cuda:
            raise _lib.PkError("PWGDiscriminator.forward needs CUDA tensors (no CPU fallback)")
        w = {k: v.float() for k, v in self._folded().items()}
        B, _, T = x.shape
        x8 = torch.zeros(B, T, 8, dtype=torch.float32, device=x.device)
        x8[:, :, 0] = x[:, 0]
        h = Split.from_f32(x8)
        L = _lib.lib()
        for i in range(self.layers):
            name = f"conv_layers.{2 * i}"
            wt = w[name + ".weight"]
            cout, cin, k = wt.shape
            cin_p = h.hi.shape[-1]
            wp = torch.zeros(cout, cin_p, k, dtype=torch.float32, device=x.device)
            wp[:, :cin] = wt
            y, _ = ops.conv_gemm(h, ops.pack_weight(wp, x.device), n=cout, k=cin_p, taps=k, dil=self.dilations[i], bias=w.get(name + ".bias"))
            if i < self.layers - 1:
                a = Split.empty(tuple(y.shape), y.device)
                _lib.check(L.pk_leaky_relu(_ptr(y), y.numel(), self.slope, None, _ptr(a.hi), _ptr(a.lo), _stream()), "pk_leaky_relu")
                h = a
        return y.transpose(1, 2).contiguous()


class PWGInference(Layer):
    """reference parallel_wavegan.py:766-775."""

    def __init__(self, normalizer, pwg_generator):
        super().__init__(pwg_generator.device)
        self.normalizer = normalizer
        self.pwg_generator = pwg_generator

    def forward(self, logmel, x=None):
        normalized_mel = self.normalizer(logmel)
        return self.pwg_generator.inference(normalized_mel, x=x)
