"""WaveFlow training step on H100 (reference: examples/waveflow/train.py:95-118 `Experiment.train_batch`):
`z, log_det = model(wav, mel)`, `loss = WaveFlowLoss(sigma)(z, log_det)`, `loss.backward()`, `paddle.optimizer.Adam(lr)`.

The step runs its own forward: it keeps what the backward needs (each layer's input planes and pre-gate `a|g`, each flow's
skip sum, input and condition rows) and reads its weights from device buffers that weight norm and one packing gather rebuild
on the device at the start of every step, so forward + backward replay as one CUDA graph while the weights change.  The
backward of the residual net is one `pk_waveflow_backward_layer` launch per layer boundary (3x3 data gradient + residual
gradient, out_proj^T with dx as the register operand, gate backward); the forward's convs are `pk_conv_gemm` (the 3x3 conv as
three launches, one per kernel row, over the "net layout" of csrc/waveflow_train.cu); the weight gradients are split-K NT
matmuls (`wgrad.nt_splitk`) over transposed planes, the conv bias gradient riding along as a ones row.  Parameters,
gradients and Adam moments live in flat buffers (`training/flat.py: FlatAdam`); the model's tensors are views of the parameter buffer.
torch only allocates, views, copies and all-reduces.
"""
import ctypes as C_

import numpy as np
import torch

from .. import _lib, ops
from ..ops import Split, _ptr, _stream, ceil_to
from . import wgrad
from .flat import PdCheckpoint, TrainStep, need_cuda

SLOPE = 0.4            # UpsampleNet's leaky_relu (waveflow.py:130)
_SCRATCH = 1024 * 256  # fp32 partials of pk_waveflow_train_outer_sum / pk_waveflow_upsample_bwd


class WaveFlowTrainStep(PdCheckpoint, TrainStep):
    def __init__(self, model, learning_rate=2e-4, sigma=1.0, beta1=0.9, beta2=0.999, epsilon=1e-8, process_group=None):
        if not model._eligible():
            raise NotImplementedError("the WaveFlow training step needs 64 or 128 channels, 64 < n_mels <= 128 (a multiple of 8) "
                                      "and 2 to 8 layers per flow")
        need_cuda(model)
        if not sigma > 0:
            raise ValueError("sigma must be positive")
        self.sigma = float(sigma)
        # a captured graph pins its own memory pool: ~20 GB at the recipe's batch and 128 channels, so only a few shapes are kept
        super().__init__(model, learning_rate, process_group, max_graphs=2, beta1=beta1, beta2=beta2, epsilon=epsilon)
        dev, names = self.dev, self.buffers.names
        self.off = dict(zip(names, self.buffers.offsets))
        self.weff = torch.zeros_like(self.flat)     # weights as the forward uses them: weight norm folded into the weight_v slots
        self.dweff = torch.zeros_like(self.flat)    # gradients with respect to weff
        self._wn = []                                # (v offset, g offset, rows, inner) of every weight-normed tensor
        for k in names:
            if k.endswith(".weight_v"):
                v = model._params[k]
                self._wn.append((self.off[k], self.off[k[:-1] + "g"], v.shape[0], v.numel() // v.shape[0]))
        G = model.n_group
        self.perms, cmaps, cm = model.perms, [], list(range(G))
        for pm in self.perms:
            cmaps.append(cm)
            cm = [cm[j] for j in pm]
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)
        self.cmaps = [i32(c) for c in cmaps]                                   # condition height of each height, per flow
        self.inv_perms = [i32(np.argsort(pm).tolist()) for pm in self.perms]
        self._build_packs()
        self._lens = {}

    # ------------------------------------------------------------------------------------------------------------
    # weights: offsets into the flat buffers and the packed GEMM operands
    # ------------------------------------------------------------------------------------------------------------
    def _w(self, name):
        """offset of the (folded) weight `name` in weff / dweff."""
        return self.off[name + ".weight_v"] if name + ".weight_v" in self.off else self.off[name + ".weight"]

    def _idx(self, name, shape):
        return torch.arange(int(np.prod(shape)), dtype=torch.int64).view(shape) + self._w(name)

    def _build_packs(self):
        """Index maps from weff to every packed operand (K-major [N][taps * Kp], split-bf16), gathered by ONE launch per step."""
        m = self.m
        C, M, NL = m.channels, m.n_mels, m.n_layers
        segs, self._packs = [], []
        total = 0

        def add(ix):
            nonlocal total
            ix = ix.reshape(ix.shape[0], -1)
            segs.append((total, ix))
            o = total
            total += ceil_to(ix.numel(), 64)
            return (o, tuple(ix.shape))

        for fl in range(m.n_flows):
            layers = []
            for l in range(NL):
                q = f"decoder.{fl}.resnet.{l}."
                w1 = self._idx(q + "conv", (2 * C, C, 3, 3))
                wc = self._idx(q + "condition_proj", (2 * C, M))
                w2 = self._idx(q + "out_proj", (2 * C, C))
                wcp = torch.full((2 * C, ceil_to(M, 64)), -1, dtype=torch.int64)
                wcp[:, :M] = wc
                layers.append(dict(
                    w1f=[add(w1[:, :, kh, :].permute(0, 2, 1)) for kh in range(3)],             # (o, kw, c): output row q reads input row q + kh
                    wcf=add(wcp), w2f=add(w2), w2b=add(w2.t()),
                    # (c, (s, tap, o)): conv^T of pk_waveflow_backward_layer, kernel row s reads dh row q + s
                    w1b=add(torch.cat([w1[:, :, 2 - s, :].flip(-1).permute(1, 2, 0).reshape(C, 6 * C) for s in range(3)], dim=1))))
            wcb = torch.cat([self._idx(f"decoder.{fl}.resnet.{l}.condition_proj", (2 * C, M)) for l in range(NL)]).t()
            self._packs.append(dict(layers=layers, wcb=add(wcb)))
        idx = torch.full((total,), -1, dtype=torch.int64)
        for o, ix in segs:
            idx[o:o + ix.numel()] = ix.reshape(-1)
        self._pack_idx = idx.to(torch.int32).to(self.dev)
        self._packed = Split.empty((total,), self.dev)

    def _op(self, ent):
        o, shape = ent
        n = shape[0] * shape[1]
        return Split(self._packed.hi[o:o + n].view(shape), self._packed.lo[o:o + n].view(shape))

    def _v(self, buf, key, n):
        o = self.off[key]
        return buf[o:o + n]

    @staticmethod
    def _p(buf, off):
        return C_.c_void_p(buf.data_ptr() + 4 * off)

    # ------------------------------------------------------------------------------------------------------------
    # forward + backward
    # ------------------------------------------------------------------------------------------------------------
    def _forward_backward(self, audio, mel):
        """audio (B, T) fp32, mel (B, n_mels, T') fp32: loss (1,) on the device; the gradient of every parameter in self.gflat
        (written whole, so there is no prologue)."""
        m, L, st, dev = self.m, _lib.lib(), _stream(), self.dev
        G, C, NL, NF, M = m.n_group, m.channels, m.n_layers, m.n_flows, m.n_mels
        lens = self._net_lens(audio.shape[0], audio.shape[-1] // G)
        chk, p = _lib.check, self._p
        weff, dweff = self.weff, self.dweff
        # weights of this step: weight norm folded (weff), packed operands gathered from it
        weff.copy_(self.flat)
        for vo, go, rows, inner in self._wn:
            chk(L.pk_weight_norm_fwd(p(self.flat, vo), p(self.flat, go), rows, inner, p(weff, vo), None, st), "pk_weight_norm_fwd")
        chk(L.pk_waveflow_train_gather_split(_ptr(weff), _ptr(self._pack_idx), self._pack_idx.numel(), _ptr(self._packed.hi),
                                             _ptr(self._packed.lo), st), "pk_waveflow_train_gather_split")
        # encoder (UpsampleNet without the trim)
        B = audio.shape[0]
        enc = [mel]
        for i, f in enumerate(m.upsample_factors):
            x = enc[-1]
            y = torch.empty(B, M, x.shape[-1] * f, device=dev)
            chk(L.pk_waveflow_upsample(_ptr(x), p(weff, self._w(f"encoder.{i}")), p(weff, self.off[f"encoder.{i}.bias"]), B, M, x.shape[-1], f,
                                       0, SLOPE, _ptr(y), st), "pk_waveflow_upsample")
            enc.append(y)
        cond = enc[-1]
        t_cond = cond.shape[-1]
        W = audio.shape[-1] // G
        Q = B * (G + 1)
        PQ = Q * W
        xs = [audio[:, :W * G].reshape(B, W, G).transpose(1, 2).contiguous()]
        logs = torch.empty(NF, B * (G - 1) * W, device=dev)
        saved = []
        for fl in range(NF):
            pre = f"decoder.{fl}."
            cond_f = Split.empty((Q, W, M), dev)
            chk(L.pk_waveflow_train_cond_gather(_ptr(cond), _ptr(self.cmaps[fl]), B, G, W, M, t_cond, _ptr(cond_f.hi), _ptr(cond_f.lo), st),
                "pk_waveflow_train_cond_gather")
            h32 = torch.empty(Q, W, C, device=dev)
            skip = torch.empty(Q, W, C, device=dev)
            xin = [Split.zeros((Q + 2, W, C), dev) for _ in range(NL)]
            chk(L.pk_waveflow_train_input_fwd(_ptr(xs[fl]), p(weff, self._w(pre + "input_proj")), p(weff, self.off[pre + "input_proj.bias"]), B, G,
                                              W, C, _ptr(h32), _ptr(xin[0].hi), _ptr(xin[0].lo), st), "pk_waveflow_train_input_fwd")
            hs = []
            for l in range(NL):
                q = f"{pre}resnet.{l}."
                pk = self._packs[fl]["layers"][l]
                h = torch.empty(Q, W, 2 * C, device=dev)
                ops.conv_gemm(cond_f, self._op(pk["wcf"]), n=2 * C, k=M, bias=self._v(weff, q + "condition_proj.bias", 2 * C), lens=lens, y_f32=h)
                for kh in range(3):
                    xv = Split(xin[l].hi[kh:kh + Q], xin[l].lo[kh:kh + Q])
                    ops.conv_gemm(xv, self._op(pk["w1f"][kh]), n=2 * C, k=C, taps=3, dil=2 ** l,
                                  bias=self._v(weff, q + "conv.bias", 2 * C) if kh == 0 else None, residual=h, lens=lens, y_f32=h)
                z = Split.empty((Q, W, C), dev)
                chk(L.pk_gate_fwd(_ptr(h), PQ, C, None, _ptr(z.hi), _ptr(z.lo), st), "pk_gate_fwd")
                out = ops.conv_gemm(z, self._op(pk["w2f"]), n=2 * C, k=C, bias=self._v(weff, q + "out_proj.bias", 2 * C), lens=lens)[0]
                nxt = xin[l + 1] if l + 1 < NL else None
                chk(L.pk_waveflow_train_update(_ptr(out), B, G, W, C, _ptr(h32), _ptr(skip), 1 if l == 0 else 0, _ptr(nxt.hi if nxt else None),
                                               _ptr(nxt.lo if nxt else None), st), "pk_waveflow_train_update")
                hs.append(h)
            xs.append(torch.empty(B, G, W, device=dev))
            chk(L.pk_waveflow_train_tail_fwd(_ptr(skip), p(weff, self.off[pre + "output_proj.weight"]), p(weff, self.off[pre + "output_proj.bias"]),
                                             _ptr(xs[fl]), _ptr(self.inv_perms[fl]), B, G, W, C, _ptr(xs[fl + 1]), _ptr(logs[fl]), st),
                "pk_waveflow_train_tail_fwd")
            saved.append((cond_f, xin, hs, skip))
        loss = torch.empty(1, device=dev)
        n_z = B * G * W
        chk(L.pk_waveflow_train_loss(_ptr(xs[NF]), n_z, _ptr(logs), logs.numel(), self.sigma, _ptr(loss), st), "pk_waveflow_train_loss")

        # ---------------------------------------------------------------- backward
        dweff.zero_()
        scratch = torch.empty(_SCRATCH, device=dev)

        def reduce_rows(a, lda, ka, out_off, b=None, ldb=1, kb=1, os_i=1, os_j=0):
            """dweff[out_off + i * os_i + j * os_j] = sum over the PQ positions of a[:, i] * (b[:, j] or 1), in a fixed order."""
            chk(L.pk_waveflow_train_outer_sum(_ptr(a), lda, ka, _ptr(b), ldb, kb, PQ, _ptr(scratch), _SCRATCH, p(dweff, out_off), os_i, os_j, 0, st),
                "pk_waveflow_train_outer_sum")

        _, S, ks, kkp = wgrad.plan(1, PQ, 2 * C, 9 * C)
        tr = ops.transpose_planes
        dcond = torch.zeros(B, M, t_cond, device=dev)
        dnext = None
        for fl in reversed(range(NF)):
            pre = f"decoder.{fl}."
            cond_f, xin, hs, skip = saved[fl]
            a2 = Split.zeros((Q, W, 2 * C), dev)                  # GEMM2's A operand [dx | dskip]
            dskip = torch.zeros(Q, W, C, device=dev)
            dparams = torch.zeros(Q, W, 2, device=dev)
            dxin = torch.empty(B, G, W, device=dev)
            last = fl == NF - 1
            chk(L.pk_waveflow_forward_tail_bwd(_ptr(skip), p(weff, self.off[pre + "output_proj.weight"]), p(weff, self.off[pre + "output_proj.bias"]),
                                               _ptr(xs[fl]), _ptr(self.inv_perms[fl]), _ptr(dnext), _ptr(xs[NF] if last else None),
                                               1.0 / (self.sigma ** 2 * n_z), -1.0 / n_z, B, G, W, C, _ptr(dxin), _ptr(dparams), _ptr(dskip),
                                               _ptr(a2.hi), _ptr(a2.lo), 2 * C, C, st), "pk_waveflow_forward_tail_bwd")
            reduce_rows(dparams, 2, 2, self.off[pre + "output_proj.weight"], b=skip, ldb=C, kb=C, os_i=C, os_j=1)
            reduce_rows(dparams, 2, 2, self.off[pre + "output_proj.bias"])
            dX = torch.zeros(Q, W, C, device=dev)               # gradient of the residual stream h (pad rows stay zero)
            dh_all = Split.zeros((Q + 2, W, NL * 2 * C), dev)   # every layer's d(a|g), the condition GEMM's A operand
            dhT = Split.zeros((NL * 2 * C, kkp), dev)
            x9T = Split.zeros((9 * C + 8, kkp), dev)            # the nine shifted input planes + a ones row (the bias gradient)
            x9T.hi[9 * C, :PQ].fill_(1.0)
            doutT = Split.zeros((2 * C, kkp), dev)
            zT = Split.zeros((C, kkp), dev)
            z = Split.empty((Q, W, C), dev)
            for l in range(NL, -1, -1):
                # layer boundary l: dX <- gradient of layer l's input, and layer l - 1's d(a|g) into dh_all
                a = _lib.WaveflowBackwardLayerArgs()
                a.batch, a.width, a.channels, a.n_group, a.dh_ld = B, W, C, G, NL * 2 * C
                a.dx, a.a2_hi, a.a2_lo = dX.data_ptr(), a2.hi.data_ptr(), a2.lo.data_ptr()
                if l < NL:
                    w1 = self._op(self._packs[fl]["layers"][l]["w1b"])
                    a.has_gemm1, a.dilation = 1, 2 ** l
                    a.dh_in_hi, a.dh_in_lo = dh_all.hi[:, :, l * 2 * C:].data_ptr(), dh_all.lo[:, :, l * 2 * C:].data_ptr()
                    a.w1_hi, a.w1_lo = w1.hi.data_ptr(), w1.lo.data_ptr()
                if l >= 1:
                    w2 = self._op(self._packs[fl]["layers"][l - 1]["w2b"])
                    a.has_gemm2 = 1
                    a.w2_hi, a.w2_lo, a.h = w2.hi.data_ptr(), w2.lo.data_ptr(), hs[l - 1].data_ptr()
                    a.dh_out_hi, a.dh_out_lo = dh_all.hi[:, :, (l - 1) * 2 * C:].data_ptr(), dh_all.lo[:, :, (l - 1) * 2 * C:].data_ptr()
                chk(L.pk_waveflow_backward_layer(C_.byref(a), st), "pk_waveflow_backward_layer")
                if l == 0:
                    break
                lp = l - 1                                       # weight gradients of layer l - 1: dres = dX, d(a|g) = dh_all block
                q = f"{pre}resnet.{lp}."
                d = 2 ** lp
                chk(L.pk_gate_fwd(_ptr(hs[lp]), PQ, C, None, _ptr(z.hi), _ptr(z.lo), st), "pk_gate_fwd")
                tr(a2, z=1, rows=PQ, src_zstride=0, ld_src=2 * C, c0=0, cols=2 * C, shift=0, r_out=PQ, dst=doutT, dst_zstride=0, ld_dst=kkp)
                tr(z, z=1, rows=PQ, src_zstride=0, ld_src=C, c0=0, cols=C, shift=0, r_out=PQ, dst=zT, dst_zstride=0, ld_dst=kkp)
                o2 = self._w(q + "out_proj")
                wgrad.nt_splitk(doutT, zT, 2 * C, C, S, ks, kkp, out=dweff[o2:o2 + 2 * C * C].view(2 * C, C))
                reduce_rows(dX, C, C, self.off[q + "out_proj.bias"])
                reduce_rows(dskip, C, C, self.off[q + "out_proj.bias"] + C)
                cs = slice(lp * 2 * C, (lp + 1) * 2 * C)
                dh_l = Split(dhT.hi[cs], dhT.lo[cs])
                tr(dh_all, z=1, rows=PQ, src_zstride=0, ld_src=NL * 2 * C, c0=lp * 2 * C, cols=2 * C, shift=0, r_out=PQ, dst=dh_l, dst_zstride=0,
                   ld_dst=kkp)
                for kh in range(3):
                    src = Split(xin[lp].hi[kh:kh + Q], xin[lp].lo[kh:kh + Q])
                    for kw in range(3):
                        o = (kh * 3 + kw) * kkp
                        dst = Split(x9T.hi.view(-1)[o:], x9T.lo.view(-1)[o:])
                        tr(src, z=Q, rows=W, src_zstride=W * C, ld_src=C, c0=0, cols=C, shift=(kw - 1) * d, r_out=W, dst=dst, dst_zstride=W,
                           ld_dst=9 * kkp)
                dw1 = wgrad.nt_splitk(dh_l, x9T, 2 * C, 9 * C + 8, S, ks, kkp)
                o1 = self._w(q + "conv")
                dweff[o1:o1 + 18 * C * C].view(2 * C, 9 * C).copy_(dw1[:, :9 * C])
                self._v(dweff, q + "conv.bias", 2 * C).copy_(dw1[:, 9 * C])
                self._v(dweff, q + "condition_proj.bias", 2 * C).copy_(dw1[:, 9 * C])
            # input_proj
            xcol = torch.zeros(Q, W, device=dev)
            chk(L.pk_waveflow_train_input_bwd(_ptr(dX), _ptr(xs[fl]), p(weff, self._w(pre + "input_proj")), B, G, W, C, _ptr(dxin), _ptr(xcol), st),
                "pk_waveflow_train_input_bwd")
            reduce_rows(dX, C, C, self._w(pre + "input_proj"), b=xcol)
            reduce_rows(dX, C, C, self.off[pre + "input_proj.bias"])
            # condition_proj of all layers: weight gradients and the condition gradient, one GEMM each
            condT = Split.zeros((M, kkp), dev)
            tr(cond_f, z=1, rows=PQ, src_zstride=0, ld_src=M, c0=0, cols=M, shift=0, r_out=PQ, dst=condT, dst_zstride=0, ld_dst=kkp)
            dwc = wgrad.nt_splitk(dhT, condT, NL * 2 * C, M, S, ks, kkp)
            for l in range(NL):
                oc = self._w(f"{pre}resnet.{l}.condition_proj")
                dweff[oc:oc + 2 * C * M].view(2 * C, M).copy_(dwc[l * 2 * C:(l + 1) * 2 * C])
            dc = ops.conv_gemm(Split(dh_all.hi[:Q], dh_all.lo[:Q]), self._op(self._packs[fl]["wcb"]), n=M, k=NL * 2 * C, lens=lens)[0]
            chk(L.pk_waveflow_train_cond_scatter(_ptr(dc), _ptr(self.cmaps[fl]), B, G, W, M, t_cond, _ptr(dcond), st), "pk_waveflow_train_cond_scatter")
            dnext = dxin
        # encoder
        dy = dcond
        for i in reversed(range(len(m.upsample_factors))):
            f = m.upsample_factors[i]
            x, y = enc[i], enc[i + 1]
            dpre = torch.empty_like(y)
            dx = torch.empty_like(x) if i > 0 else None
            chk(L.pk_waveflow_upsample_bwd(_ptr(x), _ptr(y), _ptr(dy), p(weff, self._w(f"encoder.{i}")), B, M, x.shape[-1], f, SLOPE, _ptr(dpre),
                                           _ptr(dx), _ptr(scratch), _SCRATCH, p(dweff, self._w(f"encoder.{i}")),
                                           p(dweff, self.off[f"encoder.{i}.bias"]), st), "pk_waveflow_upsample_bwd")
            dy = dx
        # back through weight norm to (g, v)
        self.gflat.copy_(dweff)
        for vo, go, rows, inner in self._wn:
            chk(L.pk_weight_norm_bwd(p(self.flat, vo), p(self.flat, go), p(dweff, vo), rows, inner, p(self.gflat, go), p(self.gflat, vo), st),
                "pk_weight_norm_bwd")
        return loss

    def _net_lens(self, B, W):
        """int32 (B * (n_group + 1),): W on net rows, 0 on the two pad rows of each utterance (pk_conv_gemm skips and zeroes them)."""
        key = (B, W)
        if key not in self._lens:
            G = self.m.n_group
            v = ([W] * (G - 1) + [0, 0]) * B
            self._lens[key] = torch.tensor(v, dtype=torch.int32, device=self.dev)
        return self._lens[key]

    def forward_backward_graphed(self, audio, mel):
        """Forward + backward of audio (B, T) and mel (B, n_mels, T') through the CUDA graph of their shape, without an update:
        the loss, the graph's own tensor (valid until its next replay)."""
        return self._run((mel, audio), graph=True)

    def _prepare(self, batch):
        """batch = (mel, wav) as the reference's collate yields it."""
        mel, audio = batch
        if not (audio.is_cuda and mel.is_cuda):
            raise _lib.PkError("WaveFlowTrainStep needs CUDA tensors (no CPU fallback)")
        m = self.m
        if mel.dim() != 3 or mel.shape[1] != m.n_mels or audio.dim() != 2 or audio.shape[0] != mel.shape[0]:
            raise ValueError(f"expected wav (B, T) and mel (B, {m.n_mels}, T'), got {tuple(audio.shape)} and {tuple(mel.shape)}")
        t_cond = mel.shape[-1]
        for f in m.upsample_factors:
            t_cond *= f
        m._check_forward(audio.shape[-1], t_cond)
        if audio.shape[-1] < m.n_group:
            raise ValueError(f"audio shorter than n_group ({m.n_group}) samples")
        return [audio.contiguous().float(), mel.contiguous().float()], (audio.shape[0], audio.shape[-1], mel.shape[-1])
