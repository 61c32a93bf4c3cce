"""ConditionalWaveFlow inference and density estimation on H100 - host side (reference parakeet/models/waveflow.py:714-909).

Same constructor as the reference (`upsample_factors, n_flows, n_layers, n_group, channels, n_mels, kernel_size`), same
state-dict keys (`encoder.{i}.{weight_g,weight_v,bias}`, `decoder.{f}.input_proj.*`,
`decoder.{f}.resnet.{l}.{conv,condition_proj,out_proj}.*`, `decoder.{f}.output_proj.{weight,bias}`), `infer(mel)` and
`predict(mel)`, `forward(audio, mel)` and WaveFlowLoss.  All arithmetic is in libparakeet_b200.so; fold / permute / row
slicing are torch views and gathers.

Accepted configs: kernel_size (3, 3), n_group 8 or 16 (height dilation 1 -> a 3-row causal buffer), even n_flows, 64 or 128
residual channels and n_mels a multiple of 8; this covers the shipped config (examples/waveflow/config.py).  Within that range
the fused kernels run every config with 64 < n_mels <= 128 and 2 to 8 layers per flow (`_eligible`); `inverse` runs every
other accepted config on the two-GEMM row loop.  The density direction (`forward`: audio -> z, log-det, the held-out negative
log-likelihood with WaveFlowLoss) and its training step (parakeet_b200.training.WaveFlowTrainStep) need the fused kernels.
"""
import ctypes as C_

import numpy as np
import torch

from .. import _lib, ops
from ..layer import Layer
from ..ops import Split, _ptr, _stream


def _planes(m, dev):
    """fp32 matrix -> split-bf16 planes (2, rows, cols) in ONE allocation (the 4-D TMA maps of the fused kernels need it)."""
    m = m.detach().float().cpu()
    hi = m.to(torch.bfloat16)
    lo = (m - hi.float()).to(torch.bfloat16)
    return torch.stack([hi, lo]).contiguous().to(dev)


def _fold_wn(params):
    out = {}
    for k, v in params.items():
        if k.endswith("weight_g"):
            continue
        if k.endswith("weight_v"):
            g = params[k[:-1] + "g"]
            norm = v.reshape(v.shape[0], -1).norm(dim=1)
            out[k[:-2]] = v * (g / norm).reshape([-1] + [1] * (v.dim() - 1))
        else:
            out[k] = v
    return out


class ConditionalWaveFlow(Layer):
    def __init__(self, upsample_factors, n_flows, n_layers, n_group, channels, n_mels, kernel_size=(3, 3), device=None, seed=0):
        super().__init__(device)
        if isinstance(kernel_size, int):
            kernel_size = (kernel_size, kernel_size)
        if tuple(kernel_size) != (3, 3) or n_group not in (8, 16):
            raise NotImplementedError("this round supports kernel_size (3,3) and n_group 8 / 16 (height dilation 1)")
        if n_group % 2 or n_flows % 2:
            raise ValueError("number of flows and number of group must be even")
        if channels not in (64, 128):
            # the two-GEMM row loop's gate and update epilogues hold at most 2C = 256 output channels
            raise NotImplementedError(f"channels must be 64 or 128 (got {channels})")
        if n_mels % 8:
            # condition rows are GEMM / TMA operands whose row stride (n_mels bf16 elements) must be a multiple of 16 bytes
            raise NotImplementedError(f"n_mels must be a multiple of 8 (got {n_mels})")
        self.upsample_factors = list(upsample_factors)
        self.n_flows, self.n_layers, self.n_group, self.channels, self.n_mels = n_flows, n_layers, n_group, channels, n_mels
        g = torch.Generator().manual_seed(seed)

        def u(*shape, std):
            return (torch.rand(*shape, generator=g) * 2 - 1) * std

        def wn(name, w):
            self._register(name + ".weight_g", w.reshape(w.shape[0], -1).norm(dim=1))
            self._register(name + ".weight_v", w)

        import math
        for i, f in enumerate(self.upsample_factors):
            std = math.sqrt(1 / (3 * 2 * f))
            wn(f"encoder.{i}", u(1, 1, 3, 2 * f, std=std))
            self._register(f"encoder.{i}.bias", u(1, std=std))
        C = channels
        for fl in range(n_flows):
            pre = f"decoder.{fl}."
            wn(pre + "input_proj", u(C, 1, 1, 1, std=1.0))
            self._register(pre + "input_proj.bias", u(C, std=1.0))
            for l in range(n_layers):
                q = f"{pre}resnet.{l}."
                std = math.sqrt(1 / (C * 9))
                wn(q + "conv", u(2 * C, C, 3, 3, std=std))
                self._register(q + "conv.bias", u(2 * C, std=std))
                std = math.sqrt(1 / n_mels)
                wn(q + "condition_proj", u(2 * C, n_mels, 1, 1, std=std))
                self._register(q + "condition_proj.bias", u(2 * C, std=std))
                std = math.sqrt(1 / C)
                wn(q + "out_proj", u(2 * C, C, 1, 1, std=std))
                self._register(q + "out_proj.bias", u(2 * C, std=std))
            self._register(pre + "output_proj.weight", torch.zeros(2, C, 1, 1))   # reference: Constant(0.)
            self._register(pre + "output_proj.bias", torch.zeros(2))
        idx = list(range(n_group))
        half = n_group // 2
        self.perms = [idx[::-1] if i < n_flows // 2 else list(reversed(idx[:half])) + list(reversed(idx[half:]))
                      for i in range(n_flows)]                                       # waveflow.py:602-615

    def _pack(self):
        if self._packed is not None:
            return self._packed
        p = {k: v.detach().float().cpu() for k, v in _fold_wn(self._params).items()}
        dev, C = self.device, self.channels
        pk = {"enc": [(p[f"encoder.{i}.weight"].reshape(3, -1).contiguous().to(dev), p[f"encoder.{i}.bias"].to(dev))
                      for i in range(len(self.upsample_factors))], "flows": []}
        fused = self._eligible()
        for fl in range(self.n_flows):
            pre = f"decoder.{fl}."
            layers = []
            for l in range(self.n_layers):
                q = f"{pre}resnet.{l}."
                w = p[q + "conv.weight"]                                  # [2C, C, kh, kw]
                if fused:
                    # operands of pk_waveflow_flow / pk_waveflow_forward_layer (include/parakeet_b200.h): channels in blocks of 64;
                    # gate rows a_blk | g_blk per block, out_proj rows skip_blk | res_blk; GEMM1 columns [tap][slot][c] | condition_proj
                    nb = C // 64
                    g_rows = torch.cat([torch.cat([torch.arange(64 * k, 64 * k + 64), torch.arange(C + 64 * k, C + 64 * k + 64)])
                                        for k in range(nb)])
                    o_rows = torch.cat([torch.cat([torch.arange(C + 64 * k, C + 64 * k + 64), torch.arange(64 * k, 64 * k + 64)])
                                        for k in range(nb)])
                    cw = p[q + "condition_proj.weight"][:, :, 0, 0]
                    w1 = []
                    for v in range(3):
                        m = torch.zeros(2 * C, 9 * C + 128)
                        for tap in range(3):
                            for s in range(3):
                                m[:, (3 * tap + s) * C:(3 * tap + s + 1) * C] = w[:, :, (s - v) % 3, tap]
                        m[:, 9 * C:9 * C + self.n_mels] = cw
                        w1.append(_planes(m[g_rows], dev))
                    ow, ob = p[q + "out_proj.weight"][:, :, 0, 0], p[q + "out_proj.bias"]
                    b1 = (p[q + "conv.bias"] + p[q + "condition_proj.bias"])[g_rows].numpy().astype("float32").copy()
                    layers.append(dict(fused=dict(w1=w1, w2=_planes(ow[o_rows], dev), b1=b1, b2=ob[o_rows].numpy().astype("float32").copy())))
                else:
                    # operands of the two-GEMM row loop (pk_conv_gemm_ex)
                    variants = []
                    for v in range(3):                                    # row step i with i % 3 == v: slot s holds kh = (s - i) % 3
                        wk = torch.zeros(2 * C, 3 * C, 3)
                        for s in range(3):
                            wk[:, s * C:(s + 1) * C, :] = w[:, :, (s - v) % 3, :]
                        variants.append(ops.pack_weight(wk, dev))
                    layers.append(dict(conv=variants, conv_b=p[q + "conv.bias"].to(dev),
                                       out=ops.pack_weight(p[q + "out_proj.weight"][:, :, 0, 0], dev), out_b=p[q + "out_proj.bias"].to(dev)))
            f32 = lambda t: t.detach().float().contiguous().numpy().astype("float32").copy()
            host = dict(in_w=f32(p[pre + "input_proj.weight"].reshape(-1)), in_b=f32(p[pre + "input_proj.bias"]),
                        out_w=f32(p[pre + "output_proj.weight"].reshape(2, C)), out_b=f32(p[pre + "output_proj.bias"]))
            flow = dict(host=host, in_w=p[pre + "input_proj.weight"].reshape(-1).contiguous().to(dev),
                        in_b=p[pre + "input_proj.bias"].to(dev), layers=layers)
            if not fused:
                # the condition projections of all layers of a flow in one GEMM per row step (they do not depend on the recurrence)
                cond_w = torch.cat([p[f"{pre}resnet.{l}.condition_proj.weight"][:, :, 0, 0] for l in range(self.n_layers)], dim=0)
                cond_b = torch.cat([p[f"{pre}resnet.{l}.condition_proj.bias"] for l in range(self.n_layers)])
                flow.update(cond_all=ops.pack_weight(cond_w, dev), cond_all_b=cond_b.contiguous().to(dev),
                            out_w=p[pre + "output_proj.weight"].reshape(2, C).contiguous().to(dev),
                            out_b=p[pre + "output_proj.bias"].to(dev))
            pk["flows"].append(flow)
        pk["perms"] = [torch.tensor(pm, dtype=torch.int64, device=dev) for pm in self.perms]   # device-side gather indices
        self._packed = pk
        return pk

    def _eligible(self):
        """Whether the fused kernels cover this config: 64 or 128 residual channels, 64 < n_mels <= 128 (a multiple of 8) and 2
        to 8 layers per flow.  Then inverse runs pk_waveflow_flow (one persistent launch per flow); any other config runs it as
        the two-GEMM row loop (pk_conv_gemm_ex) and has no density direction.  One layer is excluded because pk_waveflow_flow's
        dataflow needs the last layer's write of the next row into layer 0's ring to be a later layer-step than layer 0's reads
        of that ring slot."""
        return self.channels in (64, 128) and 64 < self.n_mels <= 128 and self.n_mels % 8 == 0 and 2 <= self.n_layers <= 8

    def _run_flow(self, fw, z, x, cond_s, cmap, bufs, skip, flags, st):
        """Rows 1 .. G-1 of one flow in one launch (row 0 and the ring contents are prepared by the caller)."""
        L = _lib.lib()
        B, G, W = z.shape
        NL = self.n_layers
        lay = [l_["fused"] for l_ in fw["layers"]]
        vpa = lambda ptrs: (C_.c_void_p * len(ptrs))(*ptrs)
        keep = dict(cond_rows=(C_.c_int32 * G)(*cmap), ring_hi=vpa([_ptr(b_.hi) for b_ in bufs]), ring_lo=vpa([_ptr(b_.lo) for b_ in bufs]),
                    w1_hi=vpa([_ptr(f["w1"][v][0]) for f in lay for v in range(3)]),
                    w1_lo=vpa([_ptr(f["w1"][v][1]) for f in lay for v in range(3)]),
                    w2_hi=vpa([_ptr(f["w2"][0]) for f in lay]), w2_lo=vpa([_ptr(f["w2"][1]) for f in lay]),
                    bias1=vpa([f["b1"].ctypes.data for f in lay]), bias2=vpa([f["b2"].ctypes.data for f in lay]))
        a = _lib.WaveflowFlowArgs()
        a.batch, a.width, a.channels, a.n_mels, a.n_layers, a.n_group = B, W, self.channels, self.n_mels, NL, G
        for k, v in keep.items():
            setattr(a, k, C_.cast(v, C_.c_void_p))
        a.cond_hi, a.cond_lo = _ptr(cond_s.hi), _ptr(cond_s.lo)
        h = fw["host"]
        a.in_w, a.in_b, a.out_w, a.out_b = (h[k].ctypes.data for k in ("in_w", "in_b", "out_w", "out_b"))
        a.z, a.x, a.skip, a.flags, a.flags_len = _ptr(z), _ptr(x), _ptr(skip), _ptr(flags), flags.numel()
        _lib.check(L.pk_waveflow_flow(C_.byref(a), st), "pk_waveflow_flow")

    def encode(self, mel, trim_conv_artifact=True):
        """UpsampleNet.forward (:103-132): (B, n_mels, T') -> (B, n_mels, T)."""
        pk = self._pack()
        x = mel.contiguous().float()
        L = _lib.lib()
        for (w, b), f in zip(pk["enc"], self.upsample_factors):
            B, Cm, Tin = x.shape
            y = torch.empty(B, Cm, Tin * f - (f if trim_conv_artifact else 0), device=x.device)
            _lib.check(L.pk_waveflow_upsample(_ptr(x), _ptr(w), _ptr(b), B, Cm, Tin, f, 1 if trim_conv_artifact else 0, 0.4,
                                              _ptr(y), _stream()), "pk_waveflow_upsample")
            x = y
        return x

    def inverse(self, z, condition):
        """WaveFlow.inverse (:674-711): z (B, T), condition (B, n_mels, T) -> audio (B, T')."""
        pk = self._pack()
        L = _lib.lib()
        G, C, NL = self.n_group, self.channels, self.n_layers
        pruned = z.shape[-1] // G * G
        z, condition = z[:, :pruned].float(), condition[:, :, :pruned]
        B = z.shape[0]
        W = pruned // G
        dev = z.device
        z = z.reshape(B, W, G).transpose(1, 2).contiguous()                               # (B, H, W): sample t = w*G + h
        cond = condition.reshape(B, self.n_mels, W, G).permute(0, 3, 2, 1).contiguous()   # (B, H, W, n_mels) channels-last
        cond_s = Split.from_f32(cond)
        cmap = list(range(G))                                                             # cumulative row permutation of the condition
        state = torch.empty(B, W, C, device=dev)
        skip = torch.empty(B, W, C, device=dev)
        h_all = torch.empty(B, W, NL * 2 * C, device=dev)                                 # condition projections of one row step
        zt = Split.empty((B, W, C), dev)
        bufs = [Split.zeros((B, W, 3 * C), dev) for _ in range(NL)]
        st = _stream()
        fused = self._eligible()
        flags = torch.empty((G - 1) * NL * B * ((W + 255) // 256), dtype=torch.int32, device=dev) if fused else None
        for fi in reversed(range(self.n_flows)):
            perm = self.perms[fi]
            z = z.index_select(1, pk["perms"][fi])                                        # geo.shuffle_dim(z, 2, perm)
            cmap = [cmap[j] for j in perm]
            fw = pk["flows"][fi]
            x = torch.empty_like(z)
            x[:, 0] = z[:, 0]
            for b_ in bufs:
                b_.hi.zero_()
                b_.lo.zero_()
            if fused:
                z = z.contiguous()
                _lib.check(L.pk_waveflow_input_proj(_ptr(x[:, 0]), G * W, _ptr(fw["in_w"]), _ptr(fw["in_b"]), B, W, C,
                                                    _ptr(state), _ptr(bufs[0].hi), _ptr(bufs[0].lo), 3 * C, 0, st),
                           "pk_waveflow_input_proj")
                flags.zero_()
                self._run_flow(fw, z, x, cond_s, cmap, bufs, skip, flags, st)
                z = x
                continue
            for i in range(1, G):
                slot = (i - 1) % 3                                                        # ring slot of the newest row (row i-1)
                _lib.check(L.pk_waveflow_input_proj(_ptr(x[:, i - 1]), G * W, _ptr(fw["in_w"]), _ptr(fw["in_b"]), B, W, C,
                                                    _ptr(state), _ptr(bufs[0].hi), _ptr(bufs[0].lo), 3 * C, slot * C, st),
                           "pk_waveflow_input_proj")
                c_row = Split(cond_s.hi[:, cmap[i]], cond_s.lo[:, cmap[i]])              # (B, W, n_mels) views, batch stride G*W*n_mels
                ops.conv_gemm(c_row, fw["cond_all"], n=NL * 2 * C, k=self.n_mels, bias=fw["cond_all_b"], y_f32=h_all)
                for l, lay in enumerate(fw["layers"]):
                    # dilated conv over the 3-row ring + condition slice -> tanh * sigmoid, fused in the GEMM epilogue
                    ops.conv_gemm(bufs[l], lay["conv"][i % 3], n=2 * C, k=3 * C, taps=3, dil=2 ** l, bias=lay["conv_b"], y_split=zt,
                                  epilogue=dict(mode="gate", channels=C, residual=h_all[:, :, l * 2 * C:(l + 1) * 2 * C]))
                    # out_proj -> (res | skip): state += res, skip += skip, next layer's ring slot <- new state, in the epilogue
                    nxt = bufs[l + 1] if l + 1 < NL else None
                    ops.conv_gemm(zt, lay["out"], n=2 * C, k=C, bias=lay["out_b"],
                                  epilogue=dict(mode="wf_update", channels=C, state=state, skip=skip, skip_init=(l == 0), buf=nxt,
                                                buf_col0=slot * C))
                _lib.check(L.pk_waveflow_row_out(_ptr(skip), _ptr(fw["out_w"]), _ptr(fw["out_b"]), _ptr(z[:, i]), G * W, B, W, C,
                                                 _ptr(x[:, i]), G * W, st), "pk_waveflow_row_out")
            z = x
        return z.transpose(1, 2).reshape(B, -1)

    def _check_forward(self, audio_len, cond_len):
        if not self._eligible():
            raise NotImplementedError("ConditionalWaveFlow.forward needs 64 or 128 channels, 64 < n_mels <= 128 (a multiple of 8) "
                                      "and 2 to 8 layers per flow")
        if audio_len > cond_len:
            raise ValueError(f"audio ({audio_len} samples) is longer than its condition ({cond_len} samples)")

    def decoder_forward(self, audio, condition):
        """WaveFlow.forward (:627-672): audio (B, T), upsampled condition (B, n_mels, T_c >= T) ->
        (z (B, T // n_group * n_group), log_det_jacobian (1,)).  The counterpart of inverse(z, condition)."""
        self._check_forward(audio.shape[-1], condition.shape[-1])
        ops._require_cuda(audio, condition)
        pk = self._pack()
        L = _lib.lib()
        G, C, NL = self.n_group, self.channels, self.n_layers
        pruned = audio.shape[-1] // G * G                                                 # _trim (:617-625)
        B, W, dev = audio.shape[0], pruned // G, audio.device
        x = audio[:, :pruned].float().reshape(B, W, G).transpose(1, 2).contiguous()     # (B, H, W): sample t = w*G + h
        cond = condition[:, :, :pruned].float().reshape(B, self.n_mels, W, G).permute(0, 3, 2, 1).contiguous()
        cond_s = Split.from_f32(cond)                                                     # (B, H, W, n_mels), never permuted
        bufs = [Split.zeros((B * (G + 1), W, C), dev) for _ in range(2)]                  # 2 zero rows + G - 1 net rows each
        skip = torch.empty(B, G - 1, W, C, device=dev)
        log_det = torch.zeros(1, device=dev)
        partials = torch.empty(_lib.WAVEFLOW_TAIL_PARTIALS, device=dev)
        counter = torch.zeros(1, dtype=torch.int32, device=dev)
        x_next = torch.empty_like(x)
        st = _stream()
        i32 = lambda v: (C_.c_int32 * G)(*v)

        def tail(fw, perm, nxt, x_in, x_out):
            a = _lib.WaveflowForwardTailArgs()
            a.batch, a.width, a.channels, a.n_group = B, W, C, G
            keep = dict(perm=i32(perm))
            a.perm = C_.cast(keep["perm"], C_.c_void_p)
            a.x, a.x_next = _ptr(x_in), _ptr(x_out)
            if fw is not None:
                h = fw["host"]
                a.skip, a.out_w, a.out_b = _ptr(skip), h["out_w"].ctypes.data, h["out_b"].ctypes.data
                a.log_det, a.partials, a.counter = _ptr(log_det), _ptr(partials), _ptr(counter)
            if nxt is not None:
                a.in_w, a.in_b = nxt["host"]["in_w"].ctypes.data, nxt["host"]["in_b"].ctypes.data
                a.next_hi, a.next_lo = _ptr(bufs[0].hi), _ptr(bufs[0].lo)
            _lib.check(L.pk_waveflow_forward_tail(C_.byref(a), st), "pk_waveflow_forward_tail")

        flows = pk["flows"]
        tail(None, list(range(G)), flows[0], x, None)                                    # input_proj of the first flow
        cmap = list(range(G))                                                             # condition height of height h
        for fi, fw in enumerate(flows):
            rows = i32(cmap)
            src, dst = bufs
            for l, lay in enumerate(fw["layers"]):
                f = lay["fused"]
                a = _lib.WaveflowForwardLayerArgs()
                a.batch, a.width, a.channels, a.n_mels, a.n_group, a.dilation = B, W, C, self.n_mels, G, 2 ** l
                a.cond_rows = C_.cast(rows, C_.c_void_p)
                a.x_hi, a.x_lo = _ptr(src.hi), _ptr(src.lo)
                a.cond_hi, a.cond_lo = _ptr(cond_s.hi), _ptr(cond_s.lo)
                w1 = f["w1"][0]                                                           # variant 0: ring slot s = kernel row s
                a.w1_hi, a.w1_lo, a.w2_hi, a.w2_lo = _ptr(w1[0]), _ptr(w1[1]), _ptr(f["w2"][0]), _ptr(f["w2"][1])
                a.bias1, a.bias2 = f["b1"].ctypes.data, f["b2"].ctypes.data
                if l + 1 < NL:
                    a.y_hi, a.y_lo = _ptr(dst.hi), _ptr(dst.lo)
                a.skip, a.skip_init = _ptr(skip), 1 if l == 0 else 0
                _lib.check(L.pk_waveflow_forward_layer(C_.byref(a), st), "pk_waveflow_forward_layer")
                src, dst = dst, src
            # output_proj, z, log-det, the permutation of the heights and the next flow's input_proj (into bufs[0])
            tail(fw, self.perms[fi], flows[fi + 1] if fi + 1 < len(flows) else None, x, x_next)
            x, x_next = x_next, x
            cmap = [cmap[j] for j in self.perms[fi]]                                      # geo.shuffle_dim(condition, 2, perm)
        return x.transpose(1, 2).reshape(B, -1), log_det

    def forward(self, audio, mel):
        """ConditionalWaveFlow.forward (:759-783): audio (B, T), mel (B, n_mels, T') -> (z (B, T // n_group * n_group),
        log_det_jacobian (1,)), the condition being the encoder output WITHOUT the trim of infer (256 T' samples)."""
        t_cond = mel.shape[-1]
        for f in self.upsample_factors:
            t_cond *= f
        self._check_forward(audio.shape[-1], t_cond)
        if not (audio.is_cuda and mel.is_cuda):
            raise _lib.PkError("ConditionalWaveFlow needs CUDA tensors (no CPU fallback)")
        audio, mel = audio.contiguous().float(), mel.contiguous().float()
        fn = lambda a_, m_: self.decoder_forward(a_, self.encode(m_, trim_conv_artifact=False))
        z, log_det = self._graphs.run(("forward", audio.shape[0], audio.shape[-1], mel.shape[-1]), fn, [audio, mel])
        return z.clone(), log_det.clone()

    def infer(self, mel, z=None):
        """reference :784-805; the noise z (B, T_c) may be supplied (parity tests), else torch.randn."""
        if not mel.is_cuda:
            raise _lib.PkError("ConditionalWaveFlow needs CUDA tensors (no CPU fallback)")
        mel = mel.contiguous().float()
        B, _, frames = mel.shape
        t_c = frames
        for f in self.upsample_factors:                                     # each transposed conv trims f samples (:121-126)
            t_c = t_c * f - f
        if z is None:
            z = torch.randn(B, t_c, device=mel.device)
        assert z.shape == (B, t_c), (tuple(z.shape), (B, t_c))
        # one CUDA graph per (B, frames): the 5 040 small launches of the row-by-row inverse replay without host work
        fn = lambda m_, z_: self.inverse(z_, self.encode(m_, trim_conv_artifact=True))
        return self._graphs.run(("infer", B, frames), fn, [mel, z.contiguous().float()]).clone()

    @classmethod
    def from_pretrained(cls, config, checkpoint_path, device=None):
        """reference :827-852: build from a config (attribute or mapping access: config.model.*, config.data.n_mels) and load
        `checkpoint_path + ".pdparams"` (utils/checkpoint.py:load_parameters appends the extension) without PaddlePaddle."""
        import os
        from .. import checkpoint

        def get(node, key):
            return node[key] if isinstance(node, dict) else getattr(node, key)
        mc, dc = get(config, "model"), get(config, "data")
        model = cls(upsample_factors=list(get(mc, "upsample_factors")), n_flows=get(mc, "n_flows"), n_layers=get(mc, "n_layers"),
                    n_group=get(mc, "n_group"), channels=get(mc, "channels"), n_mels=get(dc, "n_mels"),
                    kernel_size=tuple(get(mc, "kernel_size")), device=device)
        path = str(checkpoint_path)
        if not os.path.exists(path) and os.path.exists(path + ".pdparams"):
            path = path + ".pdparams"
        model.set_state_dict(checkpoint.load(path))
        return model

    def predict(self, mel):
        """reference :807-825: numpy mel (n_mels, T') -> numpy audio."""
        mel = torch.as_tensor(np.asarray(mel), dtype=torch.float32, device=self.device).unsqueeze(0)
        return self.infer(mel)[0].cpu().numpy()


class WaveFlowLoss:
    """WaveFlowLoss (reference :855-891): (sum z^2 / (2 sigma^2) - log_det_jacobian) / numel(z) + log(2 pi) / 2 + log(sigma),
    shape (1,) - the negative log-likelihood per sample of a Gaussian prior.  sum z^2 is pk_sq_sum (double accumulator)."""

    def __init__(self, sigma=1.0):
        if not sigma > 0:
            raise ValueError("sigma must be positive")
        self.sigma = float(sigma)

    def forward(self, z, log_det_jacobian):
        ops._require_cuda(z, log_det_jacobian)
        L = _lib.lib()
        z = z.contiguous().float()
        log_det_jacobian = log_det_jacobian.contiguous().float()
        sq = torch.zeros(1, dtype=torch.float64, device=z.device)
        loss = torch.empty(1, device=z.device)
        st = _stream()
        _lib.check(L.pk_sq_sum(_ptr(z), z.numel(), _ptr(sq), st), "pk_sq_sum")
        _lib.check(L.pk_waveflow_nll(_ptr(sq), _ptr(log_det_jacobian), z.numel(), self.sigma, _ptr(loss), st), "pk_waveflow_nll")
        return loss

    __call__ = forward
