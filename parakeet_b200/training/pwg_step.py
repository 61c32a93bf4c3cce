"""Parallel WaveGAN training step on H100 (reference: PWGUpdater.update_core, parakeet/models/parallel_wavegan/
parallel_wavegan_updater.py:76-153; set-up examples/GANVocoder/parallelwave_gan/baker/train.py; SURVEY.md 8f.1).

    generator step      wav_ = G(noise, mel);  loss = MR-STFT(wav_, wav) [+ lambda_adv * MSE(D(wav_), 1) once
                        iteration > discriminator_train_start_steps];  backward;  ClipGradByGlobalNorm + Adam (StepDecay lr)
    discriminator step  (same condition)  wav_ = G(noise, mel) with the UPDATED generator, detached;
                        loss = MSE(D(wav), 1) + MSE(D(wav_), 0);  backward;  clip + Adam

This is the training-mode formulation of the generator: every intermediate the backward pass needs (pre-gate activations,
z, the layer inputs, the upsampling stages) is kept, so the residual stack runs as separate wgmma GEMMs (`pk_conv_gemm`:
dilated conv + aux 1x1 accumulated through the residual operand, skip|out 1x1) around the element-wise kernels of csrc/gan.cu
instead of the fused inference kernel (csrc/pwg_fc.cu), which keeps nothing.  Data gradients are convolutions with flipped taps,
weight gradients NT matmuls over the flattened batch x time axis on transposed split planes (training/wgrad.py: splitk_wgrad, the
tap shifts scaled by the dilation).  The STFT losses differentiate through pk_stft's re / im outputs: the adjoint of the windowed
DFT is a GEMM with the DFT basis followed by an overlap-add through the reflect padding.  Weight norm (g, v) is re-folded every
step and its backward maps dw to (dg, dv).  Parameters, gradients and Adam moments of each network live in flat buffers
(training/flat.py: FlatAdam; one NCCL all-reduce per network and step under data parallelism, like paddle.DataParallel's gradient
mean).
torch is used for buffers, views / copies (layout) and torch.distributed only.
"""
import math

import numpy as np
import torch
import torch.distributed as dist

from .. import _lib, ops
from ..ops import Split, _ptr, _stream, ceil_to, pack_dev
from ..modules.audio import STFT
from . import wgrad
from .conv import ConvOps
from .flat import FlatAdam, broadcast_from_rank0, step_graphs


class _Net:
    """Weight-normed conv parameters of one network in flat buffers + the folded weights of the current step."""

    def __init__(self, layer, device, eps, clip):
        self.layer = layer
        self.opt = opt = FlatAdam(layer._params, list(layer._params.keys()), device, epsilon=eps, clip_norm=clip)
        self.buffers, self.flat, self.gflat, self.grads = opt.buffers, opt.flat, opt.gflat, opt.grads
        self.w = {}                     # folded weights (fp32, Paddle layouts) of the current step
        self.dw = {}                    # gradients w.r.t. the folded weights
        layer._packed = None

    steps = property(lambda self: self.opt.steps)

    def P(self, k):
        return self.layer._params[k]

    def fold(self):
        """weight_g / weight_v -> weight (every step: the optimiser moves g and v)."""
        L = _lib.lib()
        self.w, self.dw = {}, {}
        for k, v in self.layer._params.items():
            if k.endswith("weight_v"):
                name = k[:-2]
                w = torch.empty_like(v)
                _lib.check(L.pk_weight_norm_fwd(_ptr(v), _ptr(self.P(name + "_g")), v.shape[0], v.numel() // v.shape[0], _ptr(w), None,
                                                _stream()), "pk_weight_norm_fwd")
                self.w[name] = w
            elif k.endswith("weight_g"):
                continue
            else:
                self.w[k] = v           # biases and un-normalised weights: the parameter itself
        for k, w in self.w.items():
            self.dw[k] = self.grads[k] if k in self.grads else torch.zeros_like(w)   # weight-normed: scratch, mapped in unfold()

    def unfold_grads(self):
        """dw -> (dg, dv) for the weight-normed tensors (biases / plain weights wrote into their gradient views directly)."""
        L = _lib.lib()
        for k, v in self.layer._params.items():
            if k.endswith("weight_v"):
                name = k[:-2]
                _lib.check(L.pk_weight_norm_bwd(_ptr(v), _ptr(self.P(name + "_g")), _ptr(self.dw[name]), v.shape[0], v.numel() // v.shape[0],
                                                _ptr(self.grads[name + "_g"]), _ptr(self.grads[k]), _stream()), "pk_weight_norm_bwd")

    def update(self, lr, world, group=None):
        self.opt.update(lr, world, group)
        self.layer._packed = None


class PWGTrainStep:
    def __init__(self, generator, discriminator, lr_g=1e-4, lr_d=5e-5, eps=1e-6, grad_norm_g=10.0, grad_norm_d=1.0, step_size=200000,
                 gamma=0.5, lambda_adv=4.0, discriminator_train_start_steps=100000, stft_loss_params=None, process_group=None,
                 use_graphs=None):
        """Defaults: examples/GANVocoder/parallelwave_gan/baker/conf/default.yaml (optimiser / scheduler / loss sections).
        `discriminator`: a PWGDiscriminator (models/parallel_wavegan.py); both networks must carry weight norm (the reference trains
        the g / v parametrisation)."""
        dev = generator.device
        if dev.type != "cuda":
            raise _lib.PkError("training needs a CUDA device (no CPU fallback)")
        self.G, self.D = generator, discriminator
        if not generator._weight_norm:
            generator.apply_weight_norm()
        self.g, self.d = _Net(generator, dev, eps, grad_norm_g), _Net(discriminator, dev, eps, grad_norm_d)
        self.lr_g, self.lr_d, self.step_size, self.gamma = lr_g, lr_d, step_size, gamma
        self.lambda_adv, self.d_start = lambda_adv, discriminator_train_start_steps
        self.iteration = 0
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        sp = dict(fft_sizes=[1024, 2048, 512], hop_sizes=[120, 240, 50], win_lengths=[600, 1200, 240], window="hann")
        sp.update(stft_loss_params or {})
        self.res = []
        for nf, hop, wl in zip(sp["fft_sizes"], sp["hop_sizes"], sp["win_lengths"]):
            st = STFT(nf, hop, wl, sp["window"], device=dev)
            bins = nf // 2 + 1
            bins_p = ceil_to(bins, 64)
            n = torch.arange(nf, dtype=torch.float64)[:, None]
            k = torch.arange(bins, dtype=torch.float64)[None, :]
            basis = torch.zeros(nf, 2 * bins_p, dtype=torch.float64)
            basis[:, :bins] = torch.cos(2 * math.pi * k * n / nf)              # d re[k] / d frame[n]
            basis[:, bins_p:bins_p + bins] = -torch.sin(2 * math.pi * k * n / nf)   # d im[k] / d frame[n]
            self.res.append(dict(stft=st, n_fft=nf, hop=hop, bins=bins, bins_p=bins_p, basis=pack_dev(basis.float().to(dev))))
        # forward + backward of each half of update_core replay as a CUDA graph per batch shape (the step is ~2 500 small launches;
        # the Adam kernels stay outside: their bias correction is a host-computed scalar).  PK_TRAIN_GRAPH=0 disables.
        self._graphs = step_graphs(8, use_graphs)
        # the weight-gradient operand planes are filed per (batch, length) geometry and baked into the captured graphs: if a geometry
        # is evicted (more than 16 distinct ones), every graph of this step is dropped and captured again
        self._zp = wgrad.ZeroPlanes(max_geoms=16, on_evict=lambda _: self._graphs.clear())
        self.conv = ConvOps(self._zp)
        if self.world > 1:
            for net in (self.g, self.d):
                broadcast_from_rank0(net.flat, net.layer._params, process_group)

    def conv_bwd(self, dy, x, key, w, dil, dw, db, need_dx=True, accumulate=False):
        """dy fp32 (B, T, Cout); x Split saved input (B, T, >= Cin).  Writes dw (Cout, Cin, k) / db (or accumulates); returns dx fp32
        (B, T, Cin) or None."""
        B, T, cout = dy.shape
        dys = ops.split_pad8(dy)
        if db is not None:
            ops.colsum_(dy.reshape(B * T, cout), db)       # pk_colsum ACCUMULATES: bias gradients start from the zeroed flat buffer
        dx = self.conv.dgrad(dys, key, w, dil=dil) if need_dx else None
        self._zp.begin(("pwg", B, T))    # one step visits two or three geometries (sample rate, frame rate)
        g = self.conv.wgrad(x, dys, w, dil=dil)
        if accumulate:
            ops.axpy_(1.0, g.contiguous(), dw)
        else:
            dw.copy_(g)
        return dx

    # ------------------------------------------------------------------------------------------------------------
    # schedules
    # ------------------------------------------------------------------------------------------------------------
    def _lr(self, base, epochs):
        return base * self.gamma ** (epochs // self.step_size)      # StepDecay; each scheduler steps once per update of ITS optimiser

    # ------------------------------------------------------------------------------------------------------------
    # discriminator (parallel_wavegan.py:554-614)
    # ------------------------------------------------------------------------------------------------------------
    def d_forward(self, wav, save):
        """wav fp32 (B, T) -> logits (B, T, 1); `save` collects (input split, pre-activation) per layer."""
        net, L = self.d, _lib.lib()
        B, T = wav.shape
        n_layers = self.D.layers
        x8 = torch.zeros(B, T, 8, dtype=torch.float32, device=wav.device)
        x8[:, :, 0] = wav
        h = Split.from_f32(x8)
        out = None
        for i in range(n_layers):
            name = f"conv_layers.{2 * i}"
            w, b = net.w[name + ".weight"], net.w.get(name + ".bias")
            y, _ = self.conv.fwd(h, "d" + name, w, bias=b, dil=self.D.dilations[i])
            if i < n_layers - 1:
                a = Split.empty(tuple(y.shape), y.device)
                _lib.check(L.pk_leaky_relu(_ptr(y), y.numel(), self.D.slope, None, _ptr(a.hi), _ptr(a.lo), _stream()), "pk_leaky_relu")
                save.append((h, y))
                h = a
            else:
                save.append((h, y))
                out = y
        return out

    def d_backward(self, dout, save, need_dx, param_grads, accumulate=False):
        """dout (B, T, 1) -> gradient w.r.t. the input wav (B, T) if need_dx; parameter gradients into self.d.dw."""
        net, L = self.d, _lib.lib()
        n_layers = self.D.layers
        g = dout
        for i in reversed(range(n_layers)):
            name = f"conv_layers.{2 * i}"
            h_in, pre = save[i]
            if i < n_layers - 1:
                dpre = torch.empty_like(pre)
                _lib.check(L.pk_leaky_relu_bwd(_ptr(pre), _ptr(g), pre.numel(), self.D.slope, _ptr(dpre), _stream()), "pk_leaky_relu_bwd")
                g = dpre
            w = net.w[name + ".weight"]
            last = i == 0
            if param_grads:
                dx = self.conv_bwd(g, h_in, "d" + name, w, self.D.dilations[i], net.dw[name + ".weight"], net.dw.get(name + ".bias"),
                                   need_dx=(not last) or need_dx, accumulate=accumulate)
            else:
                dx = self.conv.dgrad(ops.split_pad8(g), "d" + name, w, dil=self.D.dilations[i]) if ((not last) or need_dx) else None
            g = dx
        return g[:, :, 0].contiguous() if (need_dx and g is not None) else None

    def _mse(self, x, target, dx_coef=None):
        """MSELoss (mean) of logits (B, T, 1) against a constant; returns (loss 0-d tensor, d loss / dx * dx_coef or None)."""
        n = x.numel()
        acc = torch.zeros(1, dtype=torch.float64, device=x.device)
        dx = torch.empty_like(x) if dx_coef is not None else None
        _lib.check(_lib.lib().pk_mse_const(_ptr(x), n, 1, 0, float(target), _ptr(acc), _ptr(dx), 2.0 * (dx_coef or 0.0) / n, _stream()),
                   "pk_mse_const")
        return (acc[0] / n).float(), dx

    # ------------------------------------------------------------------------------------------------------------
    # multi-resolution STFT loss with gradient (modules/stft_loss.py:163-219)
    # ------------------------------------------------------------------------------------------------------------
    def stft_loss(self, wav_, wav, want_grad=True):
        """-> (sc_loss, mag_loss, d (sc + mag) / d wav_ (B, T) or None)."""
        L = _lib.lib()
        B, T = wav_.shape
        dev = wav_.device
        dx = torch.zeros(B, T, dtype=torch.float32, device=dev) if want_grad else None
        sc_tot, mag_tot = 0.0, 0.0
        nres = len(self.res)
        for r in self.res:
            st = r["stft"]
            ox = st._run(wav_, re=True, im=True, mag=True, mag_layout=0, power_clip=1e-7)
            oy = st._run(wav, re=True, im=True, mag=True, mag_layout=0, power_clip=1e-7)
            sums = torch.empty(3, dtype=torch.float32, device=dev)
            _lib.check(L.pk_spectral_loss_sums(_ptr(ox["mag"]), _ptr(oy["mag"]), ox["mag"].numel(), 1e-7, _ptr(sums), _stream()),
                       "pk_spectral_loss_sums")
            sc_tot = sc_tot + torch.sqrt(sums[0]) / torch.clamp(torch.sqrt(sums[1]), min=1e-10)
            mag_tot = mag_tot + sums[2] / ox["mag"].numel()
            if want_grad:
                frames = ox["re"].shape[-1]
                g = torch.zeros(B * frames, 2 * r["bins_p"], dtype=torch.float32, device=dev)
                _lib.check(L.pk_stft_loss_grad(_ptr(ox["re"]), _ptr(ox["im"]), _ptr(oy["re"]), _ptr(oy["im"]), B, r["bins"], frames, r["bins_p"],
                                               _ptr(sums), 1.0 / nres, _ptr(g), _stream()), "pk_stft_loss_grad")
                gs = Split.from_f32(g.reshape(1, B * frames, 2 * r["bins_p"]))
                fg, _ = ops.conv_gemm(gs, r["basis"], n=r["n_fft"], k=2 * r["bins_p"])           # adjoint DFT: (B * frames, n_fft)
                _lib.check(L.pk_frames_overlap_add(_ptr(fg), _ptr(st._win), B, frames, r["n_fft"], r["hop"], T, _ptr(dx), _stream()),
                           "pk_frames_overlap_add")
        return sc_tot / nres, mag_tot / nres, dx

    # ------------------------------------------------------------------------------------------------------------
    # generator, training formulation (parallel_wavegan.py:445-472)
    # ------------------------------------------------------------------------------------------------------------
    def g_forward(self, noise, mel, save=None):
        """noise (B, 1, T), mel (B, aux, frames + 2 w) -> wav_ (B, T); `save` (dict) keeps what the backward needs."""
        G, net, L = self.G, self.g, _lib.lib()
        B, _, T = noise.shape
        A, dev = G.aux_channels, noise.device
        keep = save is not None
        # conv_in (no padding, no bias) on channels-last mel, then the upsampling stages on (B * aux) rows
        mel_cl = Split.from_f32(mel.transpose(1, 2).contiguous())                     # (B, frames + 2w, aux)
        w_in = net.w["upsample_net.conv_in.weight"]
        kin = w_in.shape[-1]
        cin_full, _ = self.conv.fwd(mel_cl, "conv_in", w_in, pad=0)
        frames = mel.shape[-1] - (kin - 1)
        m1 = cin_full[:, :frames].contiguous()                                        # taps at +0 .. +kin-1: valid for the first `frames` rows
        ups = [m1.transpose(1, 2).reshape(B * A, frames).contiguous()]
        tin = frames
        for i, s in enumerate(G.upsample_scales):
            fir = net.w[f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"].reshape(-1)
            y = torch.empty(B * A, tin * s, dtype=torch.float32, device=dev)
            _lib.check(L.pk_up_stage_fwd(_ptr(ups[-1]), _ptr(fir), B * A, tin, s, _ptr(y), _stream()), "pk_up_stage_fwd")
            ups.append(y)
            tin *= s
        assert tin == T
        c = Split.from_f32(ups[-1].reshape(B, A, T).transpose(1, 2).contiguous())     # (B, T, aux)
        # first conv 1 -> R, k = 1
        n8 = torch.zeros(B, T, 8, dtype=torch.float32, device=dev)
        n8[:, :, 0] = noise[:, 0]
        n8s = Split.from_f32(n8)
        x, xs = self.conv.fwd(n8s, "first", net.w["first_conv.weight"], bias=net.w["first_conv.bias"], out_split=True)
        skips = torch.empty(B, T, 64, dtype=torch.float32, device=dev)
        layers = []
        lps = G.layers // G.stacks
        for i in range(G.layers):
            pre = f"conv_layers.{i}."
            d = 2 ** (i % lps)
            h1, _ = self.conv.fwd(xs, "g" + pre + "conv", net.w[pre + "conv.weight"], bias=net.w.get(pre + "conv.bias"), dil=d)
            h, _ = self.conv.fwd(c, "g" + pre + "aux", net.w[pre + "conv1x1_aux.weight"], residual=h1)
            z = Split.empty((B, T, 64), dev)
            _lib.check(L.pk_gate_fwd(_ptr(h), B * T, 64, None, _ptr(z.hi), _ptr(z.lo), _stream()), "pk_gate_fwd")
            w2 = torch.cat([net.w[pre + "conv1x1_skip.weight"], net.w[pre + "conv1x1_out.weight"]], dim=0)
            b2 = torch.cat([net.w[pre + "conv1x1_skip.bias"], net.w[pre + "conv1x1_out.bias"]])
            so, _ = self.conv.fwd(z, "g" + pre + "so", w2, bias=b2)
            xo = torch.empty(B, T, 64, dtype=torch.float32, device=dev)
            xos = Split.empty((B, T, 64), dev)
            _lib.check(L.pk_pwg_res_update(_ptr(so), _ptr(x), B * T, _ptr(skips), 1 if i == 0 else 0, _ptr(xo), _ptr(xos.hi), _ptr(xos.lo),
                                           _stream()), "pk_pwg_res_update")
            if keep:
                layers.append(dict(xs=xs, h=h, z=z, w2=w2, d=d))
            x, xs = xo, xos
        # tail: skips * sqrt(1/L) -> ReLU -> 1x1 -> ReLU -> 1x1
        u0 = torch.empty_like(skips)
        _lib.check(L.pk_leaky_relu(_ptr(skips), skips.numel(), 0.0, _ptr(u0), None, None, _stream()), "pk_leaky_relu")   # ReLU; scale below
        scale = math.sqrt(1.0 / G.layers)
        u0s = Split.from_f32(u0)
        w1t = net.w["last_conv_layers.1.weight"]
        # relu(s * k) = k * relu(s) for k > 0: the scale is folded into the 1x1 weights of this step
        v1, _ = self.conv.fwd(u0s, "tail1", w1t * scale, bias=net.w["last_conv_layers.1.bias"])
        u1 = Split.empty(tuple(v1.shape), dev)
        _lib.check(L.pk_leaky_relu(_ptr(v1), v1.numel(), 0.0, None, _ptr(u1.hi), _ptr(u1.lo), _stream()), "pk_leaky_relu")
        out, _ = self.conv.fwd(u1, "tail3", net.w["last_conv_layers.3.weight"], bias=net.w["last_conv_layers.3.bias"])
        if keep:
            save.update(mel_cl=mel_cl, frames=frames, ups=ups, c=c, n8s=n8s, layers=layers, skips=skips, u0s=u0s, v1=v1, u1=u1, scale=scale)
        return out[:, :, 0].contiguous()

    def g_backward(self, dwav, S):
        """dwav (B, T): d loss / d wav_.  Fills self.g.dw."""
        G, net, L = self.G, self.g, _lib.lib()
        B, T = dwav.shape
        A, dev = G.aux_channels, dwav.device
        dout = dwav.reshape(B, T, 1).contiguous()
        du1 = self.conv_bwd(dout, S["u1"], "tail3", net.w["last_conv_layers.3.weight"], 1, net.dw["last_conv_layers.3.weight"],
                            net.dw["last_conv_layers.3.bias"])
        dv1 = torch.empty_like(du1)
        _lib.check(L.pk_leaky_relu_bwd(_ptr(S["v1"]), _ptr(du1), du1.numel(), 0.0, _ptr(dv1), _stream()), "pk_leaky_relu_bwd")
        w1s = net.w["last_conv_layers.1.weight"] * S["scale"]
        dws = torch.empty_like(w1s)
        du0 = self.conv_bwd(dv1, S["u0s"], "tail1", w1s, 1, dws, net.dw["last_conv_layers.1.bias"])
        net.dw["last_conv_layers.1.weight"].copy_(dws * S["scale"])
        dskips = torch.empty_like(du0)
        _lib.check(L.pk_leaky_relu_bwd(_ptr(S["skips"]), _ptr(du0), du0.numel(), 0.0, _ptr(dskips), _stream()), "pk_leaky_relu_bwd")
        dx = torch.zeros(B, T, 64, dtype=torch.float32, device=dev)                   # d loss / d x_30 = 0 (the last block's x is unused)
        dc = torch.zeros(B, T, A, dtype=torch.float32, device=dev)
        for i in reversed(range(G.layers)):
            pre = f"conv_layers.{i}."
            c_ = S["layers"][i]
            dso = torch.empty(B, T, 128, dtype=torch.float32, device=dev)
            dx_res = torch.empty(B, T, 64, dtype=torch.float32, device=dev)
            _lib.check(L.pk_pwg_res_update_bwd(_ptr(dskips), _ptr(dx), B * T, _ptr(dso), _ptr(dx_res), _stream()), "pk_pwg_res_update_bwd")
            dw2 = torch.empty_like(c_["w2"])
            db2 = torch.zeros(128, dtype=torch.float32, device=dev)
            dz = self.conv_bwd(dso, c_["z"], "g" + pre + "so", c_["w2"], 1, dw2, db2)
            net.dw[pre + "conv1x1_skip.weight"].copy_(dw2[:64])
            net.dw[pre + "conv1x1_out.weight"].copy_(dw2[64:])
            net.dw[pre + "conv1x1_skip.bias"].copy_(db2[:64])
            net.dw[pre + "conv1x1_out.bias"].copy_(db2[64:])
            dh = torch.empty(B, T, 128, dtype=torch.float32, device=dev)
            _lib.check(L.pk_gate_bwd(_ptr(c_["h"]), _ptr(dz), B * T, 64, _ptr(dh), _stream()), "pk_gate_bwd")
            dci = self.conv_bwd(dh, S["c"], "g" + pre + "aux", net.w[pre + "conv1x1_aux.weight"], 1, net.dw[pre + "conv1x1_aux.weight"], None)
            ops.axpy_(1.0, dci, dc)
            dxi = self.conv_bwd(dh, c_["xs"], "g" + pre + "conv", net.w[pre + "conv.weight"], c_["d"], net.dw[pre + "conv.weight"],
                                net.dw.get(pre + "conv.bias"))
            ops.axpy_(1.0, dx_res, dxi)
            dx = dxi
        # first conv (input is noise: no data gradient)
        self.conv_bwd(dx, S["n8s"], "first", net.w["first_conv.weight"], 1, net.dw["first_conv.weight"], net.dw["first_conv.bias"], need_dx=False)
        # upsampling net: stages in reverse, then conv_in
        g = dc.transpose(1, 2).reshape(B * A, T).contiguous()
        tin = T
        for i in reversed(range(len(G.upsample_scales))):
            s = G.upsample_scales[i]
            tin //= s
            name = f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"
            fir = net.w[name].reshape(-1)
            dfir = torch.zeros(2 * s + 1, dtype=torch.float64, device=dev)
            gin = torch.empty(B * A, tin, dtype=torch.float32, device=dev)
            _lib.check(L.pk_up_stage_bwd(_ptr(S["ups"][i]), _ptr(g), _ptr(fir), B * A, tin, s, _ptr(gin), _ptr(dfir), _stream()), "pk_up_stage_bwd")
            net.dw[name].copy_(dfir.float().reshape(net.dw[name].shape))
            g = gin
        frames = S["frames"]
        w_in = net.w["upsample_net.conv_in.weight"]
        kin = w_in.shape[-1]
        dm1 = torch.zeros(B, frames + kin - 1, A, dtype=torch.float32, device=dev)    # rows past `frames` carried no output
        dm1[:, :frames] = g.reshape(B, A, frames).transpose(1, 2)
        # conv_in ran with pad = 0 (taps at +0 .. +kin-1): weight gradient with the matching shifts
        self._zp.begin(("pwg", B, frames + kin - 1))
        self.conv.wgrad(S["mel_cl"], ops.split_pad8(dm1), w_in, pad=0, out=net.dw["upsample_net.conv_in.weight"])

    # ------------------------------------------------------------------------------------------------------------
    # one update_core
    # ------------------------------------------------------------------------------------------------------------
    def generator_losses_and_grads(self, noise, mel, wav):
        """Forward + backward of the generator step; gradients end up in self.g.grads (g / v parametrisation).  Returns a dict of
        0-d tensors: spectral_convergence_loss, log_stft_magnitude_loss, [adversarial_loss,] generator_loss."""
        self.conv.reset()
        self.g.fold()
        self.d.fold()
        self.g.gflat.zero_()
        S = {}
        wav_ = self.g_forward(noise, mel, S)
        sc, mag, dwav = self.stft_loss(wav_, wav.reshape(wav_.shape))
        out = dict(spectral_convergence_loss=sc, log_stft_magnitude_loss=mag)
        gen_loss = sc + mag
        if self.iteration > self.d_start:
            save = []
            p_ = self.d_forward(wav_, save)
            adv, dp = self._mse(p_, 1.0, dx_coef=self.lambda_adv)
            dw_adv = self.d_backward(dp, save, need_dx=True, param_grads=False)
            ops.axpy_(1.0, dw_adv, dwav)
            out["adversarial_loss"] = adv
            gen_loss = gen_loss + self.lambda_adv * adv
        out["generator_loss"] = gen_loss
        self.g_backward(dwav, S)
        self.g.unfold_grads()
        self._wav_fake = wav_
        return out

    def discriminator_losses_and_grads(self, noise, mel, wav):
        self.conv.reset()
        self.g.fold()                                    # the generator has just been updated
        self.d.fold()
        self.d.gflat.zero_()
        wav_ = self.g_forward(noise, mel, None)
        B, T = wav_.shape
        s_real, s_fake = [], []
        p = self.d_forward(wav.reshape(B, T), s_real)
        real, dp = self._mse(p, 1.0, dx_coef=1.0)
        self.d_backward(dp, s_real, need_dx=False, param_grads=True)
        p_ = self.d_forward(wav_, s_fake)
        fake, dpf = self._mse(p_, 0.0, dx_coef=1.0)
        self.d_backward(dpf, s_fake, need_dx=False, param_grads=True, accumulate=True)
        self.d.unfold_grads()
        return dict(real_loss=real, fake_loss=fake, discriminator_loss=real + fake)

    def update_core(self, batch, noise=None):
        """batch = (wav (B, 1, T) or (B, T), mel (B, aux, frames + 2 w)); noise (B, 1, T) may be supplied (parity tests), else randn.
        Returns the losses dict of the reference (0-d device tensors)."""
        wav, mel = batch
        dev = self.G.device
        wav, mel = wav.to(dev, torch.float32), mel.to(dev, torch.float32).contiguous()
        wav = wav.reshape(wav.shape[0], -1).contiguous()
        if noise is None:
            noise = torch.randn(wav.shape[0], 1, wav.shape[1], device=dev)
        adversarial = self.iteration > self.d_start
        shape = (tuple(noise.shape), tuple(mel.shape))

        def run(tag, fn, names):
            def once(n_, m_, w_):
                res = fn(n_, m_, w_)
                return tuple(res[k] for k in names)
            vals = self._graphs.run((tag, adversarial) + shape, once, [noise, mel, wav])
            return {k: v.clone() for k, v in zip(names, vals)}
        g_names = ("spectral_convergence_loss", "log_stft_magnitude_loss") + (("adversarial_loss",) if adversarial else ()) + ("generator_loss",)
        losses = run("g", self.generator_losses_and_grads, g_names)
        self.g.update(self._lr(self.lr_g, self.g.steps), self.world, self.group)
        if adversarial:
            losses.update(run("d", self.discriminator_losses_and_grads, ("real_loss", "fake_loss", "discriminator_loss")))
            self.d.update(self._lr(self.lr_d, self.d.steps), self.world, self.group)
        self.iteration += 1
        return losses
