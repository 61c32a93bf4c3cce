"""What the FastSpeech2 and TransformerTTS training steps share: their set-up (dropout rates, Philox seed, device step counter,
side stream, BatchNorm workspace), materialised multi-head attention forward / backward, the residual sub-layer, the pre-LN
self-attention and feed-forward blocks, the FFT-block stack (Encoder.forward after the embedding) and the Tacotron2 postnet, each
with its saved context.  The FastSpeech2 step runs its encoder and decoder through `stack_fwd` / `stack_bwd`; the TransformerTTS
step its encoder, and its decoder layers are the stack's two blocks around a source attention.

Attention is materialised: S = Q K^T / sqrt(dk) into a (B*H, Tq, ceil64(Tk)) fp32 buffer, the masked softmax, dropout on the
probabilities (pk_dropout, regenerated in the backward), ctx = P V; the backward forms dP = dO V^T, the softmax backward (with the
guided attention loss folded in where requested: pk_softmax_bwd), and dQ = dS K, dK = dS^T Q, dV = P^T dO as pk_conv_gemm NT
matmuls on transposed split planes (pk_transpose_planes).  Q comes from one tensor, K and V from another (column offsets and
leading dimensions free), so the source attention reads the fused K | V memory of every decoder layer in place.

The step classes derive from TransformerTrainOps, a TrainStep (training/flat.py).
"""
import math
import os

import torch

from .. import _lib, ops
from ..ops import Split, _ptr, _stream, ceil_to
from .flat import TrainStep


class TransformerTrainOps(TrainStep):
    def __init__(self, model, dropout, seed, **base):
        """dropout: True -> the model's constructor rates (the reference trains in model.train() mode), a dict of the reference's
        rate keywords to override some, or False / None -> every rate 0 (deterministic step, parity tests).
        seed: base seed of the Philox masks; every rank should pass its own (paddle seeds each process's generator).
        base: TrainStep's arguments."""
        if model.adim > 512:
            raise NotImplementedError("pk_layer_norm_bwd supports rows of at most 512 channels (adim)")
        super().__init__(model, **base)
        self.overlap = os.environ.get("PK_TRAIN_OVERLAP", "1") != "0"      # parameter gradients on a side stream (on_side)
        self._side, self._side_used, self._keep = None, False, []
        if dropout is True:
            self.rates = dict(model.dropout_rates)
        elif isinstance(dropout, dict):
            self.rates = {**model.dropout_rates, **dropout}
        else:
            self.rates = {k: 0.0 for k in model.dropout_rates}
        self.seed = int(seed)
        # completed steps, on the device: the dropout kernels add it to their step argument, so a captured graph of forward +
        # backward draws new masks on every replay
        self.step_dev = torch.zeros(1, dtype=torch.int32, device=self.dev)
        # workspace of the BatchNorm / LayerNorm reductions: 2 floats per channel (pk_batch_norm_train / _bwd)
        widest = max([model.odim, model.adim] + [int(v.shape[0]) for k, v in model._params.items() if k.startswith("postnet.")])
        self.sums = torch.zeros(max(4096, 2 * widest), dtype=torch.float32, device=self.dev)

    def P(self, name):
        return self.m._params[name]

    @staticmethod
    def site(stack, layer, kind):
        """Dropout site: stack * 1000 + layer * 10 + kind (each step documents its numbering; oracle/fastspeech2.py: dropout_site,
        oracle/transformer_tts_train.py: dropout_site)."""
        return stack * 1000 + layer * 10 + kind

    def drop(self, x, p, site, **kw):
        """Forward AND backward: the mask depends only on (seed, step, site, element index)."""
        return ops.dropout(x, p, self.seed, site, 1, step_dev=self.step_dev, **kw)      # step = 1 + completed steps (device counter)

    def layer_fwd(self, x, wname, bname, kind, **kw):
        return self.conv.fwd(x, wname, self.P(wname), linear=kind == "lin", bias=self.P(bname) if bname else None, **kw)

    def layer_bwd(self, dy, x_saved, wname, bname, kind, need_dx=True):
        """dy fp32 (B,T,cout), x_saved split (B,T,cin): writes the grads of weight / bias, returns dx fp32 (B,T,cin)."""
        w, linear = self.P(wname), kind == "lin"
        dys = ops.split_pad8(dy)

        def param_grads():
            if bname:      # from the split copy: dy itself may be the residual-stream gradient, which LayerNorm backward updates in place
                ops.colsum_split_(dys, dy.shape[-1], self.grads[bname])
            self.conv.wgrad(x_saved, dys, w, linear=linear, out=self.grads[wname])

        # the parameter gradients are leaves of the backward graph: they run beside the dx chain (the critical path)
        self.on_side(param_grads, dys, x_saved)
        return self.conv.dgrad(dys, wname, w, linear=linear) if need_dx else None

    def on_side(self, fn, *keep):
        """Run fn() on the side stream, after everything issued so far on the current stream (fork); join_side() is the join.
        The small-batch step is launch / latency bound (~750 kernels of 5-30 us on a few SMs each): the weight-gradient
        transposes, split-K GEMMs and bias sums overlap the activation-gradient chain - in the captured graph they become
        parallel branches.  `keep`: tensors fn reads that were allocated on the current stream - held until the join so that the
        caching allocator (also at capture time) cannot hand their memory to a later tensor while the side branch still reads it."""
        if not self.overlap:
            fn()
            return
        cur = torch.cuda.current_stream()
        if self._side is None:
            self._side = torch.cuda.Stream(device=self.dev)
        self._side.wait_stream(cur)
        self._keep.extend(keep)
        with torch.cuda.stream(self._side):
            fn()
        self._side_used = True

    def join_side(self):
        if self._side_used:
            torch.cuda.current_stream().wait_stream(self._side)
            self._side_used = False
        self._keep.clear()

    def zbuf(self, role, shape):
        """Persistent zero-initialised operand planes of the current batch shape (training/wgrad.py: ZeroPlanes)."""
        return self._zp.get(role, shape, self.dev)

    def wqkv(self, q):
        """The fused Q | K | V projection of layer prefix `q` as one Paddle Linear weight [A, 3A]."""
        return torch.cat([self.P(q + "self_attn.linear_q.weight"), self.P(q + "self_attn.linear_k.weight"),
                          self.P(q + "self_attn.linear_v.weight")], dim=1)

    # ------------------------------------------------------------------------------------------------------------
    # materialised multi-head attention
    # ------------------------------------------------------------------------------------------------------------
    def mha_fwd(self, q, kv, *, heads, dk, q_col0, k_col0, v_col0, key_lens, causal=False, rate=0.0, site=0):
        """q Split (B, Tq, q_ld): head h's query at columns q_col0 + h dk; kv Split (B, Tk, kv_ld): keys at k_col0 + h dk, values at
        v_col0 + h dk; key_lens int32 (B,).  -> (ctx Split (B, Tq, heads dk), saved context for mha_bwd).  dk: a multiple of 64."""
        B, Tq, q_ld = q.hi.shape
        Tk, kv_ld = kv.hi.shape[1], kv.hi.shape[2]
        A = heads * dk
        Tp = ceil_to(Tk, 64)
        s_buf = torch.empty(B * heads, Tq, Tp, dtype=torch.float32, device=q.hi.device)
        q_spec = dict(rows=Tq, cols=q_ld, ld=q_ld, batch_stride=Tq * q_ld, batches=B, bmul=1, hmul=0, col0=q_col0, colh=dk)
        k_spec = dict(rows=Tk, cols=kv_ld, ld=kv_ld, batch_stride=Tk * kv_ld, batches=B, bmul=1, hmul=0, col0=k_col0, colh=dk)
        ops.batched_matmul_nt(q, kv, batch=B, heads=heads, m=Tq, n=Tk, k=dk, a_spec=q_spec, b_spec=k_spec, scale=1.0 / math.sqrt(dk),
                              y_f32=s_buf, y_batch_stride=heads * Tq * Tp, y_head_stride=Tq * Tp, y_ld=Tp)
        p = ops.masked_softmax(s_buf, key_lens, B, heads, Tq, Tk, causal=causal)
        pd = self.drop(p, rate, site, out_f32=False, out_split=True)[1] if rate > 0 else p
        vt = ops.transpose_heads(kv, col0=v_col0, dk=dk, heads=heads, ld_dst=Tp)
        ctx = Split.empty((B, Tq, A), q.hi.device)
        p_spec = dict(rows=Tq, cols=Tp, ld=Tp, batch_stride=Tq * Tp, batches=B * heads, bmul=heads, hmul=1, col0=0, colh=0)
        v_spec = dict(rows=dk, cols=Tp, ld=Tp, batch_stride=dk * Tp, batches=B * heads, bmul=heads, hmul=1, col0=0, colh=0)
        ops.batched_matmul_nt(pd, vt, batch=B, heads=heads, m=Tq, n=dk, k=Tp, a_spec=p_spec, b_spec=v_spec, y_split=ctx,
                              y_batch_stride=Tq * A, y_head_stride=dk, y_ld=A)
        return ctx, dict(q=q, kv=kv, p=p, pd=pd, heads=heads, dk=dk, q_col0=q_col0, k_col0=k_col0, v_col0=v_col0, rate=rate, site=site)

    def mha_bwd(self, dctx_s, S, dq, dkv, guided=None):
        """dctx_s Split (B, Tq, A): gradient w.r.t. mha_fwd's ctx.  Writes dQ into dq (fp32 (B, Tq, >= q_col0 + A)) at mha_fwd's
        q_col0, dK and dV into dkv (fp32 (B, Tk, kv_ld)) at k_col0 / v_col0 (dq may be dkv: the fused Q | K | V).
        guided: None, or dict(heads, layers, ilens, olens, sigma, lam, partials): the guided loss of ops.softmax_bwd."""
        q, kv, p, H, dk = S["q"], S["kv"], S["p"], S["heads"], S["dk"]
        B, Tq, q_ld = q.hi.shape
        Tk, kv_ld = kv.hi.shape[1], kv.hi.shape[2]
        A = H * dk
        Tkp, Tqp = ceil_to(Tk, 64), ceil_to(Tq, 64)
        dev = dctx_s.hi.device
        dq_ld, dkv_ld = dq.shape[-1], dkv.shape[-1]
        dp = torch.zeros(B * H, Tq, Tkp, dtype=torch.float32, device=dev)
        o_spec = dict(rows=Tq, cols=A, ld=A, batch_stride=Tq * A, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
        v_spec = dict(rows=Tk, cols=kv_ld, ld=kv_ld, batch_stride=Tk * kv_ld, batches=B, bmul=1, hmul=0, col0=S["v_col0"], colh=dk)
        ops.batched_matmul_nt(dctx_s, kv, batch=B, heads=H, m=Tq, n=Tk, k=dk, a_spec=o_spec, b_spec=v_spec, y_f32=dp,
                              y_batch_stride=H * Tq * Tkp, y_head_stride=Tq * Tkp, y_ld=Tkp)                  # d(drop(P)) = dO V^T
        if S["rate"] > 0:
            self.drop(dp, S["rate"], S["site"], inplace=True)                                               # -> dP
        ds = ops.softmax_bwd(p, dp, Tk, 1.0 / math.sqrt(dk), guided)                                            # includes the 1/sqrt(dk)
        # K-major operands: (B*H, Tk, Tqp) for dV / dK, (B*H, Tq, Tkp) for dQ
        z_spec = dict(rows=Tk, cols=Tqp, ld=Tqp, batch_stride=Tk * Tqp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
        dq_spec = dict(rows=Tq, cols=Tkp, ld=Tkp, batch_stride=Tq * Tkp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)

        def d_spec(tp):
            return dict(rows=dk, cols=tp, ld=tp, batch_stride=dk * tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)

        def t_sq(src):       # (B*H, Tq, Tkp) -> transposed (B*H, Tk, Tqp)
            dst = self.zbuf("tsq", (B * H, Tk, Tqp))
            ops.transpose_planes(src, z=B * H, rows=Tq, src_zstride=Tq * Tkp, ld_src=Tkp, c0=0, cols=Tk, shift=0, r_out=Tq, dst=dst,
                                 dst_zstride=Tk * Tqp, ld_dst=Tqp)
            return dst

        def t_heads(src, rows, col0):   # (B, rows, ld)[.., col0 + h*dk + d] -> (B*H, dk, ceil64(rows))
            ld_src, tp = src.hi.shape[-1], ceil_to(rows, 64)
            dst = self.zbuf(("th", rows), (B, H, dk, tp))
            for h in range(H):
                ops.transpose_planes(src, z=B, rows=rows, src_zstride=rows * ld_src, ld_src=ld_src, c0=col0 + h * dk, cols=dk, shift=0,
                                     r_out=rows, dst=Split(dst.hi[:, h], dst.lo[:, h]), dst_zstride=H * dk * tp, ld_dst=tp)
            return dst

        pt, dot = t_sq(S["pd"]), t_heads(dctx_s, Tq, 0)                                                    # dV uses the dropped P
        ops.batched_matmul_nt(pt, dot, batch=B, heads=H, m=Tk, n=dk, k=Tqp, a_spec=z_spec, b_spec=d_spec(Tqp), y_f32=dkv[:, :, S["v_col0"]:],
                              y_batch_stride=Tk * dkv_ld, y_head_stride=dk, y_ld=dkv_ld)                  # dV = P^T dO
        kt = t_heads(kv, Tk, S["k_col0"])
        ops.batched_matmul_nt(ds, kt, batch=B, heads=H, m=Tq, n=dk, k=Tkp, a_spec=dq_spec, b_spec=d_spec(Tkp), y_f32=dq[:, :, S["q_col0"]:],
                              y_batch_stride=Tq * dq_ld, y_head_stride=dk, y_ld=dq_ld)                    # dQ = dS K
        dst_, qt = t_sq(ds), t_heads(q, Tq, S["q_col0"])
        ops.batched_matmul_nt(dst_, qt, batch=B, heads=H, m=Tk, n=dk, k=Tqp, a_spec=z_spec, b_spec=d_spec(Tqp), y_f32=dkv[:, :, S["k_col0"]:],
                              y_batch_stride=Tk * dkv_ld, y_head_stride=dk, y_ld=dkv_ld)                  # dK = dS^T Q

    def qkv_bwd(self, q, dqkv, h1, dev):
        """Backward of the fused Q | K | V projection of layer prefix `q` (h1 Split (B, T, A) -> (B, T, 3A)): the weight and bias
        gradients on the side stream, returns d h1 fp32."""
        B, T, ld = dqkv.shape
        A = ld // 3
        dqs = Split.from_f32(dqkv)
        wqkv = self.wqkv(q)

        def qkv_param_grads(q=q, dqkv=dqkv, dqs=dqs, h1=h1, wqkv=wqkv):
            bsum = torch.zeros(ld, dtype=torch.float32, device=dev)
            ops.colsum_(dqkv.reshape(B * T, ld), bsum)
            for j, nm in enumerate(("linear_q", "linear_k", "linear_v")):
                self.grads[q + "self_attn." + nm + ".bias"].copy_(bsum[j * A:(j + 1) * A])
            gw = self.conv.wgrad(h1, dqs, wqkv, linear=True)
            for j, nm in enumerate(("linear_q", "linear_k", "linear_v")):
                self.grads[q + "self_attn." + nm + ".weight"].copy_(gw[:, j * A:(j + 1) * A])

        self.on_side(qkv_param_grads, dqkv, dqs, h1)
        return self.conv.dgrad(dqs, q + "qkv", wqkv, linear=True)

    # ------------------------------------------------------------------------------------------------------------
    # pre-LN blocks (EncoderLayer / DecoderLayer.forward, concat_after=False) with saved context in `c`
    # ------------------------------------------------------------------------------------------------------------
    def sub_fwd(self, ctx, name, x, rate, site, kind="lin"):
        """x + dropout(layer `name`(ctx)): the residual add rides in the GEMM epilogue when there is no dropout."""
        if rate > 0:
            y, _ = self.layer_fwd(ctx, name + ".weight", name + ".bias", kind)
            self.drop(y, rate, site, inplace=True)
            ops.axpy_(1.0, x, y)
            return y
        return self.layer_fwd(ctx, name + ".weight", name + ".bias", kind, residual=x)[0]

    def sub_bwd(self, dx, ctx, name, rate, site, kind="lin"):
        """The gradient at the ctx input of sub_fwd (its weight / bias gradients written)."""
        dsub = self.drop(dx, rate, site)[0] if rate > 0 else dx
        return self.layer_bwd(dsub, ctx, name + ".weight", name + ".bias", kind)

    def attn_fwd(self, x, q, key_lens, c, *, heads, causal, r_attn, r_layer, sid, l):
        """x + dropout(out_proj(self-attention(norm1(x)))) of layer prefix q; dropout sites (sid, l, 1) and (sid, l, 2)."""
        A = x.shape[2]
        c["x0"] = x
        _, c["h1"] = ops.layer_norm(x, self.P(q + "norm1.weight"), self.P(q + "norm1.bias"))
        bqkv = torch.cat([self.P(q + "self_attn.linear_q.bias"), self.P(q + "self_attn.linear_k.bias"), self.P(q + "self_attn.linear_v.bias")])
        _, qkv = self.conv.fwd(c["h1"], q + "qkv", self.wqkv(q), linear=True, bias=bqkv, out_f32=False, out_split=True)
        c["ctx1"], c["a1"] = self.mha_fwd(qkv, qkv, heads=heads, dk=A // heads, q_col0=0, k_col0=A, v_col0=2 * A, key_lens=key_lens,
                                          causal=causal, rate=r_attn, site=self.site(sid, l, 1))
        return self.sub_fwd(c["ctx1"], q + "self_attn.linear_out", x, r_layer, self.site(sid, l, 2))

    def attn_bwd(self, dx, c, q, *, r_layer, sid, l):
        """dx: gradient at attn_fwd's output, updated in place to the gradient at its input."""
        B, T, A = dx.shape
        dctx_s = Split.from_f32(self.sub_bwd(dx, c["ctx1"], q + "self_attn.linear_out", r_layer, self.site(sid, l, 2)))
        dqkv = torch.zeros(B, T, 3 * A, dtype=torch.float32, device=dx.device)
        self.mha_bwd(dctx_s, c["a1"], dqkv, dqkv)
        dh1 = self.qkv_bwd(q, dqkv, c["h1"], dx.device)
        ops.layer_norm_bwd(c["x0"], self.P(q + "norm1.weight"), dh1, dx, True, self.grads[q + "norm1.weight"], self.grads[q + "norm1.bias"])

    def ffn_fwd(self, x, q, norm, c, *, kind, r_layer, sid, l):
        """x + dropout(w_2(dropout(relu(w_1(norm(x)))))) of layer prefix q; kind: "lin" or "conv" (the position-wise layers);
        dropout sites (sid, l, 3) and (sid, l, 4)."""
        c["xf"] = x
        _, c["hf"] = ops.layer_norm(x, self.P(q + norm + ".weight"), self.P(q + norm + ".bias"))
        _, c["u"] = self.layer_fwd(c["hf"], q + "feed_forward.w_1.weight", q + "feed_forward.w_1.bias", kind, act="relu", out_f32=False,
                                   out_split=True)
        c["ud"] = self.drop(c["u"], r_layer, self.site(sid, l, 3), out_f32=False, out_split=True)[1] if r_layer > 0 else c["u"]
        return self.sub_fwd(c["ud"], q + "feed_forward.w_2", x, r_layer, self.site(sid, l, 4), kind)

    def ffn_bwd(self, dx, c, q, norm, *, kind, r_layer, sid, l):
        """dx: gradient at ffn_fwd's output, updated in place to the gradient at its input."""
        du = self.sub_bwd(dx, c["ud"], q + "feed_forward.w_2", r_layer, self.site(sid, l, 4), kind)
        if r_layer > 0:
            self.drop(du, r_layer, self.site(sid, l, 3), inplace=True)
        du_f, _ = ops.relu_bwd(du, c["u"], want_f32=True)
        dh = self.layer_bwd(du_f, c["hf"], q + "feed_forward.w_1.weight", q + "feed_forward.w_1.bias", kind)
        ops.layer_norm_bwd(c["xf"], self.P(q + norm + ".weight"), dh, dx, True, self.grads[q + norm + ".weight"], self.grads[q + norm + ".bias"])

    # ------------------------------------------------------------------------------------------------------------
    # FFT-block stack (Encoder.forward after the embedding) with saved context
    # ------------------------------------------------------------------------------------------------------------
    def stack_fwd(self, x, pre, n_layers, key_lens, *, heads, ffn, sid, r_layer, r_attn):
        """x fp32 (B, T, A) -> (after_norm output fp32, its split planes, saved context).  ffn: "lin" or "conv" (the position-wise
        layers' kind); sid: the stack's dropout-site number; r_layer / r_attn: the sub-layer and attention-probability rates."""
        ctxs = []
        for i in range(n_layers):
            q, c = f"{pre}encoders.{i}.", {}
            x1 = self.attn_fwd(x, q, key_lens, c, heads=heads, causal=False, r_attn=r_attn, r_layer=r_layer, sid=sid, l=i)
            x = self.ffn_fwd(x1, q, "norm2", c, kind=ffn, r_layer=r_layer, sid=sid, l=i)
            ctxs.append(c)
        y, ys = ops.layer_norm(x, self.P(pre + "after_norm.weight"), self.P(pre + "after_norm.bias"), want_f32=True, want_split=True)
        return y, ys, dict(layers=ctxs, x_last=x, pre=pre, n=n_layers, sid=sid, r_layer=r_layer, ffn=ffn)

    def stack_bwd(self, dy, S):
        """dy: gradient w.r.t. the after_norm output (fp32).  Returns the gradient w.r.t. the stack input."""
        pre, sid, r_layer = S["pre"], S["sid"], S["r_layer"]
        dx = torch.empty_like(dy)
        ops.layer_norm_bwd(S["x_last"], self.P(pre + "after_norm.weight"), dy, dx, False, self.grads[pre + "after_norm.weight"],
                           self.grads[pre + "after_norm.bias"])
        for i in reversed(range(S["n"])):
            q, c = f"{pre}encoders.{i}.", S["layers"][i]
            self.ffn_bwd(dx, c, q, "norm2", kind=S["ffn"], r_layer=r_layer, sid=sid, l=i)
            self.attn_bwd(dx, c, q, r_layer=r_layer, sid=sid, l=i)
        return dx

    # ------------------------------------------------------------------------------------------------------------
    # Tacotron2 postnet (tacotron2/decoder.py:144-180): Conv1D -> train-mode BatchNorm1D over all B x T rows (-> tanh but on
    # the last layer) -> Dropout at site (5, i, 6); after = before + postnet(before)
    # ------------------------------------------------------------------------------------------------------------
    def postnet_fwd(self, before, before_split):
        """before fp32 / before_split Split (B, T, odim) -> (after fp32, saved context)."""
        m, L, st, dev = self.m, _lib.lib(), _stream(), self.dev
        rate = self.rates["postnet_dropout_rate"]
        post, h, rows = [], before_split, before.shape[0] * before.shape[1]
        for i in range(m.postnet_layers):
            last = i == m.postnet_layers - 1
            q = f"postnet.postnet.{i}.1."
            conv_out, _ = self.layer_fwd(h, f"postnet.postnet.{i}.0.weight", None, "conv")
            cdim = conv_out.shape[-1]
            y = torch.empty_like(conv_out)
            ysplit = Split.empty(tuple(conv_out.shape), dev) if not last else None
            mean, rstd = torch.empty(cdim, device=dev), torch.empty(cdim, device=dev)
            _lib.check(L.pk_batch_norm_train(_ptr(conv_out), rows, cdim, _ptr(self.P(q + "weight")), _ptr(self.P(q + "bias")), 1e-5,
                                             0 if last else 2, 0.9, _ptr(m._params[q + "_mean"]), _ptr(m._params[q + "_variance"]),
                                             _ptr(self.sums), _ptr(y), _ptr(ysplit.hi) if ysplit else None,
                                             _ptr(ysplit.lo) if ysplit else None, _ptr(mean), _ptr(rstd), st), "pk_batch_norm_train")
            yd = y
            if rate > 0:
                yd, ysplit = self.drop(y, rate, self.site(5, i, 6), out_f32=True, out_split=not last)
            post.append(dict(x=h, conv=conv_out, y=y, yd=yd, mean=mean, rstd=rstd))
            h = ysplit
        after = before.clone()
        if post:
            ops.axpy_(1.0, post[-1]["yd"], after)
        return after, post

    def postnet_bwd(self, g_after, g_before, post):
        """The gradients at `after` and `before` -> the gradient at postnet_fwd's `before` (the postnet's parameter gradients
        written)."""
        L, st = _lib.lib(), _stream()
        rate = self.rates["postnet_dropout_rate"]
        g = g_after
        for i in reversed(range(len(post))):
            last = i == len(post) - 1
            c = post[i]
            q = f"postnet.postnet.{i}.1."
            rows, cdim = c["conv"].shape[0] * c["conv"].shape[1], c["conv"].shape[-1]
            dconv = torch.empty_like(c["conv"])
            if rate > 0:
                g = self.drop(g, rate, self.site(5, i, 6))[0]
            _lib.check(L.pk_batch_norm_bwd(_ptr(c["conv"]), _ptr(g), _ptr(c["y"]), _ptr(c["mean"]), _ptr(c["rstd"]), _ptr(self.P(q + "weight")),
                                           0 if last else 2, rows, cdim, _ptr(self.sums), _ptr(dconv), st), "pk_batch_norm_bwd")
            self.grads[q + "bias"].copy_(self.sums[:cdim])
            self.grads[q + "weight"].copy_(self.sums[cdim:2 * cdim])
            g = self.layer_bwd(dconv, c["x"], f"postnet.postnet.{i}.0.weight", None, "conv")
        if post:
            ops.axpy_(1.0, g_after, g)                         # the residual path of `after`
            ops.axpy_(1.0, g_before, g)                        # the loss on `before` itself
        else:
            g = g_before.clone()
            ops.axpy_(1.0, g_after, g)
        return g
