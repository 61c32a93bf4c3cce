"""The transformer pieces of the training steps: materialised multi-head attention forward / backward and the FFT-block stack
(pre-LN self-attention + position-wise feed-forward, Encoder.forward after the embedding) with its saved context.  The FastSpeech2
step runs its encoder and decoder through `stack_fwd` / `stack_bwd`; the TransformerTTS step its encoder, and its decoder layers
call `mha_fwd` / `mha_bwd` for the causal self-attention and the source attention.

Attention is materialised: S = Q K^T / sqrt(dk) into a (B*H, Tq, ceil64(Tk)) fp32 buffer, the masked softmax, dropout on the
probabilities (pk_dropout, regenerated in the backward), ctx = P V; the backward forms dP = dO V^T, the softmax backward (with the
guided attention loss folded in where requested: pk_softmax_bwd), and dQ = dS K, dK = dS^T Q, dV = P^T dO as pk_conv_gemm NT
matmuls on transposed split planes (pk_transpose_planes).  Q comes from one tensor, K and V from another (column offsets and
leading dimensions free), so the source attention reads the fused K | V memory of every decoder layer in place.

A step class mixes TransformerTrainOps in and provides m (the model), grads (name -> gradient view), conv (ConvOps), seed,
step_dev (device step counter), _zp (ZeroPlanes) and the side-stream state of on_side (_side, _side_used, _keep, overlap).
"""
import math

import torch

from .. import ops
from ..ops import Split, ceil_to


class TransformerTrainOps:
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
    # FFT-block stack (Encoder.forward after the embedding) with saved context
    # ------------------------------------------------------------------------------------------------------------
    def stack_fwd(self, x, pre, n_layers, key_lens, *, heads, ffn, sid, r_layer, r_attn):
        """x fp32 (B, T, A) -> (after_norm output fp32, its split planes, saved context).  ffn: "lin" or "conv" (the position-wise
        layers' kind); sid: the stack's dropout-site number; r_layer / r_attn: the sub-layer and attention-probability rates."""
        A = x.shape[2]
        ctxs = []
        for i in range(n_layers):
            q = f"{pre}encoders.{i}."
            c = dict(x0=x)
            _, c["h1"] = ops.layer_norm(x, self.P(q + "norm1.weight"), self.P(q + "norm1.bias"))
            bqkv = torch.cat([self.P(q + "self_attn.linear_q.bias"), self.P(q + "self_attn.linear_k.bias"), self.P(q + "self_attn.linear_v.bias")])
            _, qkv = self.conv.fwd(c["h1"], q + "qkv", self.wqkv(q), linear=True, bias=bqkv, out_f32=False, out_split=True)
            ctx, c["attn"] = self.mha_fwd(qkv, qkv, heads=heads, dk=A // heads, q_col0=0, k_col0=A, v_col0=2 * A, key_lens=key_lens,
                                          rate=r_attn, site=self.site(sid, i, 1))
            c["ctx"] = ctx
            if r_layer > 0:      # x1 = x + dropout(attention): the residual add cannot ride in the GEMM epilogue any more
                a_out, _ = self.layer_fwd(ctx, q + "self_attn.linear_out.weight", q + "self_attn.linear_out.bias", "lin")
                self.drop(a_out, r_layer, self.site(sid, i, 2), inplace=True)
                ops.axpy_(1.0, x, a_out)
                x1 = a_out
            else:
                x1, _ = self.layer_fwd(ctx, q + "self_attn.linear_out.weight", q + "self_attn.linear_out.bias", "lin", residual=x)
            c["x1"] = x1
            _, c["h2"] = ops.layer_norm(x1, self.P(q + "norm2.weight"), self.P(q + "norm2.bias"))
            _, c["u"] = self.layer_fwd(c["h2"], q + "feed_forward.w_1.weight", q + "feed_forward.w_1.bias", ffn, act="relu", out_f32=False, out_split=True)
            c["ud"] = self.drop(c["u"], r_layer, self.site(sid, i, 3), out_f32=False, out_split=True)[1] if r_layer > 0 else c["u"]
            if r_layer > 0:
                f_out, _ = self.layer_fwd(c["ud"], q + "feed_forward.w_2.weight", q + "feed_forward.w_2.bias", ffn)
                self.drop(f_out, r_layer, self.site(sid, i, 4), inplace=True)
                ops.axpy_(1.0, x1, f_out)
                x = f_out
            else:
                x, _ = self.layer_fwd(c["u"], q + "feed_forward.w_2.weight", q + "feed_forward.w_2.bias", ffn, residual=x1)
            ctxs.append(c)
        y, ys = ops.layer_norm(x, self.P(pre + "after_norm.weight"), self.P(pre + "after_norm.bias"), want_f32=True, want_split=True)
        return y, ys, dict(layers=ctxs, x_last=x, pre=pre, n=n_layers, sid=sid, r_layer=r_layer, ffn=ffn)

    def stack_bwd(self, dy, S):
        """dy: gradient w.r.t. the after_norm output (fp32).  Returns the gradient w.r.t. the stack input."""
        pre = S["pre"]
        B, T, A = dy.shape
        dev = dy.device
        kind = S["ffn"]
        dx = torch.empty_like(dy)
        ops.layer_norm_bwd(S["x_last"], self.P(pre + "after_norm.weight"), dy, dx, False, self.grads[pre + "after_norm.weight"],
                           self.grads[pre + "after_norm.bias"])
        sid, r_layer = S["sid"], S["r_layer"]
        for i in reversed(range(S["n"])):
            q = f"{pre}encoders.{i}."
            c = S["layers"][i]
            # x2 = x1 + drop(conv2(drop(relu(conv1(LN2(x1))))))
            dsub = self.drop(dx, r_layer, self.site(sid, i, 4))[0] if r_layer > 0 else dx
            du = self.layer_bwd(dsub, c["ud"], q + "feed_forward.w_2.weight", q + "feed_forward.w_2.bias", kind)
            if r_layer > 0:
                self.drop(du, r_layer, self.site(sid, i, 3), inplace=True)
            du_f, _ = ops.relu_bwd(du, c["u"], want_f32=True)
            dh2 = self.layer_bwd(du_f, c["h2"], q + "feed_forward.w_1.weight", q + "feed_forward.w_1.bias", kind)
            ops.layer_norm_bwd(c["x1"], self.P(q + "norm2.weight"), dh2, dx, True, self.grads[q + "norm2.weight"], self.grads[q + "norm2.bias"])
            # x1 = x0 + drop(out_proj(attention(LN1(x0))))
            dsub = self.drop(dx, r_layer, self.site(sid, i, 2))[0] if r_layer > 0 else dx
            dctx = self.layer_bwd(dsub, c["ctx"], q + "self_attn.linear_out.weight", q + "self_attn.linear_out.bias", "lin")
            dctx_s = Split.from_f32(dctx)
            dqkv = torch.zeros(B, T, 3 * A, dtype=torch.float32, device=dev)
            self.mha_bwd(dctx_s, c["attn"], dqkv, dqkv)
            dh1 = self.qkv_bwd(q, dqkv, c["h1"], dev)
            ops.layer_norm_bwd(c["x0"], self.P(q + "norm1.weight"), dh1, dx, True, self.grads[q + "norm1.weight"], self.grads[q + "norm1.bias"])
        return dx
