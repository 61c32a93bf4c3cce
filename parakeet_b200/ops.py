"""Torch-tensor level wrappers over the C-ABI (device memory + streams are torch's; all math is in the .so)."""
import ctypes as C
import math

import torch

from . import _lib
from ._lib import PK_ACT_NONE, PK_ACT_RELU, PK_ACT_TANH, ConvGemmArgs, Operand  # noqa: F401

ACTS = {None: PK_ACT_NONE, "none": PK_ACT_NONE, "relu": PK_ACT_RELU, "tanh": PK_ACT_TANH}


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _require_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise _lib.PkError("parakeet_b200 ops need CUDA tensors (no CPU fallback)")


class Split:
    """split-bf16 tensor: value = hi + lo (two bf16 planes of identical shape / strides)."""

    __slots__ = ("hi", "lo")

    def __init__(self, hi, lo):
        assert hi.dtype == torch.bfloat16 and lo.dtype == torch.bfloat16 and hi.shape == lo.shape
        self.hi, self.lo = hi, lo

    @property
    def shape(self):
        return self.hi.shape

    # Both planes come from ONE allocation, lo right after hi: kernels that stream a tile of both planes can then fetch them
    # with a single 4-D TMA box (the plane is the outermost dimension; csrc/pwg_fc.cu) instead of two loads.
    @staticmethod
    def empty(shape, device):
        buf = torch.empty((2,) + tuple(shape), dtype=torch.bfloat16, device=device)
        return Split(buf[0], buf[1])

    @staticmethod
    def zeros(shape, device):
        buf = torch.zeros((2,) + tuple(shape), dtype=torch.bfloat16, device=device)
        return Split(buf[0], buf[1])

    @staticmethod
    def from_f32(x):
        """fp32 CUDA tensor -> split planes (pk_split_f32)."""
        _require_cuda(x)
        x = x.contiguous().float()
        out = Split.empty(x.shape, x.device)
        _lib.check(_lib.lib().pk_split_f32(_ptr(x), _ptr(out.hi), _ptr(out.lo), x.numel(), _stream()), "pk_split_f32")
        return out

    def float(self):
        return self.hi.float() + self.lo.float()


def pack_weight(w, device=None):
    """Conv1D weight [out, in, k] (Paddle/torch layout) or Linear weight given as [out, in] ->
    K-major GEMM operand [out, k * Kp] (tap-major, each tap's channels zero-padded to a multiple of 64), split-bf16.
    Host-side, done once at load time."""
    w = w.detach().float().cpu()
    if w.dim() == 2:
        w = w.unsqueeze(-1)
    n, k, taps = w.shape
    kp = (k + 63) // 64 * 64
    packed = torch.zeros(n, taps, kp, dtype=torch.float32)
    packed[:, :, :k] = w.permute(0, 2, 1)
    packed = packed.reshape(n, taps * kp)
    hi = packed.to(torch.bfloat16)
    lo = (packed - hi.float()).to(torch.bfloat16)
    dev = device or "cuda"
    return Split(hi.to(dev).contiguous(), lo.to(dev).contiguous())


def ceil_to(n, m):
    return (n + m - 1) // m * m


def pack_dev(w):
    """[n, k, taps] (or [n, k]) fp32 CUDA tensor -> K-major split planes [n, taps * Kp] (pack_weight on the device: the training
    steps pack the weights of every step)."""
    if w.dim() == 2:
        w = w.unsqueeze(-1)
    n, k, taps = w.shape
    kp = ceil_to(k, 64)
    packed = torch.zeros(n, taps, kp, dtype=torch.float32, device=w.device)
    packed[:, :, :k] = w.permute(0, 2, 1)
    return Split.from_f32(packed.reshape(n, taps * kp))


def pad8(t):
    """(..., C) -> (..., ceil_to(C, 8)) zero padded: TMA row pitches are multiples of 16 bytes."""
    c = t.shape[-1]
    if c % 8 == 0:
        return t.contiguous()
    out = torch.zeros(t.shape[:-1] + (ceil_to(c, 8),), dtype=t.dtype, device=t.device)
    out[..., :c] = t
    return out


def split_pad8(dy):
    """fp32 gradient (..., C) -> its split planes, the channel axis padded to a multiple of 8 (a GEMM operand)."""
    return Split.from_f32(pad8(dy))


def _operand(s, rows, cols, ld, batch_stride, batches, bmul=1, hmul=0, col0=0, colh=0):
    return Operand(hi=s.hi.data_ptr(), lo=s.lo.data_ptr(), batch_stride=batch_stride, ld=ld, rows=rows, cols=cols,
                   batches=batches, bmul=bmul, hmul=hmul, col0=col0, colh=colh)


def conv_gemm(a, w, *, n, k, taps=1, dil=1, pad=None, bias=None, act=None, residual=None, lens=None, scale=1.0,
              out_f32=True, out_split=False, passes=3, simt=False, y_f32=None, y_split=None, epilogue=None):
    """Channels-last Conv1D / Linear.  a: Split (B, T, C_total); w: packed weight Split [n, taps*Kp].

    Returns (y_f32 or None, y_split or None), each (B, T, n).
    `epilogue` selects a fused pair epilogue of pk_conv_gemm_ex (n == 2 * C, the GEMM result itself is not written):
      dict(mode="gate", channels=C, residual=(tensor (B, T, >= 2C) fp32 view with last stride 1) or None) -> y_split (B, T, C)
      dict(mode="wf_update", channels=C, state=, skip=, skip_init=bool, buf=Split or None, buf_col0=int)
    """
    _require_cuda(a.hi, w.hi)
    B, T, Ctot = a.hi.shape
    if pad is None:
        pad = (taps - 1) // 2
    dev = a.hi.device
    if epilogue is not None:
        out_f32 = False
        out_split = False
        y_f32 = None
        if epilogue["mode"] == "gate" and y_split is None:
            y_split = Split.empty((B, T, epilogue["channels"]), dev)
    if out_f32 and y_f32 is None:
        y_f32 = torch.empty(B, T, n, dtype=torch.float32, device=dev)
    if out_split and y_split is None:
        y_split = Split.empty((B, T, n), dev)
    args = ConvGemmArgs()
    # A's extent ends at k: the last 64-column K chunk is zero-filled past it instead of reading columns the weight has no
    # taps for (a zero weight times a NaN or Inf there would still poison the output)
    args.a = _operand(a, rows=T, cols=min(Ctot, k), ld=a.hi.stride(1), batch_stride=a.hi.stride(0), batches=B)
    args.b = _operand(w, rows=w.hi.shape[0], cols=w.hi.shape[1], ld=w.hi.stride(0), batch_stride=0, batches=1, bmul=0)
    args.batch, args.heads, args.m, args.n, args.k = B, 1, T, n, k
    args.taps, args.dil, args.pad = taps, dil, pad
    args.scale = scale
    args.bias = bias.data_ptr() if bias is not None else None
    args.act = ACTS[act]
    args.residual = residual.data_ptr() if residual is not None else None
    args.lens = lens.data_ptr() if lens is not None else None
    args.y_f32 = y_f32.data_ptr() if y_f32 is not None else None
    args.y_hi = y_split.hi.data_ptr() if y_split is not None else None
    args.y_lo = y_split.lo.data_ptr() if y_split is not None else None
    args.y_batch_stride, args.y_head_stride, args.y_ld = T * n, 0, n
    args.passes = passes
    if epilogue is not None:
        ep = _lib.GemmEpilogue()
        Cc = int(epilogue["channels"])
        ep.channels = Cc
        if epilogue["mode"] == "gate":
            ep.mode = _lib.PK_EPI_GATE
            args.y_batch_stride, args.y_ld = T * y_split.hi.stride(1), y_split.hi.stride(1)
            res = epilogue.get("residual")
            if res is not None:
                assert res.dtype == torch.float32 and res.stride(-1) == 1 and res.shape[0] == B and res.shape[1] == T
                ep.residual, ep.residual_batch_stride, ep.residual_ld = res.data_ptr(), res.stride(0), res.stride(1)
        else:
            ep.mode = _lib.PK_EPI_WF_UPDATE
            state, skip = epilogue["state"], epilogue["skip"]
            assert state.is_contiguous() and skip.is_contiguous() and tuple(state.shape) == (B, T, Cc) == tuple(skip.shape)
            ep.state, ep.skip, ep.skip_init = state.data_ptr(), skip.data_ptr(), 1 if epilogue.get("skip_init") else 0
            buf = epilogue.get("buf")
            if buf is not None:
                assert buf.hi.is_contiguous() and buf.hi.shape[0] == B and buf.hi.shape[1] == T
                ep.buf_hi, ep.buf_lo, ep.buf_ld, ep.buf_col0 = buf.hi.data_ptr(), buf.lo.data_ptr(), buf.hi.stride(1), int(epilogue.get("buf_col0", 0))
        _lib.check(_lib.lib().pk_conv_gemm_ex(C.byref(args), C.byref(ep), _stream()), "pk_conv_gemm_ex")
        return None, y_split
    fn = _lib.lib().pk_conv_gemm_simt if simt else _lib.lib().pk_conv_gemm
    _lib.check(fn(C.byref(args), _stream()), "pk_conv_gemm")
    return y_f32, y_split


def k_tail_overlap(spec, heads, k):
    """First head whose K slice [col0 + h * colh, + k) is followed, up to the next multiple of 64 columns, by columns inside
    the operand's `cols`, or None.  pk_conv_gemm loads K in 64-column chunks bounded only by `cols`, so such columns would
    enter the product (the SIMT path stops at k: the two paths would disagree)."""
    if k % 64 == 0:
        return None
    for h in range(heads):
        end = spec.get("col0", 0) + h * spec.get("colh", 0) + k
        if end < spec["cols"]:
            return h
    return None


def batched_matmul_nt(a, b, *, batch, heads, m, n, k, a_spec, b_spec, scale=1.0, y_f32=None, y_split=None,
                      y_batch_stride=None, y_head_stride=None, y_ld=None, lens=None, passes=3, simt=False):
    """y[b,h] = scale * A[b,h] (m x k) . B[b,h]^T (n x k); operand addressing given by a_spec / b_spec dicts
    (rows, cols, ld, batch_stride, batches, bmul, hmul, col0, colh).  With k % 64 != 0 each operand's K slice must end at
    its `cols` (k_tail_overlap): a head slice followed by live columns is refused."""
    for name, spec in (("A", a_spec), ("B", b_spec)):
        h = k_tail_overlap(spec, heads, k)
        if h is not None:
            raise _lib.PkError(f"batched_matmul_nt: k={k} is not a multiple of 64 and operand {name}'s K slice of head {h} is followed "
                               f"by live columns (col0={spec.get('col0', 0)}, colh={spec.get('colh', 0)}, cols={spec['cols']})")
    args = ConvGemmArgs()
    args.a = _operand(a, **a_spec)
    args.b = _operand(b, **b_spec)
    args.batch, args.heads, args.m, args.n, args.k = batch, heads, m, n, k
    args.taps, args.dil, args.pad = 1, 1, 0
    args.scale = scale
    args.act = PK_ACT_NONE
    args.lens = lens.data_ptr() if lens is not None else None
    args.y_f32 = y_f32.data_ptr() if y_f32 is not None else None
    args.y_hi = y_split.hi.data_ptr() if y_split is not None else None
    args.y_lo = y_split.lo.data_ptr() if y_split is not None else None
    args.y_batch_stride, args.y_head_stride, args.y_ld = y_batch_stride, y_head_stride, y_ld
    args.passes = passes
    fn = _lib.lib().pk_conv_gemm_simt if simt else _lib.lib().pk_conv_gemm
    _lib.check(fn(C.byref(args), _stream()), "pk_conv_gemm")


def length_regulator_lens(dur):
    """dur: int64 (B, T) CUDA -> int32 (B,) total frames per utterance (device tensor, no sync)."""
    _require_cuda(dur)
    dur = dur.contiguous()
    B, T = dur.shape
    out = torch.empty(B, dtype=torch.int32, device=dur.device)
    _lib.check(_lib.lib().pk_length_regulator_lens(_ptr(dur), B, T, _ptr(out), _stream()), "pk_length_regulator_lens")
    return out


def length_regulate(x, dur, t_out, want_f32=True, want_split=False):
    """x fp32 (B, T, C), dur int64 (B, T) -> (B, t_out, C) repeat-expanded; rows past sum(d) are zero."""
    _require_cuda(x, dur)
    x = x.contiguous()
    dur = dur.contiguous()
    B, T, Cc = x.shape
    y = torch.empty(B, t_out, Cc, dtype=torch.float32, device=x.device) if want_f32 else None
    ys = Split.empty((B, t_out, Cc), x.device) if want_split else None
    if t_out == 0:   # every duration is zero: empty output, as in the reference (t_dec = 0)
        return y, ys
    _lib.check(_lib.lib().pk_length_regulate(_ptr(x), _ptr(dur), B, T, Cc, t_out, _ptr(y),
                                             _ptr(ys.hi) if ys else None, _ptr(ys.lo) if ys else None, _stream()),
               "pk_length_regulate")
    return y, ys


# ----------------------------------------------------------------------------------------------------------------
# FastSpeech2 row-wise kernels
# ----------------------------------------------------------------------------------------------------------------
def embed_pe(ids, table, x_in, alpha, lens, padding_idx=0):
    """Embedding(padding_idx)+ScaledPositionalEncoding (ids given) or ScaledPositionalEncoding only (x_in given)."""
    if ids is not None:
        B, T = ids.shape
        d = table.shape[1]
        dev = ids.device
        ids = ids.contiguous()
    else:
        B, T, d = x_in.shape
        dev = x_in.device
        x_in = x_in.contiguous()
    y = torch.empty(B, T, d, dtype=torch.float32, device=dev)
    _lib.check(_lib.lib().pk_embed_pe(_ptr(ids), _ptr(table), table.shape[0] if table is not None else 0, padding_idx,
                                      _ptr(x_in), _ptr(alpha), _ptr(lens), B, T, d, _ptr(y), _stream()), "pk_embed_pe")
    return y


def layer_norm(x, gamma, beta, lens=None, want_f32=False, want_split=True, eps=1e-5):
    B, T, d = x.shape
    y = torch.empty_like(x) if want_f32 else None
    ys = Split.empty((B, T, d), x.device) if want_split else None
    _lib.check(_lib.lib().pk_layer_norm(_ptr(x), _ptr(gamma), _ptr(beta), eps, _ptr(lens), B, T, d, _ptr(y),
                                        _ptr(ys.hi) if ys else None, _ptr(ys.lo) if ys else None, _stream()), "pk_layer_norm")
    return y, ys


def masked_softmax(s, key_lens, batch, heads, rows, keys, causal=False):
    """s fp32 (batch*heads, rows, ld) -> split planes of the same shape; causal adds the j <= i mask."""
    ld = s.shape[-1]
    p = Split.empty(tuple(s.shape), s.device)
    _lib.check(_lib.lib().pk_masked_softmax(_ptr(s), _ptr(key_lens), batch, heads, rows, keys, ld, 1 if causal else 0, _ptr(p.hi),
                                            _ptr(p.lo), _stream()), "pk_masked_softmax")
    return p


def transpose_heads(src, col0, dk, heads, ld_dst):
    B, T, ld_src = src.hi.shape
    dst = Split.empty((B * heads, dk, ld_dst), src.hi.device)
    _lib.check(_lib.lib().pk_transpose_heads(_ptr(src.hi), _ptr(src.lo), B, T, ld_src, col0, dk, heads, ld_dst, _ptr(dst.hi),
                                             _ptr(dst.lo), _stream()), "pk_transpose_heads")
    return dst


def l2_normalize_axis1(x, eps=1e-12):
    """paddle F.normalize(x) (p=2, axis=1): (B, D) over D; (B, T, D) over T (the reference's batched tone path)."""
    x = x.contiguous().float()
    outer, n = x.shape[0], x.shape[1]
    inner = x.numel() // (outer * n)
    y = torch.empty_like(x)
    _lib.check(_lib.lib().pk_l2_normalize(_ptr(x), outer, n, inner, float(eps), _ptr(y), _stream()), "pk_l2_normalize")
    return y


def fused_attention(qkv, heads, key_lens=None, row_lens=None, ctx=None):
    """qkv Split (B, T, 3A) -> ctx Split (B, T, A): softmax(q k^T / sqrt(d_k), key mask) v per head, one kernel
    (pk_fused_attention) after the per-head transpose of v."""
    B, T, ld = qkv.hi.shape
    A = ld // 3
    dk = A // heads
    Tp = (T + 63) // 64 * 64
    vt = transpose_heads(qkv, col0=2 * A, dk=dk, heads=heads, ld_dst=Tp)
    if ctx is None:
        ctx = Split.empty((B, T, A), qkv.hi.device)
    _lib.check(_lib.lib().pk_fused_attention(_ptr(qkv.hi), _ptr(qkv.lo), _ptr(vt.hi), _ptr(vt.lo), B, T, heads, dk, Tp, _ptr(key_lens),
                                             _ptr(row_lens), 1.0 / math.sqrt(dk), _ptr(ctx.hi), _ptr(ctx.lo), _stream()),
               "pk_fused_attention")
    return ctx


def fused_attention_ex(q, k, *, heads, q_col0, k_col0, v_col0, key_lens=None, row_lens=None, causal=False, ctx=None):
    """pk_fused_attention_ex: ctx Split (B, T_q, heads d_k) = softmax(q k^T / sqrt(d_k), key mask[, causal]) v per head, with Q at
    columns q_col0 + h d_k of the Split q (B, T_q, ·) and K / V at columns k_col0 / v_col0 + h d_k of the Split k (B, T_k, ·)."""
    B, Tq, q_ld = q.hi.shape
    Tk, k_ld = k.hi.shape[1], k.hi.shape[2]
    dk = ctx.hi.shape[2] // heads                    # ctx (B, T_q, heads d_k) is given: its width fixes d_k
    Tp = (Tk + 63) // 64 * 64
    vt = transpose_heads(k, col0=v_col0, dk=dk, heads=heads, ld_dst=Tp)
    a = _lib.AttentionArgs()
    a.q_hi, a.q_lo, a.k_hi, a.k_lo, a.vt_hi, a.vt_lo = (t.data_ptr() for t in (q.hi, q.lo, k.hi, k.lo, vt.hi, vt.lo))
    a.batch, a.t_q, a.t_k, a.heads, a.dk, a.tp, a.q_ld, a.k_ld = B, Tq, Tk, heads, dk, Tp, q_ld, k_ld
    a.q_col0, a.k_col0, a.causal = q_col0, k_col0, 1 if causal else 0
    a.key_lens, a.row_lens = _ptr(key_lens).value, _ptr(row_lens).value
    a.scale = 1.0 / math.sqrt(dk)
    a.ctx_hi, a.ctx_lo = ctx.hi.data_ptr(), ctx.lo.data_ptr()
    _lib.check(_lib.lib().pk_fused_attention_ex(C.byref(a), _stream()), "pk_fused_attention_ex")
    return ctx


def duration_post(x, lens, offset=1.0):
    B, T = x.shape
    x = x.contiguous()
    d_f = torch.empty(B, T, dtype=torch.float32, device=x.device)
    d_i = torch.empty(B, T, dtype=torch.int64, device=x.device)
    _lib.check(_lib.lib().pk_duration_post(_ptr(x), _ptr(lens), B, T, offset, _ptr(d_f), _ptr(d_i), _stream()),
               "pk_duration_post")
    return d_f, d_i


def duration_scale(d, alpha):
    d = d.contiguous()
    out = torch.empty_like(d)
    _lib.check(_lib.lib().pk_duration_scale(_ptr(d), alpha, d.numel(), _ptr(out), _stream()), "pk_duration_scale")
    return out


def mask_rows_(x, lens):
    B, T = x.shape[:2]
    inner = x.numel() // (B * T)
    _lib.check(_lib.lib().pk_mask_rows(_ptr(x), _ptr(lens), B, T, inner, _stream()), "pk_mask_rows")
    return x


def variance_embed_add(hs, pitch, energy, wp, bp, we, be, lens=None):
    B, T, c = hs.shape
    hs, pitch, energy = hs.contiguous(), pitch.contiguous(), energy.contiguous()   # locals: must outlive the launch call
    y = torch.empty_like(hs)
    _lib.check(_lib.lib().pk_variance_embed_add(_ptr(hs), _ptr(pitch), _ptr(energy), _ptr(wp), _ptr(bp),
                                                wp.shape[-1], _ptr(we), _ptr(be), we.shape[-1], _ptr(lens), B, T, c, _ptr(y),
                                                _stream()), "pk_variance_embed_add")
    return y


def ss_residual_block(x, xs, convs, taps, pad_left, lens=None):
    """SpeedySpeech ResidualBlock (pk_ss_residual_block): x fp32 (B, T, 128) and its Split xs -> (y fp32, y Split).
    convs: one or two dicts(w=packed Split, b=bias, s=BN scale, t=BN shift), each fp32 [128] on the device."""
    _require_cuda(x, xs.hi)
    B, T, Cc = x.shape
    y = torch.empty_like(x)
    ys = Split.empty((B, T, Cc), x.device)
    a = _lib.SsResidualBlockArgs()
    a.batch, a.t, a.channels, a.n_convs, a.taps, a.pad_left = B, T, Cc, len(convs), taps, pad_left
    a.lens = lens.data_ptr() if lens is not None else None
    a.x, a.x_hi, a.x_lo = x.data_ptr(), xs.hi.data_ptr(), xs.lo.data_ptr()
    c1 = convs[0]
    a.w1_hi, a.w1_lo, a.bias1, a.scale1, a.shift1 = c1["w"].hi.data_ptr(), c1["w"].lo.data_ptr(), c1["b"].data_ptr(), \
        c1["s"].data_ptr(), c1["t"].data_ptr()
    if len(convs) == 2:
        c2 = convs[1]
        a.w2_hi, a.w2_lo, a.bias2, a.scale2, a.shift2 = c2["w"].hi.data_ptr(), c2["w"].lo.data_ptr(), c2["b"].data_ptr(), \
            c2["s"].data_ptr(), c2["t"].data_ptr()
    a.y, a.y_hi, a.y_lo = y.data_ptr(), ys.hi.data_ptr(), ys.lo.data_ptr()
    _lib.check(_lib.lib().pk_ss_residual_block(C.byref(a), _stream()), "pk_ss_residual_block")
    return y, ys


def relu_split(x):
    """ReLU of an fp32 tensor into split planes (pk_leaky_relu with slope 0)."""
    _require_cuda(x)
    x = x.contiguous()
    ys = Split.empty(tuple(x.shape), x.device)
    _lib.check(_lib.lib().pk_leaky_relu(_ptr(x), x.numel(), 0.0, None, _ptr(ys.hi), _ptr(ys.lo), _stream()), "pk_leaky_relu")
    return ys


def zscore(x, mu, sigma, inverse=False):
    x = x.contiguous().float()
    y = torch.empty_like(x)
    _lib.check(_lib.lib().pk_zscore(_ptr(x), _ptr(mu), _ptr(sigma), x.shape[-1], x.numel(), 1 if inverse else 0, _ptr(y), _stream()),
               "pk_zscore")
    return y


# ----------------------------------------------------------------------------------------------------------------
# training-step helpers (train.cu)
# ----------------------------------------------------------------------------------------------------------------
def transpose_planes(src, *, z, rows, src_zstride, ld_src, c0, cols, shift, r_out, dst, dst_zstride, ld_dst):
    """dst[z*dst_zstride + c*ld_dst + r] = src[z*src_zstride + (r+shift)*ld_src + c0 + c]; src / dst are Split (views allowed)."""
    _lib.check(_lib.lib().pk_transpose_planes(_ptr(src.hi), _ptr(src.lo), z, rows, src_zstride, ld_src, c0, cols, shift, r_out,
                                              _ptr(dst.hi), _ptr(dst.lo), dst_zstride, ld_dst, _stream()), "pk_transpose_planes")


def layer_norm_bwd(x, gamma, dy, dx, accumulate, dgamma, dbeta, eps=1e-5):
    rows, d = x.numel() // x.shape[-1], x.shape[-1]
    _lib.check(_lib.lib().pk_layer_norm_bwd(_ptr(x), _ptr(gamma), _ptr(dy), eps, rows, d, _ptr(dx), 1 if accumulate else 0,
                                            _ptr(dgamma), _ptr(dbeta), _stream()), "pk_layer_norm_bwd")


def softmax_bwd(p, dp, keys, scale, guided=None):
    """pk_softmax_bwd: p split planes, dp fp32 (..., rows, ld) -> dS split planes of the same shape.  guided: None, or
    dict(heads, layers, ilens, olens, sigma, lam, partials) to fold the guided attention loss into heads h < guided["heads"] of
    a (batch * heads, rows, ld) layout, batch = ilens.numel(); the loss's row partials (batch, guided["heads"], rows) go to
    `partials` (a contiguous fp32 view)."""
    rows, ld = (dp.shape[-2] if dp.dim() > 1 else 1), dp.shape[-1]
    z = dp.numel() // (rows * ld)
    ds = Split.empty(tuple(dp.shape), dp.device)
    g = guided or dict(heads=0, layers=1, ilens=None, olens=None, sigma=1.0, lam=0.0, partials=None)
    batch = g["ilens"].numel() if guided else z
    if z % batch:
        raise ValueError(f"softmax_bwd: {z} (batch * heads) rows of attention for {batch} utterances")
    _lib.check(_lib.lib().pk_softmax_bwd(_ptr(p.hi), _ptr(p.lo), _ptr(dp), batch, z // batch, rows, keys, ld, float(scale), g["heads"],
                                         g["layers"], _ptr(g["ilens"]), _ptr(g["olens"]), float(g["sigma"]), float(g["lam"]),
                                         _ptr(g["partials"]), _ptr(ds.hi), _ptr(ds.lo), _stream()), "pk_softmax_bwd")
    return ds


def colsum_(x, out):
    c = x.shape[-1]
    _lib.check(_lib.lib().pk_colsum(_ptr(x), x.numel() // c, c, _ptr(out), _stream()), "pk_colsum")


def colsum_split_(xs, cols, out):
    """out[c] += sum over all rows of (hi + lo)[..., c], c < cols, for a contiguous Split (..., ld)."""
    ld = xs.hi.shape[-1]
    assert xs.hi.is_contiguous() and cols <= ld
    _lib.check(_lib.lib().pk_colsum_split(_ptr(xs.hi), _ptr(xs.lo), xs.hi.numel() // ld, cols, ld, _ptr(out), _stream()), "pk_colsum_split")


def sum_slices(part, out):
    """out = part.sum(0) for fp32 part (S, ...) and contiguous out (split-K reduction; overwrites out)."""
    s = part.shape[0]
    assert part.is_contiguous() and out.is_contiguous() and part.numel() == s * out.numel()
    _lib.check(_lib.lib().pk_sum_slices(_ptr(part), s, out.numel(), _ptr(out), _stream()), "pk_sum_slices")
    return out


def relu_bwd(dy, y_split, want_f32=False):
    dx = torch.empty_like(dy) if want_f32 else None
    dxs = Split.empty(tuple(dy.shape), dy.device)
    _lib.check(_lib.lib().pk_relu_bwd(_ptr(dy), _ptr(y_split.hi), dy.numel(), _ptr(dx), _ptr(dxs.hi), _ptr(dxs.lo), _stream()), "pk_relu_bwd")
    return dx, dxs


def axpy_(a, x, y):
    _lib.check(_lib.lib().pk_axpy(float(a), _ptr(x), x.numel(), _ptr(y), _stream()), "pk_axpy")


def spk_embed_fwd(table, ids, padding_idx=0, eps=1e-12):
    """Speaker-table lookup + F.normalize (pk_spk_embed_fwd): table fp32 (N, D), ids int64 (B,) on the device ->
    (e fp32 (B, D), norms fp32 (B,) for spk_normalize_bwd)."""
    _require_cuda(table, ids)
    table, ids = table.contiguous(), ids.contiguous()
    B, (N, D) = ids.numel(), table.shape
    e = torch.empty(B, D, dtype=torch.float32, device=table.device)
    norms = torch.empty(B, dtype=torch.float32, device=table.device)
    _lib.check(_lib.lib().pk_spk_embed_fwd(_ptr(table), N, D, _ptr(ids), B, padding_idx, float(eps), _ptr(e), _ptr(norms), _stream()),
               "pk_spk_embed_fwd")
    return e, norms


def spk_time_sum(dx, col0, ncols, dhs_cols=0):
    """dx fp32 (B, T, C) -> (sum over all T rows of dx[..., col0:col0 + ncols] (B, ncols), dx[..., :dhs_cols] contiguous or None)."""
    _require_cuda(dx)
    assert dx.is_contiguous() and dx.dtype == torch.float32
    B, T, Cc = dx.shape
    out = torch.empty(B, ncols, dtype=torch.float32, device=dx.device)
    dhs = torch.empty(B, T, dhs_cols, dtype=torch.float32, device=dx.device) if dhs_cols else None
    _lib.check(_lib.lib().pk_spk_time_sum(_ptr(dx), B, T, Cc, col0, ncols, _ptr(dhs), dhs_cols, _ptr(out), _stream()), "pk_spk_time_sum")
    return out, dhs


def spk_normalize_bwd(e, norms, g, ids, num_speakers, padding_idx=0, eps=1e-12):
    """Backward of spk_embed_fwd's normalisation: (B, D) gradient w.r.t. the looked-up table rows (zeros for padding ids)."""
    B, D = e.shape
    dx = torch.empty_like(e)
    _lib.check(_lib.lib().pk_spk_normalize_bwd(_ptr(e), _ptr(norms), _ptr(g), _ptr(ids), B, num_speakers, padding_idx, D, float(eps),
                                               _ptr(dx), _stream()), "pk_spk_normalize_bwd")
    return dx


def spk_table_grad(de, ids, out, padding_idx=0):
    """Dense table gradient (pk_spk_table_grad) written into out (N, D), e.g. a view of a flat gradient buffer."""
    assert out.is_contiguous() and de.is_contiguous()
    N, D = out.shape
    _lib.check(_lib.lib().pk_spk_table_grad(_ptr(de), _ptr(ids), ids.numel(), N, D, padding_idx, _ptr(out), _stream()), "pk_spk_table_grad")
    return out


def ss_scratch_elems(rows, batch=0, l=0, odim=0):
    """fp32 elements of workspace the SpeedySpeech training kernels need for `rows` BatchNorm rows and a (batch, l, odim) loss."""
    return max(256 * ((rows + 127) // 128), 2 * batch * ((l + 15) // 16) + 3 * batch * l * odim, 256)


def ss_bn_train_fwd(r, gamma, beta, run_mean, run_var, scratch, residual=None, want_f32=True, want_split=True, eps=1e-5, momentum=0.9):
    """Train-mode BatchNorm1D on r fp32 (..., 128) (pk_ss_bn_train_fwd) -> (y fp32 or None, y Split or None, mean, rstd);
    run_mean / run_var are updated in place, residual (same shape as r) is added to y."""
    _require_cuda(r, gamma, beta, scratch)
    assert r.is_contiguous() and (residual is None or residual.is_contiguous())
    c = r.shape[-1]
    rows = r.numel() // c
    y = torch.empty_like(r) if want_f32 else None
    ys = Split.empty(tuple(r.shape), r.device) if want_split else None
    mean = torch.empty(c, dtype=torch.float32, device=r.device)
    rstd = torch.empty(c, dtype=torch.float32, device=r.device)
    _lib.check(_lib.lib().pk_ss_bn_train_fwd(_ptr(r), rows, c, _ptr(gamma), _ptr(beta), eps, momentum, _ptr(run_mean), _ptr(run_var),
                                             _ptr(residual), _ptr(scratch), _ptr(y), _ptr(ys.hi if ys else None),
                                             _ptr(ys.lo if ys else None), _ptr(mean), _ptr(rstd), _stream()), "pk_ss_bn_train_fwd")
    return y, ys, mean, rstd


def ss_bn_relu_bwd(dy, r, mean, rstd, gamma, scratch, dgamma, dbeta, dbias=None, want_f32=False, want_split=True):
    """Backward of ReLU -> train-mode BatchNorm1D (pk_ss_bn_relu_bwd): writes dgamma / dbeta / dbias [128] (views of a gradient
    buffer) and returns (dr fp32 or None, dr Split or None), the gradient at the conv's output."""
    _require_cuda(dy, r, scratch)
    assert dy.is_contiguous() and r.is_contiguous() and dy.shape == r.shape
    c = r.shape[-1]
    dr = torch.empty_like(r) if want_f32 else None
    drs = Split.empty(tuple(r.shape), r.device) if want_split else None
    _lib.check(_lib.lib().pk_ss_bn_relu_bwd(_ptr(dy), _ptr(r), _ptr(mean), _ptr(rstd), _ptr(gamma), r.numel() // c, c, _ptr(scratch),
                                            _ptr(dgamma), _ptr(dbeta), _ptr(dbias), _ptr(dr), _ptr(drs.hi if drs else None),
                                            _ptr(drs.lo if drs else None), _stream()), "pk_ss_bn_relu_bwd")
    return dr, drs


def ss_loss(decoded, feats, num_frames, pred_durations, durations, num_phones, scratch, want_grads=True):
    """SpeedySpeech's L1 + SSIM + duration losses (pk_ss_loss) -> (losses fp32 [4] = loss, l1, duration, ssim; d loss / d decoded
    or None; d loss / d pred_durations or None).  num_frames / num_phones int32, durations int64, all on the device."""
    _require_cuda(decoded, feats, num_frames, pred_durations, durations, num_phones, scratch)
    assert decoded.is_contiguous() and feats.is_contiguous() and pred_durations.is_contiguous() and durations.is_contiguous()
    B, L, odim = decoded.shape
    T = pred_durations.shape[1]
    losses = torch.empty(4, dtype=torch.float32, device=decoded.device)
    g_dec = torch.empty_like(decoded) if want_grads else None
    g_dur = torch.empty_like(pred_durations) if want_grads else None
    _lib.check(_lib.lib().pk_ss_loss(_ptr(decoded), _ptr(feats), _ptr(num_frames), B, L, odim, _ptr(pred_durations), _ptr(durations),
                                     _ptr(num_phones), T, _ptr(scratch), _ptr(losses), _ptr(g_dec), _ptr(g_dur), _stream()), "pk_ss_loss")
    return losses, g_dec, g_dur


def dropout(x, p, seed, site, step, out_f32=True, out_split=False, inplace=False, step_dev=None):
    """pk_dropout: x fp32 tensor or Split (any shape, contiguous) -> (y fp32 or None, y Split or None).  p == 0 is not a
    special case here (callers skip the call)."""
    is_split = isinstance(x, Split)
    ref = x.hi if is_split else x
    assert ref.is_contiguous()
    n = ref.numel()
    y = (x if (inplace and not is_split) else torch.empty(ref.shape, dtype=torch.float32, device=ref.device)) if out_f32 else None
    ys = (x if (inplace and is_split) else Split.empty(tuple(ref.shape), ref.device)) if out_split else None
    _lib.check(_lib.lib().pk_dropout(_ptr(None if is_split else x), _ptr(x.hi if is_split else None), _ptr(x.lo if is_split else None), n,
                                     float(p), int(seed) & 0xFFFFFFFFFFFFFFFF, int(site), int(step), _ptr(step_dev), _ptr(y), _ptr(ys.hi if ys else None),
                                     _ptr(ys.lo if ys else None), _stream()), "pk_dropout")
    return y, ys


LSTM_ROWS, LSTM_SLICE = 64, 32          # csrc/lstm.cu: rows per tile, hidden units per CTA


def lstm_schedule(rows, hidden, max_ctas):
    """The grid of pk_lstm_fwd / pk_lstm_bwd (csrc/lstm.cu `schedule`): -> (slices, tiles, groups, grid).  CTA b serves hidden
    slice b % slices and row tiles b // slices + k * groups; grid 0 means the launch is refused (not one CTA per slice fits)."""
    slices, tiles = hidden // LSTM_SLICE, -(-rows // LSTM_ROWS)
    groups = min(tiles, max_ctas // slices)
    return slices, tiles, groups, groups * slices if groups >= 1 else 0


def lstm_counters(rows, t, device):
    return torch.empty(t * -(-rows // LSTM_ROWS), dtype=torch.int32, device=device)


def lstm_gate_perm(hidden, device):
    """Row order of the packed W_hh of pk_lstm_fwd: packed row 128 s + 8 (2 (u // 4) + g // 2) + 2 (u % 4) + g % 2 is W_hh row
    g * H + 32 s + u, so that one thread's wgmma accumulator fragment holds the four gates (i, f, g, o) of its units."""
    perm = torch.empty(4 * hidden, dtype=torch.int64)
    for s in range(hidden // LSTM_SLICE):
        for u in range(LSTM_SLICE):
            for g in range(4):
                perm[4 * LSTM_SLICE * s + 8 * (2 * (u // 4) + g // 2) + 2 * (u % 4) + g % 2] = g * hidden + LSTM_SLICE * s + u
    return perm.to(device)


def lstm_pack_fwd(w_hh, perm):
    """W_hh [4H, H] fp32 -> the split planes pk_lstm_fwd keeps resident (rows in lstm_gate_perm order)."""
    return Split.from_f32(w_hh.index_select(0, perm))


def lstm_pack_bwd(w_hh):
    """W_hh [4H, H] fp32 -> W_hh^T [H, 4H] split planes, the resident operand of pk_lstm_bwd."""
    return Split.from_f32(w_hh.t())


def lstm_fwd(g_in, b_hh, w_packed, h_all, h_split, c, gates=None, counters=None):
    """One LSTM layer over all steps (pk_lstm_fwd).  g_in (T, rows, 4H) = x W_ih^T + b_ih; w_packed from lstm_pack_fwd;
    h_all (T+1, rows, H) fp32 and h_split its Split planes, both with h0 in slab 0; c (rows, H) updated in place, or
    (T+1, rows, H) with c0 in slab 0 (then every c_t is kept, with the gates, for the backward)."""
    _require_cuda(g_in, b_hh, w_packed.hi, h_all, h_split.hi, c, gates, counters)
    T, rows, H4 = g_in.shape
    H = H4 // 4
    counters = lstm_counters(rows, T, g_in.device) if counters is None else counters
    c_step = 0 if c.dim() == 2 else rows * H
    _lib.check(_lib.lib().pk_lstm_fwd(_ptr(g_in), _ptr(b_hh), _ptr(w_packed.hi), _ptr(w_packed.lo), rows, T, H, _ptr(h_all),
                                      _ptr(h_split.hi), _ptr(h_split.lo), _ptr(c), c_step, _ptr(gates), _ptr(counters), counters.numel(),
                                      _stream()), "pk_lstm_fwd")


def lstm_bwd(wt_packed, gates, c_all, dh_in, dh_last, dgates, dg, dc=None, counters=None):
    """Backward through time of one layer (pk_lstm_bwd): wt_packed from lstm_pack_bwd -> dgates (T, rows, 4H) fp32 and its split
    planes `dg` (T * rows rows, 4H; one allocation)."""
    _require_cuda(wt_packed.hi, gates, c_all, dh_in, dh_last, dgates, dg.hi, dc, counters)
    T, rows, H4 = gates.shape
    H = H4 // 4
    dc = torch.empty(rows, H, dtype=torch.float32, device=gates.device) if dc is None else dc
    counters = lstm_counters(rows, T, gates.device) if counters is None else counters
    _lib.check(_lib.lib().pk_lstm_bwd(_ptr(wt_packed.hi), _ptr(wt_packed.lo), _ptr(gates), _ptr(c_all), _ptr(dh_in), _ptr(dh_last), rows,
                                      T, H, _ptr(dc), _ptr(dgates), _ptr(dg.hi), _ptr(dg.lo), _ptr(counters), counters.numel(), _stream()),
               "pk_lstm_bwd")
    return dgates


def ge2e_loss(embeds, n, m, c, w, b, want_grads=False):
    """GE2E loss on embeds viewed as (n, m, c) -> (loss (1,), sim (n*m, n), d_embeds, dw (1,), db (1,)); the gradients are None
    unless want_grads (dw, db already times 0.01)."""
    _require_cuda(embeds, w, b)
    dev = embeds.device
    L = _lib.lib()
    scratch = torch.empty(int(L.pk_ge2e_loss_scratch(n, m, c)), dtype=torch.float64, device=dev)
    loss = torch.empty(1, dtype=torch.float32, device=dev)
    sim = torch.empty(n * m, n, dtype=torch.float32, device=dev)
    de = torch.empty_like(embeds) if want_grads else None
    dw = torch.empty(1, dtype=torch.float32, device=dev) if want_grads else None
    db = torch.empty(1, dtype=torch.float32, device=dev) if want_grads else None
    _lib.check(L.pk_ge2e_loss(_ptr(embeds), n, m, c, _ptr(w), _ptr(b), _ptr(scratch), scratch.numel(), _ptr(loss), _ptr(sim), _ptr(de),
                              _ptr(dw), _ptr(db), _stream()), "pk_ge2e_loss")
    return loss, sim, de, dw, db


def ge2e_embed_bwd(e, dy, eps=1e-12):
    """backward of F.normalize(relu(z)) (rows, n), given e = relu(z)."""
    _require_cuda(e, dy)
    dz = torch.empty_like(e)
    rows, n = e.shape
    _lib.check(_lib.lib().pk_ge2e_embed_bwd(_ptr(e), _ptr(dy), rows, n, float(eps), _ptr(dz), _stream()), "pk_ge2e_embed_bwd")
    return dz


def segment_mean_normalize(x, offsets, eps=1e-12):
    """x (rows, n), offsets int32 (S + 1,) on the device -> (S, n): F.normalize(mean of each segment's rows, axis=0)."""
    _require_cuda(x, offsets)
    s = offsets.numel() - 1
    y = torch.empty(s, x.shape[1], dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().pk_segment_mean_normalize(_ptr(x), _ptr(offsets), s, x.shape[1], float(eps), _ptr(y), _stream()),
               "pk_segment_mean_normalize")
    return y


# ----------------------------------------------------------------------------------------------------------------
# Tacotron2 (csrc/tacotron2.cu)
# ----------------------------------------------------------------------------------------------------------------
TACO2_PRENET_SITES = (0, 1)          # Philox sites of the two prenet dropouts (pk_taco2_decode)


def taco2_embed(ids, table, tones=None, tone_table=None):
    """ids int64 (B, T) -> (B, T, C) = table[ids] (+ tone_table[tones], zero for tone 0)."""
    _require_cuda(ids, table, tones, tone_table)
    ids = ids.contiguous()
    tones = tones.contiguous() if tones is not None else None
    B, T = ids.shape
    y = torch.empty(B, T, table.shape[1], dtype=torch.float32, device=ids.device)
    _lib.check(_lib.lib().pk_taco2_embed(_ptr(ids), _ptr(table), _ptr(tones), _ptr(tone_table), B, T, table.shape[1], _ptr(y), _stream()),
               "pk_taco2_embed")
    return y


def taco2_time_major(x, lens=None, reverse=False):
    """x (B, T, C) -> (T, B, C); with reverse each sequence is reversed within its length (lens int32 or None = T)."""
    x = x.contiguous()
    B, T, Cc = x.shape
    y = torch.empty(T, B, Cc, dtype=torch.float32, device=x.device)
    _lib.check(_lib.lib().pk_taco2_time_major(_ptr(x), _ptr(lens), 1 if reverse else 0, B, T, Cc, _ptr(y), _stream()), "pk_taco2_time_major")
    return y


def taco2_bilstm_merge(h_fwd, h_bwd, lens=None, gc=None):
    """h_fwd / h_bwd (T, B, H) -> (B, T, 2H + G): [forward | backward at its own position | gc], rows past lens zero."""
    T, B, H = h_fwd.shape
    G = 0 if gc is None else gc.shape[1]
    gc = gc.contiguous().float() if gc is not None else None
    out = torch.empty(B, T, 2 * H + G, dtype=torch.float32, device=h_fwd.device)
    _lib.check(_lib.lib().pk_taco2_bilstm_merge(_ptr(h_fwd), _ptr(h_bwd), _ptr(lens), _ptr(gc), B, T, H, G, _ptr(out), _stream()),
               "pk_taco2_bilstm_merge")
    return out


def taco2_decode(w, keys, pkeys, steps, *, teacher, mels=None, text_lens=None, p_prenet=0.5, seed=0, prof=None):
    """pk_taco2_decode -> (mel_out (B, steps, dmr), align (B, steps, T_enc), stop (B, steps) or None, frames int32 (B,)); w is the
    dict of packed decoder weights (models/tacotron2.py).  prof: optional int64 tensor of pk_taco2_prof_len() per-CTA phase
    timers (scripts/time_tacotron2.py)."""
    _require_cuda(keys, pkeys, mels, text_lens)
    B, T_enc, d_enc = keys.shape
    dmr = w["proj_w"].shape[0]
    dev = keys.device
    L = _lib.lib()
    ws = torch.empty(int(L.pk_taco2_workspace(B, T_enc, d_enc)), dtype=torch.float32, device=dev)
    mel = torch.empty(B, steps, dmr, dtype=torch.float32, device=dev)
    align = torch.empty(B, steps, T_enc, dtype=torch.float32, device=dev)
    stop = torch.empty(B, steps, dtype=torch.float32, device=dev) if w.get("stop_w") is not None else None
    frames = torch.empty(B, dtype=torch.int32, device=dev)
    a = _lib.Taco2DecodeArgs()
    a.batch, a.t_enc, a.d_enc, a.dmr, a.steps, a.teacher, a.loc_k = B, T_enc, d_enc, dmr, steps, 1 if teacher else 0, w["loc_w"].shape[2]
    a.p_prenet, a.seed = float(p_prenet), int(seed) & 0xFFFFFFFFFFFFFFFF
    a.keys, a.pkeys, a.text_lens, a.mels = keys.data_ptr(), pkeys.data_ptr(), _ptr(text_lens).value, _ptr(mels).value
    for n in ("pre_w1", "pre_w2", "att_w", "att_b_ih", "att_b_hh", "q_w", "loc_w", "v_w", "dec_w", "dec_b_ih", "dec_b_hh", "proj_w", "proj_b",
              "stop_w", "stop_b"):
        setattr(a, n, _ptr(w.get(n)).value)
    a.workspace, a.workspace_len = ws.data_ptr(), ws.numel()
    a.mel_out, a.align_out, a.stop_out, a.frames = mel.data_ptr(), align.data_ptr(), _ptr(stop).value, frames.data_ptr()
    if prof is not None:
        a.prof, a.prof_len = prof.data_ptr(), prof.numel()
    _lib.check(L.pk_taco2_decode(C.byref(a), _stream()), "pk_taco2_decode")
    return mel, align, stop, frames


def taco2_loss(mel, post, target, align=None, slens=None, plens=None, sigma=0.2, stop_logits=None):
    """Tacotron2Loss (pk_taco2_loss) -> fp32 (5,) = loss, mel_loss, post_mel_loss, guided_attn_loss, stop_loss."""
    _require_cuda(mel, post, target, align, slens, plens, stop_logits)
    mel, post, target = mel.contiguous().float(), post.contiguous().float(), target.contiguous().float()
    align = align.contiguous().float() if align is not None else None
    stop_logits = stop_logits.contiguous().float() if stop_logits is not None else None
    slens = slens.to(torch.int32).contiguous() if slens is not None else None
    plens = plens.to(torch.int32).contiguous() if plens is not None else None
    B, T, Cc = mel.shape
    out = torch.empty(5, dtype=torch.float32, device=mel.device)
    _lib.check(_lib.lib().pk_taco2_loss(_ptr(mel), _ptr(post), _ptr(target), B, T, Cc, _ptr(align), align.shape[2] if align is not None else 0,
                                        _ptr(slens), _ptr(plens), float(sigma), _ptr(stop_logits), _ptr(out), _stream()), "pk_taco2_loss")
    return out


# ----------------------------------------------------------------------------------------------------------------
# TransformerTTS (csrc/transformer_tts.cu)
# ----------------------------------------------------------------------------------------------------------------
def tts_decode(w, mem_kv, pe, *, heads, steps, minlen, maxlen, threshold, p_prenet=0.5, seed=0):
    """pk_tts_decode -> (outs (steps, r * odim), probs (steps, r), att_ws (layers, heads, steps, T_enc), frames int32 (1,)); w is the
    dict of packed decoder weights (models/transformer_tts.py), mem_kv (T_enc, layers * 2 adim) the source-attention K / V,
    pe (steps, adim) the alpha-scaled positional encoding rows."""
    _require_cuda(mem_kv, pe)
    T_enc = mem_kv.shape[0]
    A, U, Up, L, r, odim = w["adim"], w["units"], w["prenet_units"], w["layers"], w["r"], w["odim"]
    dev = mem_kv.device
    lib = _lib.lib()
    ws = torch.empty(int(lib.pk_tts_workspace(A, U, Up, L, steps)), dtype=torch.float32, device=dev)
    outs = torch.empty(steps, r * odim, dtype=torch.float32, device=dev)
    probs = torch.empty(steps, r, dtype=torch.float32, device=dev)
    att = torch.empty(L, heads, steps, T_enc, dtype=torch.float32, device=dev)
    frames = torch.empty(1, dtype=torch.int32, device=dev)
    a = _lib.TtsDecodeArgs()
    a.t_enc, a.adim, a.heads, a.units, a.odim, a.r = T_enc, A, heads, U, odim, r
    a.prenet_layers, a.prenet_units, a.layers, a.steps, a.minlen, a.maxlen = w["prenet_layers"], Up, L, steps, minlen, maxlen
    a.threshold, a.p_prenet, a.seed = float(threshold), float(p_prenet), int(seed) & 0xFFFFFFFFFFFFFFFF
    a.mem_kv, a.pe = mem_kv.data_ptr(), pe.data_ptr()
    for n in ("pre_w", "pre_b", "in_w", "in_b", "layer_w", "norm", "out_w", "out_b"):
        setattr(a, n, w[n].data_ptr())
    a.workspace, a.workspace_len = ws.data_ptr(), ws.numel()
    a.outs, a.probs, a.att_ws, a.frames = outs.data_ptr(), probs.data_ptr(), att.data_ptr(), frames.data_ptr()
    _lib.check(lib.pk_tts_decode(C.byref(a), _stream()), "pk_tts_decode")
    return outs, probs, att, frames


def tts_text_eos(text, lens, eos):
    """text int64 (B, T), lens int32 (B,) -> (xs int64 (B, T + 1): text with eos at column lens[b], zeros after; ilens int32 = lens + 1)."""
    B, T = text.shape
    xs = torch.empty(B, T + 1, dtype=torch.int64, device=text.device)
    ilens = torch.empty(B, dtype=torch.int32, device=text.device)
    _lib.check(_lib.lib().pk_tts_text_eos(_ptr(text), _ptr(lens), B, T, int(eos), _ptr(xs), _ptr(ilens), _stream()), "pk_tts_text_eos")
    return xs, ilens


def tts_shift_frames(ys, r):
    """ys fp32 (B, L, odim) -> (B, L // r, odim): the frames thinned by r (the last of each group), a zero first frame, the last dropped."""
    B, L, odim = ys.shape
    out = torch.empty(B, L // r, odim, dtype=torch.float32, device=ys.device)
    _lib.check(_lib.lib().pk_tts_shift_frames(_ptr(ys), B, L, odim, r, _ptr(out), _stream()), "pk_tts_shift_frames")
    return out


def tts_prenet_dropout_(x, p, seed, site):
    """In place on fp32 (B, L, U): keep element (b, t, j) with Philox site `site`, step t, element b U + j, scale 1 / (1 - p)."""
    B, L, U = x.shape
    _lib.check(_lib.lib().pk_tts_prenet_dropout(_ptr(x), B, L, U, float(p), int(seed) & 0xFFFFFFFFFFFFFFFF, int(site), _stream()),
               "pk_tts_prenet_dropout")
    return x


def tts_stop_labels(olens, width):
    """olens int32 (B,) -> float (B, width): 1 at and after column olens[b] - 1 and in the last column, else 0."""
    B = olens.numel()
    out = torch.empty(B, width, dtype=torch.float32, device=olens.device)
    _lib.check(_lib.lib().pk_tts_stop_labels(_ptr(olens), B, width, _ptr(out), _stream()), "pk_tts_stop_labels")
    return out


def tts_guided_loss(partials, ilens, olens, rows, keys, heads_layers, lam, losses):
    """pk_tts_guided_loss: losses[4] = the guided attention loss from every guided layer's partials, added to losses[0]."""
    _lib.check(_lib.lib().pk_tts_guided_loss(_ptr(partials), partials.numel(), _ptr(ilens), _ptr(olens), ilens.numel(), rows, keys,
                                             heads_layers, float(lam), _ptr(losses), _stream()), "pk_tts_guided_loss")


TTS_LOSS_TYPES = {"L1": 0, "L2": 1, "L1+L2": 2}


def tts_loss(before, after, ys, logits, labels, olens, pos_weight=5.0, loss_type="L1", losses=None):
    """pk_tts_loss: -> losses fp32 (5,) = loss, l1, l2, bce and a slot for the guided loss (left as it was); before / after / ys
    (B, L, odim), logits / labels (B, L), olens int32 (B,), all contiguous on the device."""
    B, L, odim = before.shape
    lib = _lib.lib()
    ws = torch.empty(int(lib.pk_tts_loss_workspace(B, L)), dtype=torch.float32, device=before.device)
    if losses is None:
        losses = torch.zeros(5, dtype=torch.float32, device=before.device)
    _lib.check(lib.pk_tts_loss(_ptr(before), _ptr(after), _ptr(ys), _ptr(logits), _ptr(labels), _ptr(olens), B, L, odim, float(pos_weight),
                               TTS_LOSS_TYPES[loss_type], _ptr(ws), _ptr(losses), _stream()), "pk_tts_loss")
    return losses


def tts_loss_bwd(before, after, ys, logits, labels, olens, pos_weight=5.0, loss_type="L1"):
    """pk_tts_loss_bwd -> (d loss / d before, d loss / d after, d loss / d logits)."""
    B, L, odim = before.shape
    gb, ga, gl = torch.empty_like(before), torch.empty_like(after), torch.empty_like(logits)
    _lib.check(_lib.lib().pk_tts_loss_bwd(_ptr(before), _ptr(after), _ptr(ys), _ptr(logits), _ptr(labels), _ptr(olens), B, L, odim,
                                          float(pos_weight), TTS_LOSS_TYPES[loss_type], _ptr(gb), _ptr(ga), _ptr(gl), _stream()),
               "pk_tts_loss_bwd")
    return gb, ga, gl
