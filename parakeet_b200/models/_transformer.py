"""The FFT-block stack shared by FastSpeech2 (encoder and decoder) and TransformerTTS (encoder): the reference's
fastspeech2_transformer `Encoder` after its input layer, pre-LN, concat_after = False."""
import math
import os

import torch

from .. import ops
from ..ops import Split


def pack_fft_blocks(p, pre, layers, linear_ffn, dev):
    """`{pre}encoders.{i}.*` and `{pre}after_norm.*` of a CPU fp32 state dict -> (per-layer packed weights, after_norm (gamma, beta))."""

    def dv(t):
        return t.contiguous().to(dev)

    out = []
    for i in range(layers):
        q = f"{pre}encoders.{i}."
        sa = q + "self_attn."
        wqkv = torch.cat([p[sa + "linear_q.weight"], p[sa + "linear_k.weight"], p[sa + "linear_v.weight"]], dim=1).t()
        bqkv = torch.cat([p[sa + "linear_q.bias"], p[sa + "linear_k.bias"], p[sa + "linear_v.bias"]])
        if linear_ffn:
            w1, w2 = p[q + "feed_forward.w_1.weight"].t(), p[q + "feed_forward.w_2.weight"].t()
        else:
            w1, w2 = p[q + "feed_forward.w_1.weight"], p[q + "feed_forward.w_2.weight"]
        out.append(dict(
            wqkv=ops.pack_weight(wqkv, dev), bqkv=dv(bqkv),
            wo=ops.pack_weight(p[sa + "linear_out.weight"].t(), dev), bo=dv(p[sa + "linear_out.bias"]),
            w1=ops.pack_weight(w1, dev), b1=dv(p[q + "feed_forward.w_1.bias"]),
            w2=ops.pack_weight(w2, dev), b2=dv(p[q + "feed_forward.w_2.bias"]),
            n1=(dv(p[q + "norm1.weight"]), dv(p[q + "norm1.bias"])),
            n2=(dv(p[q + "norm2.weight"]), dv(p[q + "norm2.bias"])),
            units=w1.shape[0]))
    return out, (dv(p[pre + "after_norm.weight"]), dv(p[pre + "after_norm.bias"]))


def fft_stack(x, layers, after_norm, heads, ffn_k, row_lens, key_lens, want_split_out=False):
    """Encoder.forward after the embedding (encoder.py:189-192): N x EncoderLayer (encoder_layer.py:64-115) + after_norm.
    x fp32 (B, T, A).  row_lens: int32 lens for the independent-utterance mode (rows >= len are kept at zero) or None.
    key_lens: int32 lens of the key-padding mask (attention.py:107-119) or None."""
    B, T, A = x.shape
    H, dk = heads, A // heads
    Tp = (T + 63) // 64 * 64
    dev = x.device
    fused = dk in (64, 128, 192) and os.environ.get("PK_FUSED_ATTN", "1") != "0"
    s_buf = torch.empty(B * H, T, Tp, dtype=torch.float32, device=dev) if not fused else None
    ctx = Split.empty((B, T, A), dev)
    for lay in layers:
        _, h = ops.layer_norm(x, *lay["n1"], lens=row_lens)
        _, qkv = ops.conv_gemm(h, lay["wqkv"], n=3 * A, k=A, bias=lay["bqkv"], lens=row_lens, out_f32=False, out_split=True)
        if fused:
            # scores, key mask, softmax and P.V in one kernel (csrc/attention.cu); no (B*H, T, T) tensor in HBM
            ops.fused_attention(qkv, H, key_lens=key_lens, row_lens=row_lens, ctx=ctx)
            x, _ = ops.conv_gemm(ctx, lay["wo"], n=A, k=A, bias=lay["bo"], residual=x, lens=row_lens)
            _, h = ops.layer_norm(x, *lay["n2"], lens=row_lens)
            _, u = ops.conv_gemm(h, lay["w1"], n=lay["units"], k=A, taps=ffn_k, bias=lay["b1"], act="relu", lens=row_lens,
                                 out_f32=False, out_split=True)
            x, _ = ops.conv_gemm(u, lay["w2"], n=A, k=lay["units"], taps=ffn_k, bias=lay["b2"], residual=x, lens=row_lens)
            continue
        ld = 3 * A
        q_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
        k_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=A, colh=dk)
        ops.batched_matmul_nt(qkv, qkv, batch=B, heads=H, m=T, n=T, k=dk, a_spec=q_spec, b_spec=k_spec,
                              scale=1.0 / math.sqrt(dk), y_f32=s_buf, y_batch_stride=H * T * Tp, y_head_stride=T * Tp, y_ld=Tp)
        p = ops.masked_softmax(s_buf, key_lens, B, H, T, T)
        vt = ops.transpose_heads(qkv, col0=2 * A, dk=dk, heads=H, ld_dst=Tp)
        p_spec = dict(rows=T, cols=Tp, ld=Tp, batch_stride=T * Tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
        v_spec = dict(rows=dk, cols=Tp, ld=Tp, batch_stride=dk * Tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
        ops.batched_matmul_nt(p, vt, batch=B, heads=H, m=T, n=dk, k=Tp, a_spec=p_spec, b_spec=v_spec, y_split=ctx,
                              y_batch_stride=T * A, y_head_stride=dk, y_ld=A, lens=row_lens)
        x, _ = ops.conv_gemm(ctx, lay["wo"], n=A, k=A, bias=lay["bo"], residual=x, lens=row_lens)
        _, h = ops.layer_norm(x, *lay["n2"], lens=row_lens)
        _, u = ops.conv_gemm(h, lay["w1"], n=lay["units"], k=A, taps=ffn_k, bias=lay["b1"], act="relu", lens=row_lens,
                             out_f32=False, out_split=True)
        x, _ = ops.conv_gemm(u, lay["w2"], n=A, k=lay["units"], taps=ffn_k, bias=lay["b2"], residual=x, lens=row_lens)
    return ops.layer_norm(x, *after_norm, lens=row_lens, want_f32=True, want_split=want_split_out)
