"""pk_fused_attention_ex against fp64: causal self-attention (TransformerTTS's teacher-forced decoder) over the tile edges and
ragged key lengths, cross attention with T_q != T_k, and FastSpeech2's self-attention call bit for bit against the output the
kernel gave before it was generalised (PARENT_SHA256: the digest of the hi | lo planes that fs2_case() gave through
pk_transpose_heads + pk_fused_attention of the library built from commit 1b83b3c, on an H100).

Bound: Q, K, V and P enter the tensor cores as split-bf16 pairs (hi + lo, 3 passes), about 2^-16 relative per operand, and the
dropped lo x lo term is ~2^-16 x 2^-16; the online softmax adds exp2.approx (2 ulp) and fp32 sums over <= 1500 keys (~1500 x 2^-24).
The context is a convex combination of V rows, so its error is bounded by (a few x 2^-16) x max|V| plus the score error
(~2^-16 x |q||k| / sqrt(d_k) <= 1e-4 at these magnitudes) times max|V|: 3e-4 x max|V| covers both with a margin of ~3; a wrong mask,
tile skip or column offset moves the context by O(max|V|)."""
import hashlib
import math

import pytest
import torch

from parakeet_b200 import ops
from parakeet_b200.ops import Split

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
PARENT_SHA256 = "0b50d53f15e679853ed6d711bd33e438fdc98ee29e522db6a9d18502b834a00e"


def ref_attention(q, k, v, key_lens, causal):
    """fp64: q (B, Tq, H, dk), k / v (B, Tk, H, dk) -> (B, Tq, H dk), on q's device."""
    B, Tq, H, dk = q.shape
    Tk = k.shape[1]
    s = torch.einsum("bqhd,bkhd->bhqk", q, k) / math.sqrt(dk)
    mask = torch.arange(Tk, device=q.device)[None, :] < key_lens.to(q.device)[:, None]   # (B, Tk)
    mask = mask[:, None, None, :].expand(B, 1, Tq, Tk)
    if causal:
        mask = mask & torch.tril(torch.ones(Tq, Tk, dtype=torch.bool, device=q.device))[None, None]
    s = s.masked_fill(~mask, float("-inf"))
    p = torch.softmax(s, -1)
    return torch.einsum("bhqk,bkhd->bqhd", p, v).reshape(B, Tq, H * dk)


def split_of(x):
    return Split.from_f32(x.float().contiguous().to(DEV))


@pytest.mark.parametrize("dk", [64, 128, 192])
@pytest.mark.parametrize("T", [1, 63, 64, 65, 127, 128, 129, 800, 1500])
def test_causal_self_attention(T, dk):
    H, B = 2, 3
    g = torch.Generator().manual_seed(T * 7 + dk)
    qkv = torch.randn(B, T, 3, H, dk, generator=g, dtype=torch.float64)
    lens = torch.tensor([T, max(1, T // 2), 1])
    buf = split_of(qkv.reshape(B, T, 3 * H * dk))
    q64, k64, v64 = (Split.float(buf)[..., i * H * dk:(i + 1) * H * dk].double().cpu().reshape(B, T, H, dk) for i in range(3))
    ctx = Split.empty((B, T, H * dk), DEV)
    ops.fused_attention_ex(buf, buf, heads=H, q_col0=0, k_col0=H * dk, v_col0=2 * H * dk, key_lens=lens.to(DEV, torch.int32), causal=True,
                           ctx=ctx)
    want = ref_attention(q64, k64, v64, lens, causal=True)                                # every query row live, padded rows too
    err = (ctx.float().double().cpu() - want).abs().max().item()
    assert err < 3e-4 * v64.abs().max().item(), err


def cross_cases():
    """T_k x d_k x T_q x layers; the cases of 64-wide heads, 300 queries and 2 layers keep their T_k ids.  T_q = 1 is a
    teacher-forced batch whose speech_lengths == r; 6 layers put k_col0 = 2 A l deep into the (B, T_k, 12 A) buffer."""
    out = []
    for Tk in (1, 15, 128, 129, 700):
        for dk in (64, 128, 192):
            for Tq in (300, 1):
                for L in (2, 6):
                    tag = str(Tk) if (dk, Tq, L) == (64, 300, 2) else f"{Tk}-dk{dk}-Tq{Tq}-L{L}"
                    out.append(pytest.param(Tk, dk, Tq, L, id=tag))
    return out


@pytest.mark.parametrize("Tk,dk,Tq,L", cross_cases())
def test_cross_attention(Tk, dk, Tq, L):
    H, B = 8, 3
    A = H * dk
    g = torch.Generator().manual_seed(Tk * 1000 + dk * 10 + L + Tq)
    q = torch.randn(B, Tq, A, generator=g)
    mem = torch.randn(B, Tk, L * 2 * A, generator=g)                                      # [K_0 | V_0 | K_1 | V_1 | ...]
    lens = torch.tensor([Tk, max(1, Tk - 7), 1])
    qs, ms = split_of(q), split_of(mem)
    qf, mf = qs.float().double(), ms.float().double()                                     # the reference on the device, in fp64
    for l in range(L):
        ctx = Split.empty((B, Tq, A), DEV)
        ops.fused_attention_ex(qs, ms, heads=H, q_col0=0, k_col0=2 * A * l, v_col0=2 * A * l + A, key_lens=lens.to(DEV, torch.int32), ctx=ctx)
        k = mf[..., 2 * A * l:2 * A * l + A].reshape(B, Tk, H, dk)
        v = mf[..., 2 * A * l + A:2 * A * (l + 1)].reshape(B, Tk, H, dk)
        want = ref_attention(qf.reshape(B, Tq, H, dk), k, v, lens, causal=False)
        err = (ctx.float().double() - want).abs().max().item()
        assert err < 3e-4 * v.abs().max().item(), (l, err)


def fs2_case():
    """FastSpeech2's call: (B, T, 3A) qkv, 2 heads of 192, key and row lengths."""
    g = torch.Generator().manual_seed(2026)
    B, T, H, dk = 3, 333, 2, 192
    qkv = Split.from_f32((torch.randn(B, T, 3 * H * dk, generator=g)).to(DEV))
    lens = torch.tensor([333, 200, 17], dtype=torch.int32, device=DEV)
    return qkv, H, lens


def fs2_ctx():
    qkv, H, lens = fs2_case()
    ctx = ops.fused_attention(qkv, H, key_lens=lens, row_lens=lens)
    torch.cuda.synchronize()
    return ctx.hi.view(torch.int16).cpu().numpy(), ctx.lo.view(torch.int16).cpu().numpy()


def test_fastspeech2_self_attention_is_bit_identical_to_the_ungeneralised_kernel():
    hi, lo = fs2_ctx()
    assert hashlib.sha256(hi.tobytes() + lo.tobytes()).hexdigest() == PARENT_SHA256
