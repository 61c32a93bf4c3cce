"""pk_conv_gemm as the attention and weight-gradient code drive it (ops.batched_matmul_nt): head-sliced and head-batched operand
addressing, strided output views and ragged `lens`, against an fp64 einsum over the same addressing, on both the wgmma and the SIMT
path; and the K-tail contract (with k % 64 != 0 nothing past an operand's K slice may enter the product)."""
import math

import pytest
import torch
import torch.nn.functional as F

from parakeet_b200 import _lib, ops
from parakeet_b200.ops import Split

pytestmark = pytest.mark.gpu


def _split(x):
    return Split.from_f32(x.contiguous())


def _operand(s, spec, batch, heads, rows, k):
    """fp64 values the GEMM reads for operand `s` (Split over one contiguous allocation): (batch, heads, rows, k), zero where
    the spec puts the element outside the operand (TMA zero fill)."""
    flat = s.float().double().reshape(-1)
    dev = flat.device
    bz = torch.arange(batch, device=dev)[:, None, None, None]
    hz = torch.arange(heads, device=dev)[None, :, None, None]
    r = torch.arange(rows, device=dev)[None, None, :, None]
    kk = torch.arange(k, device=dev)[None, None, None, :]
    bi = bz * spec["bmul"] + hz * spec["hmul"]
    col = spec["col0"] + hz * spec["colh"] + kk
    ok = (r < spec["rows"]) & (col < spec["cols"]) & (bi < spec["batches"])
    idx = (bi * spec["batch_stride"] + r * spec["ld"] + col).clamp(0, flat.numel() - 1)
    return torch.where(ok, flat[idx], torch.zeros((), dtype=torch.float64, device=dev))


def _out_index(batch, heads, m, n, ybs, yhs, yld, dev):
    bz = torch.arange(batch, device=dev)[:, None, None, None]
    hz = torch.arange(heads, device=dev)[None, :, None, None]
    t = torch.arange(m, device=dev)[None, None, :, None]
    j = torch.arange(n, device=dev)[None, None, None, :]
    return bz * ybs + hz * yhs + t * yld + j


def _check_nt(a, b, *, batch, heads, m, n, k, sa, sb, scale, ybs, yhs, yld, y_numel, y_off=0, lens=None, split_out=False):
    """Run batched_matmul_nt on both paths into a NaN-filled output allocation of y_numel elements (the output is the view starting
    at y_off) and compare every written element with the fp64 einsum; every element the addressing does not cover must stay NaN."""
    dev = a.hi.device
    A = _operand(a, sa, batch, heads, m, k)
    Bm = _operand(b, sb, batch, heads, n, k)
    ref = torch.einsum("zhmk,zhnk->zhmn", A, Bm) * scale
    mag = torch.einsum("zhmk,zhnk->zhmn", A.abs(), Bm.abs()) * abs(scale)
    if lens is not None:
        live = (torch.arange(m, device=dev)[None, :] < lens.long()[:, None])[:, None, :, None]
        ref, mag = ref * live, mag * live
    # error bound per element: the 3-pass split-bf16 product drops lo*lo (<= 2^-16 of |a b|), fp32 accumulation of k products
    # (k * 2^-23 of sum |a b|: the worst case, not assuming round-to-nearest inside the tensor core), and the fp32 -> split planes
    # rounding of a split output (2^-16 of |y|)
    bound = (2.0 ** -16 + k * 2.0 ** -23) * mag + (2.0 ** -16 * ref.abs() if split_out else 0.0) + 1e-30
    idx = _out_index(batch, heads, m, n, ybs, yhs, yld, dev) + y_off
    covered = torch.zeros(y_numel, dtype=torch.bool, device=dev)
    covered[idx.reshape(-1)] = True
    for simt in (False, True):
        if split_out:
            ybuf = Split.empty((y_numel,), dev)
            ybuf.hi.fill_(float("nan"))
            ybuf.lo.fill_(float("nan"))
            ops.batched_matmul_nt(a, b, batch=batch, heads=heads, m=m, n=n, k=k, a_spec=sa, b_spec=sb, scale=scale,
                                  y_split=Split(ybuf.hi[y_off:], ybuf.lo[y_off:]), y_batch_stride=ybs, y_head_stride=yhs, y_ld=yld,
                                  lens=lens, simt=simt)
            y = ybuf.float()
        else:
            y = torch.full((y_numel,), float("nan"), dtype=torch.float32, device=dev)
            ops.batched_matmul_nt(a, b, batch=batch, heads=heads, m=m, n=n, k=k, a_spec=sa, b_spec=sb, scale=scale, y_f32=y[y_off:],
                                  y_batch_stride=ybs, y_head_stride=yhs, y_ld=yld, lens=lens, simt=simt)
        got = y[idx].double()
        err = (got - ref).abs()
        path = "simt" if simt else "wgmma"
        assert torch.isfinite(got).all(), path
        assert (err <= bound).all(), f"{path}: max err {err.max().item():.3e}, worst err / bound {(err / bound).max().item():.2f}"
        assert torch.isnan(y[~covered]).all(), f"{path} wrote outside the output view"


# (B, T, H, dk): T not a multiple of 128; T < 64; B * H * m-tiles * n-tiles beyond the 132 SMs
SHAPES = [(2, 77, 2, 64), (3, 50, 3, 128), (2, 300, 2, 192), (16, 300, 4, 64), (5, 129, 2, 192)]


@pytest.mark.parametrize("B,T,H,dk", SHAPES)
def test_scores_qk_layout(cuda, B, T, H, dk):
    """S = Q K^T / sqrt(dk) of FastSpeech2._encoder_stack (non-fused) and fs2_step.stack_fwd: both operands head slices of one
    (B, T, 3A) qkv buffer, output (B*H, T, Tp) with a row pitch Tp > T."""
    g = torch.Generator(device="cpu").manual_seed(T * 7 + dk)
    A = H * dk
    ld, Tp = 3 * A, ops.ceil_to(T, 64)
    qkv = _split(torch.randn(B, T, ld, generator=g).to(cuda))
    q_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
    k_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=A, colh=dk)
    _check_nt(qkv, qkv, batch=B, heads=H, m=T, n=T, k=dk, sa=q_spec, sb=k_spec, scale=1.0 / math.sqrt(dk), ybs=H * T * Tp, yhs=T * Tp,
              yld=Tp, y_numel=B * H * T * Tp)


@pytest.mark.parametrize("B,T,H,dk", SHAPES)
def test_context_pv_layout(cuda, B, T, H, dk):
    """ctx = P V: P (B*H, T, Tp) batched per head (bmul=H, hmul=1), V^T from transpose_heads, split output interleaving the heads
    (y_head_stride = dk, y_ld = A), `lens` with whole dead m-tiles."""
    g = torch.Generator(device="cpu").manual_seed(T * 11 + dk)
    A = H * dk
    ld, Tp = 3 * A, ops.ceil_to(T, 64)
    qkv = _split(torch.randn(B, T, ld, generator=g).to(cuda))
    p = torch.zeros(B * H, T, Tp)
    p[:, :, :T] = torch.randn(B * H, T, T, generator=g)
    p = _split(p.to(cuda))
    vt = ops.transpose_heads(qkv, col0=2 * A, dk=dk, heads=H, ld_dst=Tp)
    lens = torch.tensor([T] + [max(1, T // (2 + i)) for i in range(B - 1)], dtype=torch.int32, device=cuda)
    if T > 128:
        lens[-1] = 5      # every m-tile of the last utterance but the first is dead
    p_spec = dict(rows=T, cols=Tp, ld=Tp, batch_stride=T * Tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
    v_spec = dict(rows=dk, cols=Tp, ld=Tp, batch_stride=dk * Tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
    _check_nt(p, vt, batch=B, heads=H, m=T, n=dk, k=Tp, sa=p_spec, sb=v_spec, scale=1.0, ybs=T * A, yhs=dk, yld=A, y_numel=B * T * A,
              lens=lens, split_out=True)


@pytest.mark.parametrize("B,T,H,dk", SHAPES)
def test_attention_backward_layouts(cuda, B, T, H, dk):
    """The three backward products of fs2_step.stack_bwd at their specs: dP = dO V^T (dO head-sliced at A columns, V at 2A of the
    3A-wide qkv), dV = P^T dO and dQ / dK = dS K / dS^T Q (head-batched operands, output a column window of the (B, T, 3A) dqkv)."""
    g = torch.Generator(device="cpu").manual_seed(T * 13 + dk)
    A = H * dk
    ld, Tp = 3 * A, ops.ceil_to(T, 64)
    qkv = _split(torch.randn(B, T, ld, generator=g).to(cuda))
    do = _split(torch.randn(B, T, A, generator=g).to(cuda))
    o_spec = dict(rows=T, cols=A, ld=A, batch_stride=T * A, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
    v_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=2 * A, colh=dk)
    _check_nt(do, qkv, batch=B, heads=H, m=T, n=T, k=dk, sa=o_spec, sb=v_spec, scale=1.0, ybs=H * T * Tp, yhs=T * Tp, yld=Tp,
              y_numel=B * H * T * Tp)
    # dV / dQ / dK: (B*H, T, Tp) square operand (zero past T, as transpose_planes leaves it) times (B, H, dk, Tp) head planes
    z = torch.zeros(B * H, T, Tp)
    z[:, :, :T] = torch.randn(B * H, T, T, generator=g)
    z = _split(z.to(cuda))
    d = torch.zeros(B, H, dk, Tp)
    d[..., :T] = torch.randn(B, H, dk, T, generator=g)
    d = _split(d.to(cuda))
    z_spec = dict(rows=T, cols=Tp, ld=Tp, batch_stride=T * Tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
    d_spec = dict(rows=dk, cols=Tp, ld=Tp, batch_stride=dk * Tp, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
    for col in (0, A, 2 * A):         # dQ, dK, dV land at these columns of dqkv
        _check_nt(z, d, batch=B, heads=H, m=T, n=dk, k=Tp, sa=z_spec, sb=d_spec, scale=1.0, ybs=T * ld, yhs=dk, yld=ld,
                  y_numel=B * T * ld, y_off=col)


@pytest.mark.parametrize("m,n,kk,s", [(80, 256, 3 * 64, 3), (130, 70, 64, 1), (256, 384, 5 * 128, 5)])
def test_split_k_weight_gradient_layout(cuda, m, n, kk, s):
    """wgrad.nt_splitk's addressing: S K-slices of one (rows, S * ks) plane pair as batches (batch_stride = ks, ld = S * ks)."""
    g = torch.Generator(device="cpu").manual_seed(m + n + kk)
    ks = kk // s
    at, bt = _split(torch.randn(m, kk, generator=g).to(cuda)), _split(torch.randn(n, kk, generator=g).to(cuda))
    sa = dict(rows=m, cols=ks, ld=kk, batch_stride=ks, batches=s, bmul=1, hmul=0, col0=0, colh=0)
    sb = dict(rows=n, cols=ks, ld=kk, batch_stride=ks, batches=s, bmul=1, hmul=0, col0=0, colh=0)
    _check_nt(at, bt, batch=s, heads=1, m=m, n=n, k=ks, sa=sa, sb=sb, scale=1.0, ybs=m * n, yhs=0, yld=n, y_numel=s * m * n)


# ---------------------------------------------------------------------------------------------------------------------------
# K-tail contract
# ---------------------------------------------------------------------------------------------------------------------------
BIG = 1.0e4


@pytest.mark.parametrize("dk", [96, 32])
def test_head_sliced_k_tail_is_refused(cuda, dk):
    """A head slice of k % 64 != 0 columns inside a wider activation: the 64-column K chunks of the tensor-core path would read the
    next head's columns, so the wrapper refuses it on both paths before any launch."""
    B, T, H = 2, 70, 4
    A = H * dk
    ld = 3 * A
    qkv = _split(torch.full((B, T, ld), BIG, device=cuda))
    y = torch.zeros(B * H, T, 128, device=cuda)
    q_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
    k_spec = dict(rows=T, cols=ld, ld=ld, batch_stride=T * ld, batches=B, bmul=1, hmul=0, col0=A, colh=dk)
    before = _lib.launch_count()
    for simt in (False, True):
        with pytest.raises(_lib.PkError, match="not a multiple of 64"):
            ops.batched_matmul_nt(qkv, qkv, batch=B, heads=H, m=T, n=T, k=dk, a_spec=q_spec, b_spec=k_spec, y_f32=y,
                                  y_batch_stride=H * T * 128, y_head_stride=T * 128, y_ld=128, simt=simt)
    assert _lib.launch_count() == before
    assert (y == 0).all()


@pytest.mark.parametrize("dk", [96, 32])
def test_k_tail_ends_at_operand_extent(cuda, dk):
    """k % 64 != 0 where each operand's K slice ends at its `cols`: per-head planes (B*H, T, dk) with a row pitch ld > dk whose
    extra columns hold large values.  Both paths must use exactly the first dk columns (TMA zero-fills the chunk past cols)."""
    B, T, H = 2, 150, 3
    ld = dk + 8
    g = torch.Generator(device="cpu").manual_seed(dk)
    x = torch.full((2, B * H, T, ld), BIG)
    x[..., :dk] = torch.randn(2, B * H, T, dk, generator=g)
    q, kx = _split(x[0].to(cuda)), _split(x[1].to(cuda))
    spec = dict(rows=T, cols=dk, ld=ld, batch_stride=T * ld, batches=B * H, bmul=H, hmul=1, col0=0, colh=0)
    Tp = ops.ceil_to(T, 64)
    _check_nt(q, kx, batch=B, heads=H, m=T, n=T, k=dk, sa=spec, sb=spec, scale=0.1, ybs=H * T * Tp, yhs=T * Tp, yld=Tp,
              y_numel=B * H * T * Tp)
    # a single head sliced at col0 whose slice ends exactly at cols, pitch beyond it filled with large values
    one = dict(rows=T, cols=64 + dk, ld=ld + 64, batch_stride=T * (ld + 64), batches=B * H, bmul=H, hmul=1, col0=64, colh=0)
    xs = torch.full((B * H, T, ld + 64), BIG)
    xs[..., 64:64 + dk] = torch.randn(B * H, T, dk, generator=g)
    xs = _split(xs.to(cuda))
    _check_nt(xs, xs, batch=B, heads=H, m=T, n=T, k=dk, sa=one, sb=one, scale=1.0, ybs=H * T * Tp, yhs=T * Tp, yld=Tp, y_numel=B * H * T * Tp)


@pytest.mark.parametrize("taps,dil", [(1, 1), (3, 2)])
def test_conv_gemm_ignores_columns_past_k(cuda, taps, dil):
    """ops.conv_gemm on a view (B, T, 120) of a (B, T, 136) buffer with k = 80: columns 80.. are NaN.  The packed weight is zero
    there, but 0 * NaN is NaN, so the output equals the fp64 conv of the first k columns only if those columns are never read."""
    B, T, k, n = 2, 200, 80, 96
    g = torch.Generator(device="cpu").manual_seed(taps)
    full = torch.full((B, T, 136), float("nan"))
    full[..., :k] = torch.randn(B, T, k, generator=g)
    full = _split(full.to(cuda))
    a = Split(full.hi[..., :120], full.lo[..., :120])
    w = (torch.randn(n, k, taps, generator=g) / math.sqrt(k * taps)).to(cuda)
    wp = ops.pack_weight(w, cuda)
    xv = full.float()[..., :k].double()
    ref = F.conv1d(xv.transpose(1, 2), w.double(), padding=(taps - 1) // 2 * dil, dilation=dil).transpose(1, 2)
    mag = F.conv1d(xv.abs().transpose(1, 2), w.double().abs(), padding=(taps - 1) // 2 * dil, dilation=dil).transpose(1, 2)
    # split-bf16 weight (2^-16 of |w|; the input planes are the reference's own values) and fp32 accumulation over taps * Kp terms
    # (worst case, 2^-23 each)
    bound = (2.0 ** -16 + taps * 128 * 2.0 ** -23) * mag + 1e-30
    for simt in (False, True):
        y, _ = ops.conv_gemm(a, wp, n=n, k=k, taps=taps, dil=dil, simt=simt)
        assert torch.isfinite(y).all(), "simt" if simt else "wgmma"
        assert ((y.double() - ref).abs() <= bound).all(), "simt" if simt else "wgmma"
