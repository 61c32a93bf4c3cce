"""GPU parity tests for the generic kernels, through the C-ABI (run with -m gpu on an H100)."""
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _ref_conv(x, w, bias, taps, dil, act, residual, lens):
    pad = (taps - 1) // 2
    y = F.conv1d(x.transpose(1, 2), w, None, padding=pad * dil, dilation=dil).transpose(1, 2)
    if bias is not None:
        y = y + bias
    if act == "relu":
        y = torch.relu(y)
    if act == "tanh":
        y = torch.tanh(y)
    if residual is not None:
        y = y + residual
    if lens is not None:
        y = y * (torch.arange(y.shape[1], device=y.device)[None, :, None] < lens[:, None, None])
    return y


@pytest.mark.parametrize("B,T,Cin,N,taps,dil,act,res,lens", [
    (1, 128, 64, 64, 1, 1, None, False, False),
    (2, 300, 384, 384, 1, 1, None, False, False),
    (2, 300, 384, 1152, 1, 1, None, False, False),
    (2, 300, 384, 80, 1, 1, None, False, True),      # partial N tile
    (2, 300, 80, 256, 5, 1, "tanh", False, False),    # partial K chunk (postnet first conv)
    (2, 300, 384, 1536, 3, 1, "relu", False, True),   # FFN conv 1
    (2, 300, 1536, 384, 3, 1, None, True, True),      # FFN conv 2 + residual
    (2, 1000, 64, 128, 3, 8, None, False, False),     # dilated
    (1, 3000, 64, 128, 3, 512, None, False, False),   # dilation larger than the tile
    (3, 37, 256, 1, 1, 1, None, False, True),         # predictor head, T < one tile
    (5, 129, 128, 256, 3, 2, "relu", True, True),     # wide N, the second 128-row tile holds a single row
    (40, 448, 384, 1536, 3, 1, "relu", False, True),  # wide N, more tiles (480) than SMs (persistent walk)
    (7, 700, 256, 300, 5, 1, "tanh", False, False),   # partial N tile (300 of 512), partial 128-row tile
    (33, 250, 192, 128, 1, 1, None, True, False),     # single-CTA persistent kernel, more tiles than SMs is not required: odd counts
])
def test_conv_gemm_matches_fp64(cuda, B, T, Cin, N, taps, dil, act, res, lens):
    from parakeet_b200 import ops
    g = torch.Generator(device="cpu").manual_seed(B * 1000 + T + N)
    x = torch.randn(B, T, Cin, generator=g).to(cuda)
    w = (torch.randn(N, Cin, taps, generator=g) / math.sqrt(Cin * taps)).to(cuda)
    b = torch.randn(N, generator=g).to(cuda)
    r = torch.randn(B, T, N, generator=g).to(cuda) if res else None
    ln = torch.randint(max(T // 2, 1), T + 1, (B,), generator=g).to(device=cuda, dtype=torch.int32) if lens else None
    ref = _ref_conv(x.double(), w.double(), b.double(), taps, dil, act, r.double() if res else None, ln)
    y, ys = ops.conv_gemm(ops.Split.from_f32(x), ops.pack_weight(w, cuda), n=N, k=Cin, taps=taps, dil=dil, bias=b, act=act,
                          residual=r, lens=ln, out_f32=True, out_split=True)
    assert rel_err(y, ref) < 5e-5        # tolerance: split-bf16 operands (2^-16) through fp32 accumulation
    assert rel_err(ys.float(), ref) < 5e-5
    ysim, _ = ops.conv_gemm(ops.Split.from_f32(x), ops.pack_weight(w, cuda), n=N, k=Cin, taps=taps, dil=dil, bias=b, act=act,
                            residual=r, lens=ln, simt=True)
    assert rel_err(y, ysim) < 5e-5       # tensor-core path vs plain fp32 FMA path on identical operands


def test_length_regulator_bit_exact(cuda):
    from parakeet_b200 import ops
    g = np.load(os.path.join(GOLD, "length_regulator.npz"))   # the reference's own case (test_expansion.py:20-24)
    y, _ = ops.length_regulate(torch.from_numpy(g["enc"]).to(cuda), torch.from_numpy(g["dur"]).to(cuda), 8)
    assert list(y.shape) == [2, 8, 3]
    assert torch.equal(y.cpu(), torch.from_numpy(g["out"]))
    # ragged, zeros, C not a multiple of 4, split planes
    gen = torch.Generator().manual_seed(0)
    for B, T, C in ((4, 100, 384), (3, 17, 5), (2, 1, 384)):
        x = torch.randn(B, T, C, generator=gen)
        d = torch.randint(0, 13, (B, T), generator=gen)
        d[0, T // 2:] = 0
        lens = ops.length_regulator_lens(d.to(cuda))
        assert lens.cpu().tolist() == d.sum(1).tolist()
        tmax = int(d.sum(1).max())
        y, ys = ops.length_regulate(x.to(cuda), d.to(cuda), tmax, want_split=True)
        for b in range(B):
            idx = torch.repeat_interleave(torch.arange(T), d[b])
            assert torch.equal(y[b, :idx.numel()].cpu(), x[b, idx])                 # bit-exact copies
            assert y[b, idx.numel():].abs().max().item() == 0 if idx.numel() < tmax else True
        assert rel_err(ys.float(), y) < 1e-5
    # all-zero durations: empty output, like the reference (t_dec = 0)
    y, _ = ops.length_regulate(torch.randn(2, 5, 8).to(cuda), torch.zeros(2, 5, dtype=torch.int64).to(cuda), 0)
    assert y.shape[1] == 0


def test_length_regulator_full_size_properties(cuda):
    """cfg3-sized expand (B=32, T<=140, L up to ~1700, C=384): checksum-of-rows property, no oracle needed."""
    from parakeet_b200 import ops
    gen = torch.Generator().manual_seed(3)
    B, T, C = 32, 140, 384
    x = torch.randn(B, T, C, generator=gen).to(cuda)
    d = torch.randint(2, 13, (B, T), generator=gen).to(cuda)
    lens = ops.length_regulator_lens(d)
    tmax = int(lens.max())
    y, _ = ops.length_regulate(x, d, tmax)
    # sum over frames of y == sum_j d_j * x_j (exact in fp64), and every output row equals one source row
    lhs = y.double().sum(1)
    rhs = (x.double() * d.unsqueeze(-1).double()).sum(1)
    assert torch.allclose(lhs, rhs, rtol=1e-9, atol=1e-9)
    assert int((y.abs().sum(-1) > 0).sum()) == int(lens.sum())


def test_row_kernels(cuda):
    from parakeet_b200 import ops
    from oracle import fastspeech2 as ofs
    gen = torch.Generator().manual_seed(0)
    x = torch.randn(3, 50, 384, generator=gen)
    g_, b_ = torch.randn(384, generator=gen), torch.randn(384, generator=gen)
    lens = torch.tensor([50, 20, 37], dtype=torch.int32)
    y, ys = ops.layer_norm(x.to(cuda), g_.to(cuda), b_.to(cuda), lens=lens.to(cuda), want_f32=True)
    ref = F.layer_norm(x, (384,), g_, b_) * (torch.arange(50)[None, :, None] < lens[:, None, None])
    assert rel_err(y, ref) < 1e-5 and rel_err(ys.float(), ref) < 2e-5
    # embedding + scaled positional encoding, padding_idx -> zeros
    table = torch.randn(30, 384, generator=gen)
    ids = torch.randint(0, 30, (3, 50), generator=gen)
    alpha = torch.tensor([0.7])
    e = table[ids]
    e[ids == 0] = 0
    ref = e + alpha * ofs.positional_encoding(50, 384)
    y = ops.embed_pe(ids.to(cuda), table.to(cuda), None, alpha.to(cuda), None)
    assert rel_err(y, ref) < 1e-5
    # masked softmax incl. a fully masked batch entry
    s = torch.randn(2 * 2, 40, 64, generator=gen)
    kl = torch.tensor([33, 0], dtype=torch.int32)
    p = ops.masked_softmax(s.to(cuda), kl.to(cuda), 2, 2, 40, 40).float().cpu()
    ref0 = torch.softmax(s[:2, :, :33], -1)
    assert rel_err(p[:2, :, :33], ref0) < 2e-5 and p[:2, :, 33:].abs().max() == 0 and p[2:].abs().max() == 0
    # duration post-op: round half away from zero, clip at 0, pad -> 0
    xlog = torch.log(torch.tensor([[1.5, 2.5, 3.5, 0.2, 7.49999, 1.0]]))
    d_f, d_i = ops.duration_post(xlog.to(cuda), torch.tensor([5], dtype=torch.int32).to(cuda))
    assert d_i.cpu().tolist() == [[1, 2, 3, 0, 6, 0]]   # exp(x)-1 = .5,1.5,2.5,-.8,6.49999, (padded)
    # z-score
    mu, sg = torch.randn(80, generator=gen), torch.rand(80, generator=gen) + 0.5
    z = torch.randn(7, 80, generator=gen)
    assert rel_err(ops.zscore(z.to(cuda), mu.to(cuda), sg.to(cuda)), (z - mu) / sg) < 1e-6
    assert rel_err(ops.zscore(z.to(cuda), mu.to(cuda), sg.to(cuda), inverse=True), z * sg + mu) < 1e-6


def test_fused_attention_vs_fp64(cuda):
    """pk_fused_attention (scores, key-padding mask, softmax, P.V in one kernel) against an fp64 evaluation of
    attention.py:88-131 on the same split-bf16 inputs: ragged key lengths, query tiles past an utterance's end, T not a
    multiple of the 128-key tile, d_k = 192 (the FastSpeech2 heads) and d_k = 64."""
    import math
    from parakeet_b200 import ops
    g = torch.Generator().manual_seed(11)
    for (B, T, H, dk, lens) in ((3, 300, 2, 192, [300, 131, 17]), (2, 128, 2, 192, None), (2, 77, 4, 64, [77, 5]), (1, 1400, 2, 192, [1333])):
        A = H * dk
        qkv = ops.Split.from_f32((torch.randn(B, T, 3 * A, generator=g) * 1.5).to(cuda))
        kl = torch.tensor(lens, dtype=torch.int32, device=cuda) if lens else None
        ctx = ops.fused_attention(qkv, H, key_lens=kl, row_lens=kl).float().cpu().double()
        x = qkv.float().cpu().double()
        q, k, v = [x[..., i * A:(i + 1) * A].reshape(B, T, H, dk).transpose(1, 2) for i in range(3)]
        s = q @ k.transpose(-1, -2) / math.sqrt(dk)
        keep = torch.ones(B, T, dtype=torch.bool) if lens is None else torch.arange(T)[None, :] < torch.tensor(lens)[:, None]
        s = s.masked_fill(~keep[:, None, None, :], float("-inf"))
        ref = (torch.softmax(s, -1).masked_fill(~keep[:, None, None, :], 0.0) @ v).transpose(1, 2).reshape(B, T, A)
        ref = ref * keep[:, :, None]                                   # rows past an utterance's end are written as zero
        err = (ctx - ref).abs().max().item() / ref.abs().max().item()
        assert err < 2e-5, (B, T, H, dk, err)
        assert ctx[~keep].abs().max().item() == 0 if lens else True


def test_sum_slices_and_splitk_wgrad(cuda):
    """pk_sum_slices (split-K reduction, overwrites its output): the float4 path, the scalar path (n % 4 != 0 or a misaligned
    view of the flat gradient buffer), and wgrad.nt_splitk writing into a non-contiguous destination; the persistent zero
    planes of the transposed operands give the same gradient on a second use with other data.  wgrad.splitk_wgrad, the weight
    gradient the training steps share: a dilated 3-tap conv over padded channel counts and a view of a wider input, and the
    Linear orientation."""
    from parakeet_b200 import ops
    from parakeet_b200.training import wgrad
    g = torch.Generator().manual_seed(21)
    zp = wgrad.ZeroPlanes()
    for s, n, off in ((7, 4096, 0), (128, 384 * 3, 0), (5, 1001, 0), (3, 64, 1)):
        part = torch.randn(s, n, generator=g).to(cuda)
        flat = torch.full((n + 8,), 7.0, device=cuda)            # garbage the call must overwrite
        out = flat[off:off + n]
        ops.sum_slices(part, out)
        ref = part.double().sum(0)
        assert (out.double() - ref).abs().max().item() < 1e-5 * max(1.0, ref.abs().max().item())
        assert flat[off + n:].eq(7.0).all() and flat[:off].eq(7.0).all()
    # dW = X^T dY over (batch, time), with the padded / persistent operand planes used twice
    for rep, (B, T, cin, cout) in enumerate(((3, 150, 96, 200), (3, 150, 96, 200), (8, 700, 96, 200))):   # S = 1, 1, > 1
        x = torch.randn(B, T, cin, generator=g).to(cuda)
        dy = torch.randn(B, T, cout, generator=g).to(cuda)
        Tp, S, ks, KKp = wgrad.plan(B, T, cin, cout)
        xs, dys = ops.Split.from_f32(x), ops.Split.from_f32(dy)
        xt = zp.get(("test_xt", B, T), (cin, KKp), cuda)
        dyt = zp.get(("test_dyt", B, T), (cout, KKp), cuda)
        ops.transpose_planes(xs, z=B, rows=T, src_zstride=T * cin, ld_src=cin, c0=0, cols=cin, shift=0, r_out=T, dst=xt, dst_zstride=Tp, ld_dst=KKp)
        ops.transpose_planes(dys, z=B, rows=T, src_zstride=T * cout, ld_src=cout, c0=0, cols=cout, shift=0, r_out=T, dst=dyt, dst_zstride=Tp,
                             ld_dst=KKp)
        big = torch.zeros(cin, cout + 8, device=cuda)
        out = big[:, :cout] if rep == 1 else torch.empty(cin, cout, device=cuda)  # second pass: non-contiguous destination
        got = wgrad.nt_splitk(xt, dyt, cin, cout, S, ks, KKp, out=out)
        ref = torch.einsum("btc,btd->cd", xs.float().double().cpu(), dys.float().double().cpu())
        err = (got.double().cpu() - ref).abs().max().item() / ref.abs().max().item()
        assert err < 2e-5, (rep, S, err)
        assert rep != 2 or S > 1
    # the shared weight gradient, twice over the same planes: dW[j] = dY^T shift(X, shifts[j]), rows past either end of an utterance are zero
    B, T, cin, cout, dil = 8, 700, 40, 20, 3                                      # S > 1
    for rep in range(2):
        wide = ops.Split.from_f32(torch.randn(B, T, cin + 8, generator=g).to(cuda))
        xs = ops.Split(wide.hi[:, :, :cin], wide.lo[:, :, :cin])                  # a view: the source strides are the wide tensor's
        dys = ops.split_pad8(torch.randn(B, T, cout, generator=g).to(cuda))       # 20 -> 24 columns, the last four zero
        xd, dyd = xs.float().double().cpu(), dys.float().double().cpu()
        shifts = [-dil, 0, dil]
        got = wgrad.splitk_wgrad(zp, xs, dys, 24, cin, shifts)
        assert got.shape == (3, 24, cin) and got[:, cout:].abs().max().item() == 0
        for j, sh in enumerate(shifts):
            xsh = torch.zeros_like(xd)
            xsh[:, max(0, -sh):T - max(0, sh)] = xd[:, max(0, sh):T - max(0, -sh)]
            ref = torch.einsum("btd,btc->dc", dyd, xsh)
            assert (got[j].double().cpu() - ref).abs().max().item() / ref.abs().max().item() < 2e-5, (rep, sh)
        big = torch.zeros(cin, cout + 4, device=cuda)
        out = big[:, :cout] if rep else torch.empty(cin, cout, device=cuda)
        lin = wgrad.splitk_wgrad(zp, xs, dys, cout, cin, [0], x_first=True, out=out)
        ref = torch.einsum("btc,btd->cd", xd, dyd[..., :cout])
        assert lin is out and (lin.double().cpu() - ref).abs().max().item() / ref.abs().max().item() < 2e-5, rep


@pytest.mark.parametrize("shape,linear,dil,pad", [
    ((64, 1, 1), False, 1, None),      # PWG first_conv: 1-channel input
    ((64, 1, 3), False, 1, None),      # PWG discriminator, first layer
    ((1, 64, 3), False, 2, None),      # PWG discriminator, last layer: 1-channel output
    ((1, 64, 1), False, 1, None),      # PWG last_conv_layers.3
    ((1, 8, 3), False, 1, None),
    ((128, 64, 3), False, 4, None),    # dilated
    ((80, 80, 5), False, 1, None),
    ((64, 80, 1), False, 1, None),
    ((128, 128, 4), False, 1, 1),      # SpeedySpeech even kernel: one more row on the right
    ((384, 1), True, 1, None),         # Paddle Linear [in, out]
    ((96, 200), True, 1, None),
])
def test_conv_ops_equal_the_per_step_formulations(cuda, shape, linear, dil, pad):
    """training/conv.py ConvOps against the packings it replaced, restated here: FastSpeech2 / SpeedySpeech (Linear transposed
    for the forward, Conv1D taps flipped for the data gradient) and Parallel WaveGAN (Cin zero-padded to the operand width for
    the forward, Cout padded to 8 in the data-gradient pack, the weight gradient over the padded widths, then sliced).  Packs
    (both planes), GEMM outputs and weight gradients are compared bit for bit."""
    from parakeet_b200 import ops
    from parakeet_b200.ops import pack_dev, pad8
    from parakeet_b200.training import wgrad
    from parakeet_b200.training.conv import ConvOps
    g = torch.Generator().manual_seed(sum(shape) + dil)
    B, T = 3, 150
    zp = wgrad.ZeroPlanes()
    zp.begin(("test", B, T))
    conv = ConvOps(zp)
    w = torch.randn(*shape, generator=g).to(cuda)
    cout, cin, taps = (shape[1], shape[0], 1) if linear else shape
    x = ops.Split.from_f32(pad8(torch.randn(B, T, cin, generator=g)).to(cuda))        # a 1-channel input rides 8 wide
    dys = ops.split_pad8(torch.randn(B, T, cout, generator=g).to(cuda))
    same = lambda a, b: torch.equal(a.hi, b.hi) and torch.equal(a.lo, b.lo)
    y = conv.fwd(x, "w", w, linear=linear, dil=dil, pad=pad)[0]
    dx = conv.dgrad(dys, "w", w, linear=linear, dil=dil, pad=pad)
    dw = conv.wgrad(x, dys, w, linear=linear, dil=dil, pad=pad)
    pf, pb = conv.packs[("f", "w")], conv.packs[("b", "w")]
    if linear:
        old_f, old_b = pack_dev(w.t().contiguous()), pack_dev(w)                         # FastSpeech2 w_fwd / w_bwd, SpeedySpeech lin_*
        assert same(pf, old_f) and same(pb, old_b)
        assert torch.equal(y, ops.conv_gemm(x, old_f, n=cout, k=cin)[0])
        assert torch.equal(dx, ops.conv_gemm(dys, old_b, n=cin, k=cout)[0])
        assert torch.equal(dw, wgrad.splitk_wgrad(zp, x, dys, cout, cin, [0], x_first=True))
        return
    cin_p, cout_p = x.hi.shape[-1], dys.hi.shape[-1]
    wp = torch.zeros(cout, cin_p, taps, device=cuda)
    wp[:, :cin] = w
    old_f = pack_dev(wp)                                                                   # PWG _ConvOps.fwd
    old_b = pack_dev(pad8(w.flip(-1).permute(1, 2, 0)).permute(0, 2, 1))                 # PWG _ConvOps.dgrad
    assert same(pf, pack_dev(w)) and same(pf, old_f)                                       # FastSpeech2 w_fwd, SpeedySpeech block_fwd
    assert same(pb, pack_dev(w.flip(-1).permute(1, 0, 2).contiguous())) and same(pb, old_b)   # FastSpeech2 w_bwd, SpeedySpeech block_bwd
    assert torch.equal(y, ops.conv_gemm(x, old_f, n=cout, k=cin_p, taps=taps, dil=dil, pad=pad)[0])
    assert torch.equal(dx, ops.conv_gemm(dys, old_b, n=cin, k=cout_p, taps=taps, dil=dil, pad=None if pad is None else taps - 1 - pad)[0])
    left = (taps - 1) // 2 if pad is None else pad
    old_w = wgrad.splitk_wgrad(zp, x, dys, cout_p, cin_p, [(tap - left) * dil for tap in range(taps)])[:, :cout, :cin].permute(1, 2, 0)
    assert dw.shape == w.shape and torch.equal(dw, old_w)
