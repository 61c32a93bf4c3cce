"""The row-wise and reduction kernels shared by the training steps (csrc/train.cu, gan.cu, fs2.cu, stft.cu), each against an fp64
autograd or closed-form restatement at the shapes where such kernels go wrong: partial row / column blocks, padding columns,
accumulating outputs, ties and clips.

Every bound below is an elementwise worst case built from the arithmetic: u = 2^-24 is the fp32 unit roundoff (2^-23 where the
order or rounding of a sum is not known), a sum evaluated with a tree / sequence of depth D errs by at most D * 2^-23 of the sum of
the magnitudes of its terms, and split-bf16 planes hold a value to 2^-16 of its magnitude."""
import math

import pytest
import torch
import torch.nn.functional as F

from parakeet_b200 import _lib, ops
from parakeet_b200.ops import Split, _ptr, _stream

pytestmark = pytest.mark.gpu
U = 2.0 ** -23          # unit of the worst-case bounds (one fp32 rounding, order unknown)
SPLIT = 2.0 ** -16      # split-bf16 representation of an fp32 value
SPLIT_ABS = 2.0 ** -133  # ... and of an fp32 subnormal: the lo plane's bf16 subnormal spacing


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _within(got, ref, bound, what):
    got, ref = got.double(), ref.double()
    err = (got - ref).abs()
    bound = (bound.double() if torch.is_tensor(bound) else bound) + 1e-300
    assert torch.isfinite(got).all(), what
    assert (err <= bound).all(), f"{what}: max err {err.max().item():.3e}, worst err / bound {(err / bound).max().item():.2f}"


def _L():
    return _lib.lib()


# ---------------------------------------------------------------------------------------------------------------------------
# LayerNorm backward
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [80, 256, 257, 384, 512])
@pytest.mark.parametrize("rows", [37, 1003])
def test_layer_norm_bwd(cuda, d, rows):
    g = _gen(d * 10 + rows)
    x = (torch.randn(rows, d, generator=g) * 2 + 0.5).to(cuda)
    gamma = (1 + 0.3 * torch.randn(d, generator=g)).to(cuda)
    dy = torch.randn(rows, d, generator=g).to(cuda)
    dx0 = torch.randn(rows, d, generator=g).to(cuda)
    dg0, db0 = torch.randn(d, generator=g).to(cuda), torch.randn(d, generator=g).to(cuda)
    xd = x.double().requires_grad_(True)
    gd = gamma.double().requires_grad_(True)
    bd = torch.zeros(d, dtype=torch.float64, device=cuda, requires_grad=True)
    F.layer_norm(xd, (d,), gd, bd, eps=1e-5).backward(dy.double())
    # magnitudes: xhat, g = dy * gamma, the row means of g and g * xhat
    mean, var = x.double().mean(-1, keepdim=True), x.double().var(-1, unbiased=False, keepdim=True)
    rstd = (var + 1e-5).rsqrt()
    xh = (x.double() - mean) * rstd
    gg = dy.double() * gamma.double()
    mag_dx = rstd * (gg.abs() + gg.abs().mean(-1, keepdim=True) + xh.abs() * (gg * xh).abs().mean(-1, keepdim=True))
    # row sums of d terms (mean, variance, the two means of g) in warp order: depth d / 32 + 5 each, four of them chained into each
    # output, and xhat / rstd through them: (4 (d / 32 + 5) + 2 d / 32 + 16) * U of the magnitudes (the d-term sums enter via xhat)
    tol_row = (6 * (d // 32 + 6) + 16) * U
    for accumulate in (False, True):
        dx = dx0.clone()
        dgam, dbet = dg0.clone(), db0.clone()
        ops.layer_norm_bwd(x, gamma, dy, dx, accumulate, dgam, dbet)
        ref = xd.grad + (dx0.double() if accumulate else 0)
        _within(dx, ref, tol_row * (mag_dx + xh.abs() * mag_dx) + U * ref.abs(), f"dx accumulate={accumulate}")
        # dgamma / dbeta: per-block shared-memory atomics (<= 8 rows) then one global atomic per block onto the start value
        depth = 8 + (rows + 7) // 8 + 1
        _within(dgam, dg0.double() + gd.grad, (depth * U + tol_row) * ((dy.double() * xh).abs().sum(0) + dg0.double().abs()), "dgamma")
        _within(dbet, db0.double() + bd.grad, depth * U * (dy.double().abs().sum(0) + db0.double().abs()), "dbeta")
        xd.grad, gd.grad, bd.grad = None, None, None
        F.layer_norm(xd, (d,), gd, bd, eps=1e-5).backward(dy.double())


# ---------------------------------------------------------------------------------------------------------------------------
# softmax backward
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("keys", [1, 31, 33, 300])
@pytest.mark.parametrize("scale", [1.0, 0.125])
def test_softmax_bwd(cuda, keys, scale):
    g = _gen(keys)
    rows, ld = 77, ops.ceil_to(keys, 64) + 64
    logits = torch.randn(rows, keys, generator=g)
    p32 = torch.full((rows, ld), 7.0)                 # padding columns: live garbage the kernel must ignore
    p32[:, :keys] = torch.softmax(logits, -1)
    dp = torch.randn(rows, ld, generator=g) * 3
    p, dp = Split.from_f32(p32.to(cuda)), dp.to(cuda)
    ds = ops.softmax_bwd(p, dp, keys, scale)
    pv = p.float().double()[:, :keys]
    dpv = dp.double()[:, :keys]
    dot = (pv * dpv).sum(-1, keepdim=True)
    ref = scale * pv * (dpv - dot)
    # dot: `keys` terms, depth keys / 32 + 5; then two roundings; then the split of the output
    bound = scale * pv * ((keys // 32 + 8) * U * ((pv * dpv).abs().sum(-1, keepdim=True) + dpv.abs())) + SPLIT * ref.abs()
    out = ds.float()
    _within(out[:, :keys], ref, bound, "ds")
    assert (ds.hi[:, keys:] == 0).all() and (ds.lo[:, keys:] == 0).all(), "padding columns must be exactly zero"


# ---------------------------------------------------------------------------------------------------------------------------
# column sums (bias gradients): accumulate onto `out`
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [1, 63, 65, 5601])
@pytest.mark.parametrize("c", [1, 80, 129])
def test_colsum(cuda, rows, c):
    g = _gen(rows + c)
    x = torch.randn(rows, c, generator=g).to(cuda)
    out0 = torch.randn(c, generator=g).to(cuda)
    out = out0.clone()
    ops.colsum_(x, out)
    # per thread <= 16 sequential rows, 4 partials, one atomic per 64-row block onto the start value
    depth = 16 + 4 + (rows + 63) // 64 + 1
    _within(out, out0.double() + x.double().sum(0), depth * U * (x.double().abs().sum(0) + out0.double().abs()), "colsum")


@pytest.mark.parametrize("rows", [1, 63, 65, 5601])
@pytest.mark.parametrize("c", [1, 80, 129])
def test_colsum_split(cuda, rows, c):
    g = _gen(rows * 3 + c)
    ld = ops.ceil_to(c, 8) + 8
    x = torch.full((rows, ld), 1.0e6)                 # columns past `cols`: large, must not be summed
    x[:, :c] = torch.randn(rows, c, generator=g)
    xs = Split.from_f32(x.to(cuda))
    out0 = torch.randn(c + 4, generator=g).to(cuda)
    out = out0.clone()
    ops.colsum_split_(xs, c, out)
    xv = xs.float().double()[:, :c]
    depth = 16 + 4 + (rows + 63) // 64 + 1
    _within(out[:c], out0[:c].double() + xv.sum(0), depth * U * (xv.abs().sum(0) + out0[:c].double().abs()), "colsum_split")
    assert torch.equal(out[c:], out0[c:]), "colsum_split wrote past cols"


# ---------------------------------------------------------------------------------------------------------------------------
# BatchNorm1D, train mode (postnet of the FastSpeech2 step)
# ---------------------------------------------------------------------------------------------------------------------------
def _bn_train(x, gamma, beta, act, run_mean, run_var, momentum=0.9, eps=1e-5, want_split=True):
    rows, c = x.shape
    dev = x.device
    y = torch.empty_like(x)
    ys = Split.empty((rows, c), dev) if want_split else None
    sums = torch.empty(2 * c, device=dev)
    mean, rstd = torch.empty(c, device=dev), torch.empty(c, device=dev)
    _lib.check(_L().pk_batch_norm_train(_ptr(x), rows, c, _ptr(gamma), _ptr(beta), eps, act, momentum, _ptr(run_mean), _ptr(run_var),
                                        _ptr(sums), _ptr(y), _ptr(ys.hi) if ys else None, _ptr(ys.lo) if ys else None, _ptr(mean),
                                        _ptr(rstd), _stream()), "pk_batch_norm_train")
    return y, ys, mean, rstd


@pytest.mark.parametrize("act", [0, 2])
@pytest.mark.parametrize("rows,c,offset", [(1001, 80, 0.0), (130, 257, 0.0), (5003, 80, 30.0)])
def test_batch_norm_train_and_bwd(cuda, act, rows, c, offset):
    """offset 30: columns whose mean is large against their spread (30 + N(0, 1)), where E[x^2] - mean^2 cancels."""
    g = _gen(rows + c + act)
    x = (offset + torch.randn(rows, c, generator=g) * (0.5 + torch.rand(c, generator=g))).to(cuda)
    gamma = (1 + 0.2 * torch.randn(c, generator=g)).to(cuda)
    beta = (0.1 * torch.randn(c, generator=g)).to(cuda)
    rm0, rv0 = torch.randn(c, generator=g).to(cuda), (1 + torch.rand(c, generator=g)).to(cuda)
    rm, rv = rm0.clone(), rv0.clone()
    y, ys, mean, rstd = _bn_train(x, gamma, beta, act, rm, rv)
    xd = x.double()
    m_ref, v_ref = xd.mean(0), xd.var(0, unbiased=False)
    rstd_ref = (v_ref + 1e-5).rsqrt()
    # a numerically sound fp32 evaluation: the mean and the variance are sums of `rows` terms (depth <= rows / 4 + 16 + 4 + 1 in this
    # kernel's order: 16 rows per thread, 4 partials, one atomic per 64-row block); the variance's terms are (x - mean)^2, so its
    # error is that depth times the variance itself, not times E[x^2]
    depth = 16 + 4 + (rows + 63) // 64 + 4
    _within(mean, m_ref, depth * U * xd.abs().mean(0), "batch mean")
    _within(rstd, rstd_ref, (depth * U + 4 * U) * rstd_ref, "batch rstd")
    _within(rm, 0.9 * rm0.double() + 0.1 * m_ref, depth * U * (xd.abs().mean(0) + rm0.double().abs()) + 4 * U * rm0.double().abs(),
            "running mean")
    _within(rv, 0.9 * rv0.double() + 0.1 * v_ref, (depth + 4) * U * (v_ref + rv0.double()), "running var (biased)")
    # y from the kernel's own mean / rstd errors propagated: |dmean| rstd + |x - mean| rstd |drstd / rstd| + a few roundings
    xh_ref = (xd - m_ref) * rstd_ref
    pre = xh_ref * gamma.double() + beta.double()
    y_ref = torch.tanh(pre) if act == 2 else pre
    dpre = gamma.double().abs() * (depth * U * xd.abs().mean(0) * rstd_ref + xh_ref.abs() * (depth + 4) * U) + 4 * U * pre.abs()
    _within(y, y_ref, dpre + 2 * U * y_ref.abs(), "y")
    _within(ys.float(), y_ref, dpre + (2 * U + SPLIT) * y_ref.abs(), "y split")

    # backward, given the kernel's saved mean / rstd and activation output (its own inputs): closed form in fp64
    dy = torch.randn(rows, c, generator=g).to(cuda)
    dx = torch.empty_like(x)
    sums = torch.empty(2 * c, device=cuda)
    _lib.check(_L().pk_batch_norm_bwd(_ptr(x), _ptr(dy), _ptr(y), _ptr(mean), _ptr(rstd), _ptr(gamma), act, rows, c, _ptr(sums), _ptr(dx),
                                      _stream()), "pk_batch_norm_bwd")
    gd = dy.double() * ((1 - y.double() ** 2) if act == 2 else 1.0)
    xh = (xd - mean.double()) * rstd.double()
    s1, s2 = gd.sum(0), (gd * xh).sum(0)
    N = float(rows)
    ref = gamma.double() * rstd.double() / N * (N * gd - s1 - xh * s2)
    mag = gamma.double().abs() * rstd.double() / N * (N * gd.abs() + gd.abs().sum(0) + xh.abs() * (gd * xh).abs().sum(0))
    _within(dx, ref, (depth + 8) * U * mag, "dx")
    _within(sums[:c], s1, depth * U * gd.abs().sum(0) + 4 * U * gd.abs().sum(0), "dbeta")
    _within(sums[c:], s2, (depth + 4) * U * (gd * xh).abs().sum(0), "dgamma")


# ---------------------------------------------------------------------------------------------------------------------------
# ReLU / LeakyReLU
# ---------------------------------------------------------------------------------------------------------------------------
EDGES = [0.0, -0.0, 1e-30, 2.0 ** -126, 1e-38, -1e-30, -2.0 ** -126, 3.0, -3.0]


def _edge_tensor(n, seed):
    x = torch.randn(n, generator=_gen(seed))
    x[:len(EDGES)] = torch.tensor(EDGES)
    x[len(EDGES):2 * len(EDGES)] = torch.tensor(EDGES)
    return x


def test_relu_bwd(cuda):
    n = 1000 + 37
    y = torch.relu(_edge_tensor(n, 1))
    y[:len(EDGES)] = torch.tensor(EDGES).clamp_min(0.0)       # relu outputs: exact 0, -0 (clamp keeps it) and tiny positives
    y[1] = -0.0
    ys = Split.from_f32(y.to(cuda))
    dy = torch.randn(n, generator=_gen(2)).to(cuda)
    dx, dxs = ops.relu_bwd(dy, ys, want_f32=True)
    ref = torch.where(y.to(cuda) > 0, dy, torch.zeros_like(dy))
    assert torch.equal(dx, ref)
    _within(dxs.float(), ref, SPLIT * ref.abs() + SPLIT_ABS, "relu_bwd split")


@pytest.mark.parametrize("slope", [0.2, 0.0])
def test_leaky_relu_fwd_bwd(cuda, slope):
    n = 4096 + 7
    x = _edge_tensor(n, 3).to(cuda)
    y = torch.empty_like(x)
    ys = Split.empty((n,), cuda)
    _lib.check(_L().pk_leaky_relu(_ptr(x), n, slope, _ptr(y), _ptr(ys.hi), _ptr(ys.lo), _stream()), "pk_leaky_relu")
    ref = torch.where(x > 0, x, x * slope)          # x == 0 (either sign) takes the slope branch, as Paddle's leaky_relu does
    assert torch.equal(y, ref)
    _within(ys.float(), ref, SPLIT * ref.abs() + SPLIT_ABS, "leaky_relu split")
    dy = torch.randn(n, generator=_gen(4)).to(cuda)
    dx = torch.empty_like(x)
    _lib.check(_L().pk_leaky_relu_bwd(_ptr(x), _ptr(dy), n, slope, _ptr(dx), _stream()), "pk_leaky_relu_bwd")
    assert torch.equal(dx, torch.where(x > 0, dy, dy * slope))
    assert torch.equal(dx[:2], dy[:2] * slope), "x = +-0 must take the slope branch"


# ---------------------------------------------------------------------------------------------------------------------------
# Embedding + scaled positional encoding backward
# ---------------------------------------------------------------------------------------------------------------------------
def _pe_angles(T, d, dev):
    """The fp32 angles of the positional encoding (oracle.fastspeech2.positional_encoding), as float64."""
    position = torch.arange(0, T, dtype=torch.float32).unsqueeze(1)
    div_term = torch.exp(torch.arange(0, d, 2, dtype=torch.float32) * -(math.log(10000.0) / d))
    return (position * div_term).double().to(dev)


@pytest.mark.parametrize("B,T,d,with_ids", [(3, 37, 384, True), (2, 1700, 384, True), (2, 1700, 256, False), (4, 5, 80, False)])
def test_embed_pe_bwd(cuda, B, T, d, with_ids):
    g = _gen(T + d)
    V, pad = 11, 0
    dx = torch.randn(B, T, d, generator=g).to(cuda)
    ids = torch.randint(0, V, (B, T), generator=g)
    ids[0, :3] = pad
    ids[:, -1] = 5                                     # one id repeated in every utterance
    ids = ids.to(cuda)
    dtab0 = torch.randn(V, d, generator=g).to(cuda)
    dal0 = torch.tensor([0.25], device=cuda)
    dtab, dal = dtab0.clone(), dal0.clone()
    _lib.check(_L().pk_embed_pe_bwd(_ptr(ids) if with_ids else None, _ptr(dx), V if with_ids else 0, pad, B, T, d,
                                    _ptr(dtab) if with_ids else None, _ptr(dal), _stream()), "pk_embed_pe_bwd")
    ang = _pe_angles(T, d, cuda)
    pe = torch.zeros(T, d, dtype=torch.float64, device=cuda)
    pe[:, 0::2], pe[:, 1::2] = torch.sin(ang), torch.cos(ang)
    terms = dx.double() * pe
    ref = dal0.double() + terms.sum()
    # the angle t * exp(-c ln(10000) / d) in fp32, on either side: the exponent's two roundings times |exponent| * freq <= 1/e,
    # expf's ulp and the product's rounding stay below t * 2^-22 each, so the two angles differ by < t * 2^-21; sinf / cosf by 2^-22;
    # the sum: d / 32 per lane, 5 + 3 in the block, then one atomic per block of 8 rows
    t = torch.arange(T, device=cuda, dtype=torch.float64)[None, :, None]
    depth = d // 32 + 8 + B * T // 8 + 2
    bound = (dx.double().abs() * (t * 2.0 ** -21 + 2.0 ** -21)).sum() + depth * U * (terms.abs().sum() + 0.25)
    _within(dal, ref, bound, "dalpha")
    if with_ids:
        oh = F.one_hot(ids.long(), V).double()
        oh[..., pad] = 0
        scatter = torch.einsum("btv,btd->vd", oh, dx.double())
        cnt = oh.sum((0, 1))[:, None]
        _within(dtab, dtab0.double() + scatter, (cnt + 1) * U * (torch.einsum("btv,btd->vd", oh, dx.double().abs()) + dtab0.double().abs()),
                "dtable")
        assert torch.equal(dtab[pad], dtab0[pad]), "the padding row gets no gradient"


# ---------------------------------------------------------------------------------------------------------------------------
# FastSpeech2Loss forward + backward
# ---------------------------------------------------------------------------------------------------------------------------
def test_fs2_loss_and_bwd(cuda):
    from oracle.fastspeech2 import fs2_loss
    g = _gen(7)
    B, L, T, odim = 3, 150, 40, 80
    olens = torch.tensor([150, 97, 3], dtype=torch.int32)
    ilens = torch.tensor([40, 23, 1], dtype=torch.int32)
    ys = torch.randn(B, L, odim, generator=g)
    before, after = torch.randn(B, L, odim, generator=g), torch.randn(B, L, odim, generator=g)
    before[0, :5] = ys[0, :5]                          # prediction == target: L1 subgradient 0
    after[1, 10, :7] = ys[1, 10, :7]
    ds = torch.randint(0, 6, (B, T), generator=g)
    ds[0, :4] = 0                                      # durations of 0: target log(0 + 1) = 0
    d_outs, p_outs, e_outs = torch.randn(B, T, generator=g), torch.randn(B, T, 1, generator=g), torch.randn(B, T, 1, generator=g)
    ps, es = torch.randn(B, T, 1, generator=g), torch.randn(B, T, 1, generator=g)
    dv = [t.to(cuda).contiguous() for t in (before, after, ys, d_outs, ds, p_outs, ps, e_outs, es)]
    bo, ao, yy, do_, dd, po, pp, eo, ee = dv
    ol, il = olens.to(cuda), ilens.to(cuda)
    ws = torch.empty(12, device=cuda)
    out = torch.empty(4, device=cuda)
    _lib.check(_L().pk_fs2_loss(_ptr(bo), _ptr(ao), _ptr(yy), _ptr(ol), L, odim, _ptr(do_), _ptr(dd), _ptr(po), _ptr(pp), _ptr(eo), _ptr(ee),
                                _ptr(il), T, B, _ptr(ws), _ptr(out), _stream()), "pk_fs2_loss")
    grads = [torch.empty_like(t) for t in (bo, ao, do_, po, eo)]
    _lib.check(_L().pk_fs2_loss_bwd(_ptr(bo), _ptr(ao), _ptr(yy), _ptr(ol), L, odim, _ptr(do_), _ptr(dd), _ptr(po), _ptr(pp), _ptr(eo),
                                    _ptr(ee), _ptr(il), T, B, *[_ptr(t) for t in grads], _stream()), "pk_fs2_loss_bwd")
    # the oracle's duration target is log(ds + 1) in fp32 (DurationPredictorLoss): the duration term is restated in fp64 on that
    # target below, the other three go through the oracle's autograd in fp64
    leaves = [t.double().requires_grad_(True) for t in (after, before, p_outs, e_outs)]
    l1, _, pit, ene = fs2_loss(leaves[0], leaves[1], d_outs, leaves[2], leaves[3], ys.double(), ds, ps.double(), es.double(),
                               ilens.long(), olens.long())
    (l1 + pit + ene).backward()
    a_g, b_g, p_g, e_g = [t.grad.to(cuda) for t in leaves]
    # losses: the kernel's sums run strided per thread, 5 + 3 in the block, then one atomic per block (<= 4 per SM), and a divide
    blocks = min((B * L * odim + 255) // 256, 4 * torch.cuda.get_device_properties(cuda).multi_processor_count)
    depth = (B * L * odim + blocks * 256 - 1) // (blocks * 256) + 8 + blocks + 2
    m = (torch.arange(L)[None, :] < olens[:, None].long())[..., None].double()
    tk = (torch.arange(T)[None, :] < ilens[:, None].long()).double()
    nm, nt = m.sum() * odim, tk.sum()
    tgt = torch.log(ds.to(torch.float32) + 1.0).double()
    dur = ((d_outs.double() - tgt) ** 2 * tk).sum() / nt
    d_g = (2 * (d_outs.double() - tgt) * tk / nt).to(cuda)
    mags = [(((before.double() - ys.double()).abs() + (after.double() - ys.double()).abs()) * m).sum() / nm,
            ((d_outs.double() - tgt) ** 2 * tk).sum() / nt + 4 * U * (tgt.abs() * (d_outs.double() - tgt).abs() * tk).sum() / nt,
            ((p_outs.double()[..., 0] - ps.double()[..., 0]) ** 2 * tk).sum() / nt,
            ((e_outs.double()[..., 0] - es.double()[..., 0]) ** 2 * tk).sum() / nt]
    for i, (got, ref) in enumerate(zip(out, (l1, dur, pit, ene))):
        _within(got, ref.detach().to(cuda), (depth + 4) * U * mags[i].to(cuda), f"loss[{i}]")
    # gradients: +-1 / (frames * odim) or 0 exactly up to the reciprocal; 2 (d - log(ds + 1)) / tokens up to logf and three roundings
    _within(grads[0], b_g, 2 * U * b_g.abs(), "d before")
    _within(grads[1], a_g, 2 * U * a_g.abs(), "d after")
    assert (grads[0][0, :5] == 0).all() and (grads[1][1, 10, :7] == 0).all(), "L1 subgradient at a tie must be 0"
    assert (grads[0][1, 97:] == 0).all() and (grads[2][2, 1:] == 0).all(), "padded frames / tokens get no gradient"
    tgt_c = tgt.to(cuda)
    _within(grads[2], d_g, 6 * U * (d_g.abs() + 2 * tgt_c.abs() * tk.to(cuda) / nt.item()), "d d_outs")
    _within(grads[3], p_g[..., 0].contiguous().view_as(grads[3]), 6 * U * p_g.abs().view_as(grads[3]), "d p_outs")
    _within(grads[4], e_g[..., 0].contiguous().view_as(grads[4]), 6 * U * e_g.abs().view_as(grads[4]), "d e_outs")


# ---------------------------------------------------------------------------------------------------------------------------
# length regulator backward
# ---------------------------------------------------------------------------------------------------------------------------
def test_length_regulate_bwd(cuda):
    g = _gen(9)
    B, T, C, t_out = 3, 17, 130, 60
    dur = torch.randint(0, 5, (B, T), generator=g)
    dur[0, ::3] = 0                                   # zero durations
    dur[1] = 6                                        # sum 102 > t_out: the tail tokens are truncated
    dur[2] = 0
    dur[2, 4] = 2
    dy = torch.randn(B, t_out, C, generator=g)
    dy_d, dur_d = dy.to(cuda), dur.to(cuda)            # device copies held for the launch
    dx = torch.empty(B, T, C, device=cuda)
    _lib.check(_L().pk_length_regulate_bwd(_ptr(dy_d), _ptr(dur_d), B, T, C, t_out, _ptr(dx), _stream()), "pk_length_regulate_bwd")
    ref = torch.zeros(B, T, C, dtype=torch.float64)
    mag = torch.zeros(B, T, C, dtype=torch.float64)
    for b in range(B):
        start = 0
        for j in range(T):
            e = min(start + int(dur[b, j]), t_out)
            if e > start:
                ref[b, j] = dy[b, start:e].double().sum(0)
                mag[b, j] = dy[b, start:e].double().abs().sum(0) * (e - start)
            start += int(dur[b, j])
    _within(dx, ref.to(cuda), U * mag.to(cuda), "length_regulate_bwd")


# ---------------------------------------------------------------------------------------------------------------------------
# Conv1D(1 -> C, k) weight gradient on a scalar track (pitch / energy embeddings)
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [1, 3, 5, 15])
@pytest.mark.parametrize("B,T", [(3, 45), (2, 3)])
def test_scalar_conv_wgrad(cuda, k, B, T):
    g = _gen(k * 100 + T)
    C = 384
    dhs = torch.randn(B, T, C, generator=g).to(cuda)
    track = torch.randn(B, T, generator=g).to(cuda)
    dw0, db0 = torch.randn(C, k, generator=g).to(cuda), torch.randn(C, generator=g).to(cuda)
    dw, db = dw0.clone(), db0.clone()
    _lib.check(_L().pk_scalar_conv_wgrad(_ptr(dhs), _ptr(track), B, T, C, k, _ptr(dw), _ptr(db), _stream()), "pk_scalar_conv_wgrad")
    pad = (k - 1) // 2
    tp = F.pad(track.double(), (pad, k - 1 - pad))
    win = tp.unfold(1, k, 1)                          # (B, T, k): track[b, t + q - pad]
    ref = torch.einsum("btc,btq->cq", dhs.double(), win)
    mag = torch.einsum("btc,btq->cq", dhs.double().abs(), win.abs())
    depth = 64 + (B * T + 63) // 64 + 1              # 64 rows per block sequentially, one atomic per block
    _within(dw, dw0.double() + ref, depth * U * (mag + dw0.double().abs()), "dw")
    _within(db, db0.double() + dhs.double().sum((0, 1)), depth * U * (dhs.double().abs().sum((0, 1)) + db0.double().abs()), "db")


# ---------------------------------------------------------------------------------------------------------------------------
# MSE against a constant and the squared sum (double accumulators), beyond 2^24 elements
# ---------------------------------------------------------------------------------------------------------------------------
def test_mse_const_and_sq_sum_large(cuda):
    n = (1 << 24) + 4099
    ld, col = 3, 2
    g = torch.Generator(device=cuda).manual_seed(11)
    x = torch.randn(n, ld, device=cuda, generator=g)
    acc = torch.tensor([0.5], dtype=torch.float64, device=cuda)
    dx = torch.full((n, ld), 9.0, device=cuda)
    coef, target = 2.0 / n, 0.3
    _lib.check(_L().pk_mse_const(_ptr(x), n, ld, col, target, _ptr(acc), _ptr(dx), coef, _stream()), "pk_mse_const")
    d = x[:, col].double() - target
    # each term: a subtraction and a fused multiply-add (2 U of d^2); the block sum: two warp trees, depth 10; double atomics
    _within(acc, 0.5 + (d * d).sum(), 12 * U * (d * d).sum(), "mse sum")
    _within(dx[:, col], coef * d, 2 * U * (coef * d).abs() + U * coef * abs(target), "mse dx")
    assert (dx[:, :col] == 9.0).all(), "pk_mse_const wrote outside its column"
    y = x[:, 0].contiguous()
    sq = torch.tensor([1.0], dtype=torch.float64, device=cuda)
    _lib.check(_L().pk_sq_sum(_ptr(y), n, _ptr(sq), _stream()), "pk_sq_sum")
    per_thread = (n + 2048 * 256 - 1) // (2048 * 256)   # grid-stride over at most 2048 blocks
    _within(sq, 1.0 + (y.double() ** 2).sum(), (per_thread + 12) * U * (y.double() ** 2).sum(), "sq_sum")


# ---------------------------------------------------------------------------------------------------------------------------
# Parallel WaveGAN generator residual / skip update
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("init", [1, 0])
def test_pwg_res_update(cuda, init):
    g = _gen(13 + init)
    rows = 1000 + 3
    so, x = torch.randn(rows, 128, generator=g).to(cuda), torch.randn(rows, 64, generator=g).to(cuda)
    skips0 = torch.randn(rows, 64, generator=g).to(cuda)
    skips = skips0.clone()
    xo = torch.empty(rows, 64, device=cuda)
    xos = Split.empty((rows, 64), cuda)
    _lib.check(_L().pk_pwg_res_update(_ptr(so), _ptr(x), rows, _ptr(skips), init, _ptr(xo), _ptr(xos.hi), _ptr(xos.lo), _stream()),
               "pk_pwg_res_update")
    assert torch.equal(skips, so[:, :64] if init else skips0 + so[:, :64]), "skips: = on the first layer, += after"
    ref = (so[:, 64:].double() + x.double()) * math.sqrt(0.5)
    _within(xo, ref, 2 * U * (so[:, 64:].double().abs() + x.double().abs()), "x'")
    _within(xos.float(), ref, (2 * U + SPLIT) * (so[:, 64:].double().abs() + x.double().abs()), "x' split")
    dsk, dxo = torch.randn(rows, 64, generator=g).to(cuda), torch.randn(rows, 64, generator=g).to(cuda)
    dso = torch.full((rows, 128), float("nan"), device=cuda)
    dx = torch.full((rows, 64), float("nan"), device=cuda)
    _lib.check(_L().pk_pwg_res_update_bwd(_ptr(dsk), _ptr(dxo), rows, _ptr(dso), _ptr(dx), _stream()), "pk_pwg_res_update_bwd")
    assert torch.equal(dso[:, :64], dsk)
    _within(dso[:, 64:], dxo.double() * math.sqrt(0.5), U * dxo.double().abs(), "dso out half")
    assert torch.equal(dx, dso[:, 64:]), "the residual gradient is written (not accumulated) and equals the out half"


# ---------------------------------------------------------------------------------------------------------------------------
# multi-resolution STFT loss backward: the loss sums, the gradient w.r.t. re / im, and the framing adjoint, per resolution
# ---------------------------------------------------------------------------------------------------------------------------
RES = [(1024, 120, 600), (2048, 240, 1200), (512, 50, 240)]     # (n_fft, hop, win_length) of the recipes' MultiResolutionSTFTLoss


def _spectra(B, bins, frames, seed):
    """x / y spectra (re, im) with a silent stretch in x (power below the 1e-7 clip), bins where x == y exactly, and elsewhere
    magnitude ratios bounded away from 1 (no near-ties of the log-magnitude sign)."""
    g = _gen(seed)
    xre, xim = torch.randn(B, bins, frames, generator=g), torch.randn(B, bins, frames, generator=g)
    ratio = 1 + (0.1 + 0.4 * torch.rand(B, bins, frames, generator=g)) * torch.where(torch.rand(B, bins, frames, generator=g) < 0.5, -1, 1)
    rot = torch.rand(B, bins, frames, generator=g) * 6.28
    mag = ratio * torch.sqrt(xre ** 2 + xim ** 2)
    yre, yim = mag * torch.cos(rot), mag * torch.sin(rot)
    s = frames // 3
    xre[:, :, s:s + 4] = 1e-5 * xre[:, :, s:s + 4]     # silent stretch in x: power ~1e-10 < 1e-7
    xim[:, :, s:s + 4] = 1e-5 * xim[:, :, s:s + 4]
    e = 2 * frames // 3
    yre[:, :, e:e + 3], yim[:, :, e:e + 3] = xre[:, :, e:e + 3], xim[:, :, e:e + 3]       # x == y
    return xre, xim, yre, yim, (s, e)


@pytest.mark.parametrize("n_fft,hop,win", RES)
def test_stft_loss_grad_and_sums(cuda, n_fft, hop, win):
    B, T = 2, 4001
    bins, frames = n_fft // 2 + 1, 1 + T // hop
    bins_p = ops.ceil_to(bins, 64)
    xre, xim, yre, yim, (s, e) = _spectra(B, bins, frames, n_fft)
    mx64 = torch.sqrt(torch.clamp(xre.double() ** 2 + xim.double() ** 2, min=1e-7))
    my64 = torch.sqrt(torch.clamp(yre.double() ** 2 + yim.double() ** 2, min=1e-7))
    d = [t.to(cuda).contiguous() for t in (xre, xim, yre, yim)]
    # pk_spectral_loss_sums on the fp32 magnitudes the STFT kernel would give
    xm, ym = mx64.float().to(cuda), my64.float().to(cuda)
    sums = torch.empty(3, device=cuda)
    _lib.check(_L().pk_spectral_loss_sums(_ptr(xm), _ptr(ym), xm.numel(), 1e-7, _ptr(sums), _stream()), "pk_spectral_loss_sums")
    xv, yv = xm.double(), ym.double()
    n = xm.numel()
    blocks = min((n + 255) // 256, 4 * torch.cuda.get_device_properties(cuda).multi_processor_count)
    depth = (n + blocks * 256 - 1) // (blocks * 256) + 8 + blocks + 2
    lg = (torch.log(yv) - torch.log(xv)).abs()
    _within(sums[0], ((yv - xv) ** 2).sum(), (depth + 3) * U * ((yv - xv) ** 2).sum(), "sum (y - x)^2")
    _within(sums[1], (yv ** 2).sum(), (depth + 2) * U * (yv ** 2).sum(), "sum y^2")
    _within(sums[2], lg.sum(), depth * U * lg.sum() + 4 * U * (torch.log(yv).abs() + torch.log(xv).abs()).sum(), "sum |log y - log x|")
    # the gradient kernel, given exact sums: fp64 autograd of sc + mag (one resolution, weight w)
    w = 1.0 / 3
    sums_ref = torch.stack([((my64 - mx64) ** 2).sum(), (my64 ** 2).sum(), torch.zeros((), dtype=torch.float64)]).float().to(cuda)
    gbuf = torch.zeros(B * frames, 2 * bins_p, device=cuda)
    _lib.check(_L().pk_stft_loss_grad(*[_ptr(t) for t in d], B, bins, frames, bins_p, _ptr(sums_ref), w, _ptr(gbuf), _stream()),
               "pk_stft_loss_grad")
    re_, im_ = xre.double().requires_grad_(True), xim.double().requires_grad_(True)
    mx = torch.sqrt(torch.clamp(re_ ** 2 + im_ ** 2, min=1e-7))
    loss = torch.norm(my64 - mx, p="fro") / torch.norm(my64, p="fro") + F.l1_loss(torch.log(mx), torch.log(my64))
    (w * loss).backward()
    g3 = gbuf.reshape(B, frames, 2 * bins_p)
    got_re, got_im = g3[:, :, :bins].transpose(1, 2), g3[:, :, bins_p:bins_p + bins].transpose(1, 2)
    # a dozen fp32 operations on each term: the sc term c (mx - my) / mx (mx - my rounds to 2^-23 of mx + my) and the log term
    # c' / mx^2, each times |re| or |im|
    c_sc = w / (torch.sqrt(((my64 - mx64) ** 2).sum()) * torch.sqrt((my64 ** 2).sum()))
    term = (c_sc * (mx64 + my64) / mx64 + w / n / mx64 ** 2) * 16 * U
    _within(got_re, re_.grad.to(cuda), (term * xre.double().abs()).to(cuda), "d re")
    _within(got_im, im_.grad.to(cuda), (term * xim.double().abs()).to(cuda), "d im")
    assert (got_re[:, :, s:s + 4] == 0).all() and (got_im[:, :, s:s + 4] == 0).all(), "clipped power: zero gradient"
    assert (gbuf.reshape(B * frames, 2, bins_p)[:, :, bins:] == 0).all(), "bin padding must stay zero"


@pytest.mark.parametrize("n_fft,hop,win", RES)
@pytest.mark.parametrize("T", [4001, 1100])
def test_frames_overlap_add(cuda, n_fft, hop, win, T):
    """The adjoint of framing: reflect-pad n_fft / 2 on both sides (T = 1100 with n_fft = 2048 folds frames over both ends at once),
    cut frames at hop, multiply by the window; fp64 autograd of that framing (oracle.stft's window) is the reference."""
    from oracle.stft import make_window
    B = 2
    frames = 1 + T // hop
    g = _gen(n_fft + T)
    fg = torch.randn(B * frames, n_fft, generator=g).to(cuda)
    winv = torch.tensor(make_window("hann", win, n_fft), dtype=torch.float32).to(cuda)
    dx0 = torch.randn(B, T, generator=g).to(cuda)
    dx = dx0.clone()
    _lib.check(_L().pk_frames_overlap_add(_ptr(fg), _ptr(winv), B, frames, n_fft, hop, T, _ptr(dx), _stream()), "pk_frames_overlap_add")

    def framing(x):
        xp = F.pad(x[:, None], (n_fft // 2, n_fft // 2), mode="reflect")[:, 0]
        return xp.unfold(1, n_fft, hop) * winv.double()          # (B, frames, n_fft)

    xd = torch.zeros(B, T, dtype=torch.float64, device=cuda, requires_grad=True)
    (framing(xd) * fg.double().reshape(B, frames, n_fft)).sum().backward()
    xa = torch.zeros(B, T, dtype=torch.float64, device=cuda, requires_grad=True)
    (framing(xa) * fg.double().abs().reshape(B, frames, n_fft)).sum().backward()       # sum of |terms| per position (|win| = win)
    cnt = 2 * (n_fft + hop - 1) // hop + 2                                               # terms landing on one sample, both folds
    _within(dx, dx0.double() + xd.grad, (cnt + 2) * U * (xa.grad + dx0.double().abs()), "overlap-add")
