"""The persistent LSTM recurrence kernels (csrc/lstm.cu) where one CTA serves several row tiles per step, and the GE2E glue kernels
at their edges, each against a plain fp64 evaluation of the same operation on the same fp32 inputs.

pk_lstm_fwd / pk_lstm_bwd run a grid of (hidden slice, row-tile group) CTAs; CTA (s, g) walks the row tiles g, g + groups, ...
of every step.  The groups are limited by how many CTAs are co-resident, so a large row count makes `tiles > groups` and a CTA
serves several tiles per step, publishing each through its own (step, tile) counter.  Every case below asserts that it really
reaches that branch, with the co-resident count bounded from the device's SM count and the kernels' shared memory.

Bounds.  u = 2^-24 is the fp32 unit roundoff.  The recurrence GEMMs are wgmma in bf16x3: each operand is held as a split-bf16
pair to 2^-16 of its magnitude, so a K-term product errs by at most 2^-15 of sum |w x|; for the random-sign operands used here
sum |w x| / |sum w x| grows like sqrt(K), so one step's gate error is about 2^-15 sqrt(K) of the gate scale (5e-4 at K = H = 256,
1e-3 at K = 4H = 1024 in the backward).  The forget gate (< 1) makes the forward recurrence contractive, so the error of h and c
stays at that level over T; the backward accumulates dc through the same gates.  The GE2E loss kernel works in double, so its
outputs are held to fp32 output rounding (2^-24 relative) plus double-precision noise."""
import pytest
import torch
import torch.nn.functional as F

from parakeet_b200 import ops
from parakeet_b200.models.lstm_speaker_encoder import start_states

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24


@pytest.fixture(autouse=True)
def _needs_cuda(cuda):
    """Skips without a CUDA device (the session fixture of conftest.py)."""


def _gen(seed):
    return torch.Generator(device="cpu").manual_seed(seed)


def _rel(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def _l2(a, b):
    a, b = a.double().cpu(), b.double().cpu()
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def _within(got, ref, bound, what):
    got, ref = got.double().cpu(), ref.double().cpu()
    bound = (bound.double().cpu() if torch.is_tensor(bound) else bound) + 1e-300
    err = (got - ref).abs()
    assert torch.isfinite(got).all(), what
    worst = float((err / bound).max())
    print(f"{what}: max err {float(err.max()):.3e}, worst err / bound {worst:.3f}")
    assert worst <= 1.0, f"{what}: max err {float(err.max()):.3e}, worst err / bound {worst:.2f}"


# ---------------------------------------------------------------------------------------------------------------------------
# LSTM schedule: tiles > groups
# ---------------------------------------------------------------------------------------------------------------------------
KCHUNK = 64             # csrc/lstm.cu: kChunkK (K columns per TMA box)


def smem_of(H, kernel):
    """Dynamic shared memory of lstm_{fwd,bwd}_kernel<H> (csrc/lstm.cu Geo<H>: kFwdSmem / kBwdSmem)."""
    w_chunk, h_chunk = 2 * 4 * ops.LSTM_SLICE * 128, 2 * ops.LSTM_ROWS * 128
    if kernel == "fwd":
        return 1024 + (H // KCHUNK) * (w_chunk + h_chunk) + 64
    return 1024 + (4 * H // KCHUNK) * (2 * ops.LSTM_SLICE * 128) + 4 * h_chunk + 64


def max_ctas_bound(H, kernel):
    """An upper bound on the co-resident CTAs of the kernel: shared memory per SM over the CTA's (with the 1 KB the runtime
    reserves per CTA), times the SM count.  Registers can only lower the true count, which only lowers `groups`."""
    prop = torch.cuda.get_device_properties(DEV)
    per_sm = prop.shared_memory_per_multiprocessor // (smem_of(H, kernel) + 1024)
    assert per_sm >= 1
    return per_sm * prop.multi_processor_count


def assert_multi_tile(rows, H, kernel):
    slices, tiles, groups, grid = ops.lstm_schedule(rows, H, max_ctas_bound(H, kernel))
    assert grid > 0 and tiles > groups, (rows, H, kernel, tiles, groups)
    return tiles, groups


def cell_ref(g_in, b_hh, w_hh, h0, c0):
    """fp64 recurrence of one layer, time-major g_in (T, rows, 4H) -> (h (T+1, rows, H), c (T+1, rows, H), gates (T, rows, 4H))."""
    h, c, gs = [h0], [c0], []
    for t in range(g_in.shape[0]):
        i, f, g, o = (g_in[t] + b_hh + h[-1] @ w_hh.t()).chunk(4, 1)
        i, f, g, o = torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)
        c.append(f * c[-1] + i * g)
        h.append(o * torch.tanh(c[-1]))
        gs.append(torch.cat([i, f, g, o], 1))
    return torch.stack(h), torch.stack(c), torch.stack(gs)


def lstm_inputs(seed, T, rows, H, init):
    g = _gen(seed)
    g_in = torch.randn(T, rows, 4 * H, generator=g) * 0.5
    w_hh = (torch.rand(4 * H, H, generator=g) * 2 - 1) / H ** 0.5
    b_hh = torch.randn(4 * H, generator=g) * 0.1
    h0 = torch.randn(rows, H, generator=g) * 0.3 if init else torch.zeros(rows, H)
    c0 = torch.randn(rows, H, generator=g) * 0.3 if init else torch.zeros(rows, H)
    return g_in.to(DEV), w_hh.to(DEV), b_hh.to(DEV), h0.to(DEV), c0.to(DEV)


def beyond_groups(H, kernel):
    """A row count with more tiles than the kernel's largest possible group count, and a partial last tile."""
    return ops.LSTM_ROWS * (max_ctas_bound(H, kernel) // (H // ops.LSTM_SLICE)) + 37


# 2500 rows = 40 tiles, the last one partial (4 rows), spread unevenly over the groups; at H = 64 (rows = 0: beyond_groups), four
# 50 KB CTAs fit an SM, so it takes ~17 000 rows
@pytest.mark.parametrize("rows,T,H", [(2500, 40, 256), (0, 6, 64)])
def test_lstm_fwd_tiles_beyond_groups(rows, T, H):
    rows = rows or beyond_groups(H, "fwd")
    tiles, groups = assert_multi_tile(rows, H, "fwd")
    g_in, w_hh, b_hh, h0, c0 = lstm_inputs(rows + T, T, rows, H, init=True)
    h_ref, c_ref, g_ref = cell_ref(g_in.double(), b_hh.double(), w_hh.double(), h0.double(), c0.double())
    wp = ops.lstm_pack_fwd(w_hh, ops.lstm_gate_perm(H, DEV))
    # c in place (c_step = 0): only c_T survives
    h_all, h_split, c = start_states(T, rows, H, DEV, h0, c0)
    ops.lstm_fwd(g_in, b_hh, wp, h_all, h_split, c)
    # keeping every c_t and the gates (the training layout)
    h2, h2_split, c_all = start_states(T, rows, H, DEV, h0, c0, keep_c=True)
    gates = torch.empty(T, rows, 4 * H, device=DEV)
    ops.lstm_fwd(g_in, b_hh, wp, h2, h2_split, c_all, gates)
    torch.cuda.synchronize()
    # 2^-15 sqrt(256) = 4.9e-4 of the gate scale per step (module docstring), contractive over T: 1e-3 of each tensor's max,
    # checked per step so a tile served second or third by its CTA cannot hide behind the others
    for t in range(T + 1):
        assert _rel(h_all[t], h_ref[t]) < 1e-3, ("h", t, _rel(h_all[t], h_ref[t]))
        assert _rel(c_all[t], c_ref[t]) < 1e-3, ("c_all", t, _rel(c_all[t], c_ref[t]))
    for t in range(T):
        assert _rel(gates[t], g_ref[t]) < 1e-3, ("gates", t)
    print(f"rows {rows} H {H}: tiles {tiles} > groups {groups}; h {_rel(h_all, h_ref):.2e} c {_rel(c, c_ref[-1]):.2e} "
          f"gates {_rel(gates, g_ref):.2e}")
    assert _rel(c, c_ref[-1]) < 1e-3
    # both layouts run the same arithmetic
    assert torch.equal(h2, h_all) and torch.equal(c_all[-1], c)
    # every row of the partial last tile is written
    assert torch.isfinite(h_all).all()


@pytest.mark.parametrize("rows,T,H,with_dh_in", [(2500, 40, 256, False), (2500, 40, 256, True), (640, 160, 256, False),
                                                 (640, 160, 256, True), (0, 6, 64, True)])
def test_lstm_bwd_tiles_beyond_groups(rows, T, H, with_dh_in):
    """rows = 640, T = 160 is the GE2E recipe's shape (10 tiles, one per group); the others serve several tiles per CTA."""
    rows = rows or beyond_groups(H, "bwd")
    if rows != 640:
        assert_multi_tile(rows, H, "bwd")
    g_in, w_hh, b_hh, _, _ = lstm_inputs(7 * rows + T, T, rows, H, init=False)
    g = _gen(rows + 3 * T)
    dh_in = (torch.randn(T, rows, H, generator=g) if with_dh_in else torch.zeros(T, rows, H)).to(DEV)
    dh_last = torch.randn(rows, H, generator=g).to(DEV)
    gi = g_in.double().requires_grad_(True)
    z = torch.zeros(rows, H, dtype=torch.float64, device=DEV)
    h, _, _ = cell_ref(gi, b_hh.double(), w_hh.double(), z, z)
    ((h[1:] * dh_in.double()).sum() + (h[-1] * dh_last.double()).sum()).backward()
    h_all, h_split, c_all = start_states(T, rows, H, DEV, keep_c=True)
    gd = torch.empty(T, rows, 4 * H, device=DEV)
    ops.lstm_fwd(g_in, b_hh, ops.lstm_pack_fwd(w_hh, ops.lstm_gate_perm(H, DEV)), h_all, h_split, c_all, gd)
    dg = torch.empty(T, rows, 4 * H, device=DEV)
    split = ops.Split.empty((T, rows, 4 * H), DEV)
    # dh_in = None is GE2E's case: only the last step's dh enters
    ops.lstm_bwd(ops.lstm_pack_bwd(w_hh), gd, c_all, dh_in if with_dh_in else None, dh_last, dg, split)
    torch.cuda.synchronize()
    # 2^-15 sqrt(4H) = 1e-3 per step (module docstring) on top of the forward's 1e-3 in the saved gates; the error is compared
    # in L2 over each step's tile of rows (a steady 1e-3 per step compounds a few-fold through dc over the steps)
    ref = gi.grad
    worst = max(_l2(dg[t], ref[t]) for t in range(T) if float(ref[t].norm()) > 0)
    print(f"rows {rows} T {T} H {H} dh_in {with_dh_in}: worst per-step L2 {worst:.2e}, overall {_l2(dg, ref):.2e}")
    assert worst < 5e-3
    assert torch.equal(split.hi.float() + split.lo.float(), ops.Split.from_f32(dg).float())


# ---------------------------------------------------------------------------------------------------------------------------
# GE2E loss kernel (double) against fp64 autograd
# ---------------------------------------------------------------------------------------------------------------------------
def _embeds(seed, N, M, C, near_dup=False):
    """L2-normalised non-negative rows like the encoder's (ReLU then F.normalize); near_dup makes each speaker's utterances
    copies of one row perturbed by 1e-4."""
    g = _gen(seed)
    if near_dup:
        base = torch.rand(N, 1, C, generator=g)
        e = base + 1e-4 * torch.rand(N, M, C, generator=g)
    else:
        e = torch.relu(torch.randn(N, M, C, generator=g) + 0.3)
    e = F.normalize(e.reshape(N * M, C), dim=1)
    return e.float()


@pytest.mark.parametrize("near_dup", [False, True])
@pytest.mark.parametrize("N,M,C", [(2, 2, 64), (4, 2, 256), (64, 40, 64), (7, 3, 256)])
def test_ge2e_loss_against_fp64_autograd(N, M, C, near_dup):
    from oracle import ge2e as og
    e = _embeds(N * 100 + M * 10 + C + near_dup, N, M, C, near_dup)
    w, b = torch.tensor([10.0]), torch.tensor([-5.0])
    loss, sim, de, dw, db = ops.ge2e_loss(e.to(DEV), N, M, C, w.to(DEV), b.to(DEV), want_grads=True)
    ed, wd, bd = (x.double().requires_grad_(True) for x in (e, w, b))
    l_ref, s_ref = og.loss(ed.reshape(N, M, C), wd, bd)
    de_ref, dw_ref, db_ref = torch.autograd.grad(l_ref, (ed, wd, bd))
    # the kernel's arithmetic is double (relative error ~ C 2^-53 of the terms' magnitudes, < 1e-12 of the outputs' scale);
    # each output is then rounded once to fp32: 2^-24 of its own magnitude
    tol = lambda r, scale: U * r.abs() + 1e-12 * scale
    _within(loss, l_ref.detach().reshape(1), tol(l_ref.detach().reshape(1), float(l_ref.detach().abs())), f"loss {N}x{M}x{C}")
    s_ref = s_ref.detach()
    _within(sim, s_ref, tol(s_ref, float(s_ref.abs().max())), "similarity")
    de_ref = de_ref.reshape(N * M, C)
    _within(de, de_ref, tol(de_ref, float(de_ref.abs().max())), "d_embeds")
    # do_gradient_ops: dw and db times 0.01
    _within(dw, 0.01 * dw_ref, tol(0.01 * dw_ref, float(0.01 * dw_ref.abs())), "dw")
    # db = 0.01 * sum of (softmax - onehot) / NM: zero but for the double rounding of NM N terms of size <= 1 / NM
    _within(db, 0.01 * db_ref, 0.01 * N * 1e-15 + U * float(db_ref.abs()), "db")


# ---------------------------------------------------------------------------------------------------------------------------
# GE2E embedding backward and segment mean
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n", [64, 256, 257])
def test_ge2e_embed_bwd_zero_rows_and_eps(n):
    rows = 37
    g = _gen(n)
    z = torch.randn(rows, n, generator=g)
    z[3] = -torch.rand(n, generator=g)                  # entirely negative: ReLU zeroes the row
    z[4] = 0.0                                           # entirely zero
    z[5] = -z[5].abs()
    z[5, 7] = 0.5                                        # one positive entry
    z[6] *= 2e-12 / float(torch.relu(z[6]).norm())       # norm 2e-12: above eps, the projection branch
    z[7] *= 0.5e-12 / float(torch.relu(z[7]).norm())     # norm 5e-13: below eps, F.normalize divides by eps
    z[8] *= 1e3
    z = z.float()
    dy = torch.randn(rows, n, generator=g).float()
    e = torch.relu(z)
    dz = ops.ge2e_embed_bwd(e.to(DEV), dy.to(DEV), eps=1e-12)
    zd = z.double().requires_grad_(True)
    (F.normalize(torch.relu(zd), dim=1, eps=1e-12) * dy.double()).sum().backward()
    ref = zd.grad
    # fp32: |e|^2 and e . dy are lane-strided sums of depth d = n / 32 + 5 (each within d u of the sum of its terms' magnitudes);
    # sqrt, the division by |e|^2 and the final division each add a few u.  Per element:
    #   |err| <= (d + 8) u (|dy| + |e| (sum |e dy| + |e . dy|) / |e|^2) / max(|e|, eps)
    ed, dyd = e.double(), dy.double()
    nrm = ed.norm(dim=1, keepdim=True)
    proj_mag = ((ed * dyd).abs().sum(1, keepdim=True) + (ed * dyd).sum(1, keepdim=True).abs()) / nrm.clamp_min(1e-300) ** 2
    proj_mag = torch.where(nrm > 1e-12, proj_mag, torch.zeros_like(proj_mag))
    bound = (n / 32 + 5 + 8) * U * (dyd.abs() + ed * proj_mag) / nrm.clamp_min(1e-12)
    _within(dz, ref, bound * (ed > 0), f"embed_bwd n={n}")
    for r in (3, 4):
        assert torch.equal(dz[r].cpu(), torch.zeros(n))
    assert dz[7].abs().max() > 1e11                      # dy / eps on the positive entries


def test_segment_mean_normalize_edges():
    n = 256
    g = _gen(5)
    x = torch.randn(1500, n, generator=g) + 0.2
    # empty, one row, 1000 rows, offsets not starting at 0, an empty segment between two others, and one at the very end
    offsets = torch.tensor([17, 17, 18, 1018, 1050, 1050, 1499, 1500], dtype=torch.int32)
    y = ops.segment_mean_normalize(x.to(DEV), offsets.to(DEV))
    assert y.shape == (7, n)
    xd = x.double()
    for s in range(7):
        a, b = int(offsets[s]), int(offsets[s + 1])
        if a == b:
            assert torch.equal(y[s].cpu(), torch.zeros(n)), s
            continue
        m = xd[a:b].mean(0)
        ref = m / m.norm().clamp_min(1e-12)
        # the mean is a sequential fp32 sum over the L = b - a rows: within (L - 1) u of sum |x| / L, then one division; the norm
        # is a strided sum of depth n / 256 + 5 + 8; per element:
        #   |err| <= (L + 2) u mean|x| / |m| + (n / 256 + 16) u |y|
        L = b - a
        bound = (L + 2) * U * xd[a:b].abs().mean(0) / m.norm() + (n / 256 + 16) * U * ref.abs()
        _within(y[s], ref, bound, f"segment {s} ({L} rows)")
