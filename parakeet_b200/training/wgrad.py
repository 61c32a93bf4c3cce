"""Split-K weight gradients: dW = A^T-style NT matmuls whose reduction axis is the flattened (batch, time) axis (10^4 .. 10^6)
while the output is a handful of 128 x N tiles.  K is cut into S slices so that tiles x S fills the machine: S independent NT
matmuls (`pk_conv_gemm` batched over the slices) whose fp32 partial results are summed by `pk_sum_slices`.  `splitk_wgrad` is the
weight gradient of a Conv1D or Linear layer as the FastSpeech2, SpeedySpeech and Parallel WaveGAN steps compute it."""
import torch

from .. import ops
from ..ops import Split


class ZeroPlanes:
    """Persistent zero-initialised split planes for the transposed GEMM operands of the weight gradients.

    `transpose_planes` rewrites the same valid region on every use of a (role, shape) key within one batch geometry and never
    touches the K padding, so the zeros are written once per geometry instead of by a fill kernel per use (~250 launches per
    FastSpeech2 step).  Buffers are filed under the current GEOMETRY (`begin(geom)`: the batch shape - it fixes every valid
    region, and a captured CUDA graph of that batch shape has the buffer addresses baked in).  At most `max_geoms` geometries
    are kept (LRU): evicting one frees its planes and calls `on_evict(geom)` so that the owner drops the graph captured for it.
    `role` keeps operands that are alive together apart."""

    def __init__(self, max_geoms=16, on_evict=None):
        self.max_geoms, self.on_evict = max_geoms, on_evict
        self._geoms = {}          # geom -> {(role, shape, device): Split}; insertion order = LRU order
        self._cur = None

    def begin(self, geom):
        """Make `geom` current (most recently used), evicting the least recently used geometries beyond the bound."""
        planes = self._geoms.pop(geom, None)
        self._geoms[geom] = planes if planes is not None else {}
        self._cur = geom
        while len(self._geoms) > self.max_geoms:
            old = next(iter(self._geoms))
            del self._geoms[old]
            if self.on_evict is not None:
                self.on_evict(old)

    touch = begin

    def get(self, role, shape, dev):
        if self._cur is None:
            self.begin(None)
        planes = self._geoms[self._cur]
        key = (role, tuple(shape), str(dev))
        buf = planes.get(key)
        if buf is None:
            buf = planes[key] = Split.zeros(tuple(shape), dev)
        return buf

    def __len__(self):
        return len(self._geoms)


def plan(batch, t, m, n, max_slices=128):
    """-> (Tp, S, ks, KKp): padded time, number of K slices, slice length (multiple of 64), padded reduction length S * ks."""
    tp = (t + 63) // 64 * 64
    kk = batch * tp
    tiles = ((m + 127) // 128) * ((n + 127) // 128)
    s = max(1, min(max_slices, kk // 512, -(-296 // tiles)))          # ~2 tiles per SM
    ks = ((kk + s - 1) // s + 63) // 64 * 64
    return tp, s, ks, s * ks


def nt_splitk(at, bt, m, n, s, ks, kkp, out=None):
    """at Split (m rows, kkp), bt Split (n rows, kkp) -> (m, n) fp32 = at . bt^T, reduced over the S slices."""
    dev = at.hi.device
    sa = dict(rows=m, cols=ks, ld=kkp, batch_stride=ks, batches=s, bmul=1, hmul=0, col0=0, colh=0)
    sb = dict(rows=n, cols=ks, ld=kkp, batch_stride=ks, batches=s, bmul=1, hmul=0, col0=0, colh=0)
    direct = out is not None and out.is_contiguous()
    if s == 1:
        y = out if direct else torch.empty(m, n, dtype=torch.float32, device=dev)
        ops.batched_matmul_nt(at, bt, batch=1, heads=1, m=m, n=n, k=ks, a_spec=sa, b_spec=sb, y_f32=y, y_batch_stride=0, y_head_stride=0, y_ld=n)
        if out is not None and not direct:
            out.copy_(y)
            return out
        return y
    part = torch.empty(s, m, n, dtype=torch.float32, device=dev)
    ops.batched_matmul_nt(at, bt, batch=s, heads=1, m=m, n=n, k=ks, a_spec=sa, b_spec=sb, y_f32=part, y_batch_stride=m * n, y_head_stride=0,
                          y_ld=n)
    y = out if direct else torch.empty(m, n, dtype=torch.float32, device=dev)
    ops.sum_slices(part, y)
    if out is not None and y is not out:
        out.copy_(y)
        return out
    return y


def splitk_wgrad(zp, x, dys, rows_dy, rows_x, shifts, x_first=False, out=None):
    """Conv1D weight gradient, one plane per tap: -> fp32 (len(shifts), rows_dy, rows_x),
    [j] = sum over (b, t) of dY[b, t, :rows_dy]^T X[b, t + shifts[j], :rows_x].
    x, dys: Split (B, T, >= rows_x) saved input (may be a view) and (B, T, >= rows_dy) output gradient; zp: the caller's ZeroPlanes.
    (rows_dy, rows_x) also fix the number of K slices, i.e. the summation order.
    x_first (Paddle Linear weight [in, out]; one shift): the operands swapped, (rows_x, rows_dy) written into `out`.
    Allocates and launches on the current stream only."""
    B, T = x.hi.shape[0], x.hi.shape[1]
    dev = x.hi.device
    Tp, S, ks, KKp = plan(B, T, rows_dy, rows_x)
    ld = dys.hi.shape[2]
    dyt = zp.get(("dyt", B, T), (rows_dy, KKp), dev)
    ops.transpose_planes(dys, z=B, rows=T, src_zstride=T * ld, ld_src=ld, c0=0, cols=rows_dy, shift=0, r_out=T, dst=dyt, dst_zstride=Tp,
                         ld_dst=KKp)

    def shifted(sh):                                          # ONE plane, rewritten per tap
        xt = zp.get(("xt", B, T), (rows_x, KKp), dev)
        ops.transpose_planes(x, z=B, rows=T, src_zstride=x.hi.stride(0), ld_src=x.hi.stride(1), c0=0, cols=rows_x, shift=sh, r_out=T, dst=xt,
                             dst_zstride=Tp, ld_dst=KKp)
        return xt

    if x_first:
        return nt_splitk(shifted(shifts[0]), dyt, rows_x, rows_dy, S, ks, KKp, out=out)
    res = torch.empty(len(shifts), rows_dy, rows_x, dtype=torch.float32, device=dev)
    for j, sh in enumerate(shifts):
        nt_splitk(dyt, shifted(sh), rows_dy, rows_x, S, ks, KKp, out=res[j])
    return res
