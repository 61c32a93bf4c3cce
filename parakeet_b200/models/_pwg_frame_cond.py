"""Frame-rate conditioning for the Parallel WaveGAN residual stack (every config frame_rate_exact accepts; DESIGN.md 7.2).

The upsampling network of ConvInUpsampleNet (parallel_wavegan.py:119-138,201-216) is linear and acts on every channel
alike, so the 1x1 aux convolution of a residual block (:300-303) commutes with it:

    conv1x1_aux(upsample(m'))[t, n] = sum_j U[t, j] * P[j, n],        m' = conv_in(mel),  P = W_aux m'   (frame rate)

U (T x frames) is banded: row t has at most 4 non-zero frames starting at t // hop - 2, it repeats with period hop away from
the ends of the utterance, and the zero-padding of the FIR stages only changes rows within 95 samples of either end
(scripts/ptrick_study.py).  A 256-sample pair tile starting at t0 therefore needs the K = 16 frames j0 .. j0 + 15,
j0 = floor8(t0 // hop - 2) (the window start is aligned to 8 frames = 16 bytes for TMA), and its A operand is the "tile-relative band table": row t holds U[t, j0(tile of t) + k], k < 16.
This module builds that table on the host (constants of the model, computed once per utterance length); the layer kernel
multiplies it with the matching window of P, frames outside [0, frames) reading as zero (TMA out-of-bounds fill).
"""
import torch
import torch.nn.functional as F

TILE = 256          # rows of a band-table window: both 128-row tiles of the window multiply with the SAME 16-frame window of P
KWIN = 16
EDGE = 128          # rows next to either end of an utterance that carry their own coefficients (exact while edge_reach <= EDGE)


def edge_reach(scales):
    """Samples next to either end of an utterance whose upsampled conditioning depends on the zero padding of the FIR stages
    after the first: sum over i >= 1 of s_i * prod_{k > i} s_k.  The first stage's padding needs no table rows of its own:
    it is the same as zero frames outside [0, frames), which the kernel reads as zero."""
    reach = 0
    for s in scales[1:]:
        reach = (reach + 1) * s
    return reach


def frame_rate_exact(scales):
    """True when the compact band tables reproduce the upsampled conditioning exactly: a 256-row tile touches at most two
    frames, so the 8-frame windows of its rows fit its 16-frame K window (hop >= 256, which pk_pwg_residual_layer_fc also
    requires), and the padding effects stay inside the EDGE rows that carry their own coefficients."""
    hop = 1
    for s in scales:
        hop *= s
    return hop >= TILE and edge_reach(scales) <= EDGE


def window_start(t0, hop):
    """First frame of the 16-frame K window of the tile starting at sample t0 (python ints or tensors): floor8(t0 // hop - 2)."""
    return (t0 // hop - 2) // 8 * 8


def upsample_operator(firs, scales, frames):
    """U (frames * hop, frames) in float64: column j = response of the stretch / FIR cascade to an impulse at frame j."""
    x = torch.eye(frames, dtype=torch.float64)[None, None]            # (1, 1, frames 'channels', frames)
    for fir, s in zip(firs, scales):
        x = F.interpolate(x, scale_factor=(1, s), mode="nearest")      # Stretch2D (:48-63)
        x = F.conv2d(x, fir.reshape(1, 1, 1, -1).to(torch.float64), padding=(0, s))
    return x[0, 0].transpose(0, 1).contiguous()                        # (T, frames)


def _row_windows(U, hop, width):
    """rows[t, k] = U[t, t // hop - 2 + k] (zero outside the matrix); asserts that nothing lies outside the window."""
    T, Fr = U.shape
    t = torch.arange(T)
    j = (t // hop - 2)[:, None] + torch.arange(width)[None, :]
    ok = (j >= 0) & (j < Fr)
    rows = torch.where(ok, U[t[:, None].expand_as(j), j.clamp(0, Fr - 1)], torch.zeros((), dtype=U.dtype))
    assert torch.allclose(rows.sum(1), U.sum(1), atol=1e-12), "upsampling operator is wider than the K window"
    return rows


def tile_band_table(firs, scales, frames, width=8):
    """(frames * hop, KWIN) float64: row t = U[t, j0 + k] with j0 = window_start(t // TILE * TILE, hop) (tile-relative window)."""
    hop = 1
    for s in scales:
        hop *= s
    T = frames * hop
    ref_frames = 8
    if frames <= ref_frames or T < 2 * EDGE + hop:
        rows = _row_windows(upsample_operator(firs, scales, frames), hop, width)
    else:
        ref = _row_windows(upsample_operator(firs, scales, ref_frames), hop, width)
        mid = (ref_frames // 2) * hop
        t = torch.arange(T)
        rows = ref[mid + t % hop]                                       # interior: period hop
        rows[:EDGE] = ref[:EDGE]
        rows[T - EDGE:] = ref[ref_frames * hop - EDGE:]
    t = torch.arange(T)
    # the kernel's K window starts at window_start(t0) = floor8(t0 // hop - 2): TMA needs the innermost coordinate of a box
    # 16-byte aligned (8 bf16 frames) - an unaligned start makes the copy fault
    shift = (t // hop - 2) - window_start(t // TILE * TILE, hop)        # 0 .. 8
    assert int(shift.min()) >= 0 and int(shift.max()) + width <= KWIN
    out = torch.zeros(T, KWIN, dtype=torch.float64)
    out.scatter_(1, shift[:, None] + torch.arange(width)[None, :], rows)
    return out


# ----------------------------------------------------------------------------------------------------------------------
# Compact tables: what the kernel actually reads (a few MB, L2 resident, independent of batch size and utterance length)
# ----------------------------------------------------------------------------------------------------------------------
HALF = 128                     # rows one CTA of the pair loads per tile
END_ROWS = 3 * HALF            # per-utterance end table: the (up to) two half tiles touching the last EDGE rows + a zero block


def period(hop):
    """Rows after which the interior band table repeats: the tile-relative shift depends on t mod hop, t mod TILE and on
    (t // hop) mod 8 (the 8-frame alignment of the window start) -> lcm(8 * hop, TILE)."""
    import math
    return math.lcm(8 * hop, TILE)


def end_tile_start(length):
    """First row of the first half tile that touches the last EDGE rows of an utterance of `length` samples."""
    return (length - EDGE) // HALF * HALF


def _reference_rows(firs, scales, width=8, ref_frames=8):
    """Row windows of an 8-frame utterance: everything any longer utterance's table is assembled from."""
    hop = 1
    for s_ in scales:
        hop *= s_
    return _row_windows(upsample_operator(firs, scales, ref_frames), hop, width), hop, ref_frames


def _scatter_rows(rows, t, hop, width=8):
    """rows (n, width) of samples t (n,) -> (n, KWIN) placed relative to the K window of each sample's pair tile."""
    shift = (t // hop - 2) - window_start(t // TILE * TILE, hop)
    assert int(shift.min()) >= 0 and int(shift.max()) + width <= KWIN
    out = torch.zeros(t.shape[0], KWIN, dtype=torch.float64)
    out.scatter_(1, shift[:, None] + torch.arange(width)[None, :], rows)
    return out


def end_block(firs, scales, nf, ref=None):
    """The END_ROWS rows from end_tile_start(L) on of an nf-frame utterance (zero at and past L = nf * hop), built from the
    8-frame reference rows without materialising the whole per-length table (O(END_ROWS) per distinct length)."""
    ref, hop, ref_frames = ref if ref is not None else _reference_rows(firs, scales)
    blk = torch.zeros(END_ROWS, KWIN, dtype=torch.float64)
    if nf <= 0:
        return blk
    L = nf * hop
    m1 = end_tile_start(L)
    if nf <= ref_frames or L < 2 * EDGE + hop:
        full = tile_band_table(firs, scales, nf)
        n = min(END_ROWS, L - m1)
        blk[:n] = full[m1:m1 + n]
        return blk
    t = torch.arange(m1, L)
    mid = (ref_frames // 2) * hop
    rows = torch.where((t >= L - EDGE)[:, None], ref[(ref_frames * hop - (L - t)).clamp(0, ref.shape[0] - 1)], ref[mid + t % hop])
    blk[:L - m1] = _scatter_rows(rows, t, hop)
    return blk


def compact_band_tables(firs, scales, frames_list, base=None):
    """-> (table (rows, KWIN) float64, layout dict, base).  Rows [0, P): interior rows by t mod P (P = period(hop));
    [P, P + 128): the first half tile of any utterance; then END_ROWS rows per entry of `frames_list` (utterance i): the half
    tiles starting at end_tile_start(L_i), + HALF, + 2 HALF (rows at or past L_i are zero).  `source_row` below is the
    kernel's lookup.  `base` (returned, reusable): the length-independent part + the reference rows - constants of the model."""
    if base is None:
        refpack = _reference_rows(firs, scales)
        hop = refpack[1]
        P = period(hop)
        big = tile_band_table(firs, scales, 2 * (P // hop) + 8)          # long enough for one whole interior period
        assert big.shape[0] >= 2 * P + EDGE
        base = dict(head=torch.cat([big[P:2 * P], big[:HALF]]), ref=refpack, hop=hop, period=P, ends={})
    P = base["period"]
    parts = [base["head"]]
    for nf in frames_list:
        nf = int(nf)
        if nf not in base["ends"]:
            if len(base["ends"]) > 4096:
                base["ends"].clear()
            base["ends"][nf] = end_block(firs, scales, nf, base["ref"])
        parts.append(base["ends"][nf])
    return torch.cat(parts), dict(period=P, start_row=P, end_base=P + HALF, hop=base["hop"]), base


def source_row(m, length, b, layout):
    """Row of the compact table holding the band rows of the half tile [m, m + 128) of utterance b (length samples):
    mirrors the producer of pwg_layer_fc_kernel."""
    if m == 0:
        return layout["start_row"]
    if m + HALF > length - EDGE:
        return layout["end_base"] + END_ROWS * b + min(m - end_tile_start(length), 2 * HALF)
    return m % layout["period"]
