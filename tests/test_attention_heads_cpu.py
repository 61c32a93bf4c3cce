"""Attention head widths the GEMM cannot slice are refused on the host, before any CUDA work (no GPU needed)."""
import pytest
import torch

from parakeet_b200 import _lib, ops


@pytest.mark.parametrize("adim,aheads", [(384, 4), (384, 8), (256, 8), (128, 4)])
def test_fastspeech2_refuses_head_width_not_multiple_of_64(adim, aheads):
    from parakeet_b200.models import FastSpeech2
    with pytest.raises(NotImplementedError, match="head width"):
        FastSpeech2(20, 80, adim=adim, aheads=aheads, elayers=1, dlayers=1, eunits=64, dunits=64, postnet_chans=64, device="cpu")


@pytest.mark.parametrize("adim,aheads", [(384, 2), (256, 2), (128, 1)])
def test_fastspeech2_accepts_head_widths_of_64_multiples(adim, aheads):
    from parakeet_b200.models import FastSpeech2
    m = FastSpeech2(20, 80, adim=adim, aheads=aheads, elayers=1, dlayers=1, eunits=64, dunits=64, postnet_chans=64, device="cpu")
    assert m.adim // m.aheads % 64 == 0


def _spec(cols, col0=0, colh=0):
    return dict(rows=8, cols=cols, ld=cols, batch_stride=8 * cols, batches=1, bmul=1, hmul=0, col0=col0, colh=colh)


def test_k_tail_overlap_rule():
    A, dk, H = 384, 96, 4
    qkv = 3 * A
    assert ops.k_tail_overlap(_spec(qkv, 0, dk), H, dk) == 0               # Q slice of head 0 runs into head 1
    assert ops.k_tail_overlap(_spec(qkv, 2 * A, dk), H, dk) == 0           # V slices: all but the last are followed by live columns
    assert ops.k_tail_overlap(_spec(A, 0, dk), H, dk) == 0                 # dO (B, T, A): head 0 still overlaps head 1
    assert ops.k_tail_overlap(_spec(A, 3 * dk, 0), 1, dk) is None          # the last head alone ends exactly at cols
    assert ops.k_tail_overlap(_spec(dk), H, dk) is None                    # head-batched planes (colh = 0) of width k
    assert ops.k_tail_overlap(_spec(qkv, 0, 192), 2, 192) is None          # k % 64 == 0: the chunks end where the slice ends
    assert ops.k_tail_overlap(_spec(80), 1, 80) is None                    # the PWG aux GEMM: cols == k
    assert ops.k_tail_overlap(_spec(128, 0, 0), 1, 80) == 0                # k = 80 in a 128-wide operand reads 48 live columns


def test_batched_matmul_nt_refuses_before_any_launch():
    """The refusal is host arithmetic on the specs: it raises for CPU tensors too, before the library is asked to launch."""
    A, dk, H, B, T = 384, 96, 4, 1, 8
    qkv = ops.Split(torch.zeros(B, T, 3 * A, dtype=torch.bfloat16), torch.zeros(B, T, 3 * A, dtype=torch.bfloat16))
    q = dict(rows=T, cols=3 * A, ld=3 * A, batch_stride=T * 3 * A, batches=B, bmul=1, hmul=0, col0=0, colh=dk)
    k = dict(q, col0=A)
    for simt in (False, True):
        with pytest.raises(_lib.PkError, match="operand A's K slice of head 0"):
            ops.batched_matmul_nt(qkv, qkv, batch=B, heads=H, m=T, n=T, k=dk, a_spec=q, b_spec=k, y_f32=torch.zeros(1), y_batch_stride=0,
                                  y_head_stride=0, y_ld=T, simt=simt)
