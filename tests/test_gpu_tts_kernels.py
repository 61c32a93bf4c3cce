"""The TransformerTTS kernels (csrc/transformer_tts.cu) alone, each against a plain evaluation of the same operation: the persistent
decoder `pk_tts_decode` on synthetic encoder output (so no encoder or GEMM error enters its budget) at the head-width, row-block,
prenet, reduction-factor, depth, encoder-length, seed and stop-rule edges where its loops and indices branch; and the four glue
kernels of the teacher-forced forward, bit for bit against the oracle's host construction.

The decoder's reference is oracle.transformer_tts.decode, evaluated on the GPU in float64 with TF32 off (so the fp32 run of the
same restatement, the yardstick of fp32 drift, is true fp32).  Its source-attention K / V are computed from the same encoder
output in fp64; the kernel gets them rounded once to fp32, as it gets its weights.

Decoder bound.  Every decoder quantity is a chain of fp32 FFMA dot products (warp-strided, then a butterfly), LayerNorms and
softmaxes, fed back through the prenet from step to step.  As in tests/test_gpu_taco2_kernels.py, the kernel's error against fp64
is held to max(FLOOR, 10 x the error of the same computation in fp32 torch), both measured per row (every step; every attention
row) against fp64: the fp32 run shows how far plain fp32 drifts on this very input, and FLOOR = 2e-5 covers a case whose fp32 run
rounds more favourably than the kernel's summation order (one step's dot products of depth <= 300 at 2^-24 each, on terms whose
magnitudes add up to ~10x the result, stay below ~2e-5 of the row's scale).  A wrong row block, cache row, head offset or mask
moves a row by O(1)."""
import numpy as np
import pytest
import torch

import oracle.fastspeech2 as ofs
import oracle.transformer_tts as ot
from parakeet_b200 import ops
from parakeet_b200.models import TransformerTTS

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24
FLOOR = 2e-5
THREADS = 512            # csrc/pk_decode.cuh kThreads: 16 warps, so rows_phase hands out blocks of 16 rows
BIG_SEEDS = (2 ** 40 + 5, 2 ** 62 - 1)     # seed_hi != 0, as TransformerTTS._seed draws them


@pytest.fixture(autouse=True, scope="module")
def _no_tf32(cuda):
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def row_rel(a, b, floor=1e-3):
    """worst over rows (the last axis) of max |a - b| / max |b| in the row, the denominator at least floor x the tensor's max |b|
    (a row of near-zeros is held to the tensor's scale, not to its own)."""
    a, b = a.double().cpu(), b.double().cpu()
    den = b.abs().amax(-1).clamp_min(floor * b.abs().max().item() + 1e-30)
    return ((a - b).abs().amax(-1) / den).max().item()


def assert_drift(name, got, r64, r32):
    e_k, e_32 = row_rel(got, r64), row_rel(r32, r64)
    print(f"{name}: kernel vs fp64 {e_k:.2e}, fp32 oracle vs fp64 {e_32:.2e}, bound {max(FLOOR, 10 * e_32):.2e}")
    assert e_k <= max(FLOOR, 10 * e_32), (name, e_k, e_32)


# ---------------------------------------------------------------------------------------------------------------------------
# pk_tts_decode
# ---------------------------------------------------------------------------------------------------------------------------
def decode_case(seed, t_enc=37, minlen=0, maxlen=10, threshold=2.0, steps=None, dseed=BIG_SEEDS[0], **over):
    """-> ((outs, probs, att_ws, frames) of pk_tts_decode, the fp64 oracle's decode, its fp32 run, cfg) on a model of ot.SMALL
    with `over`, its weights packed by the model itself, and encoder output hs in (-1, 1)."""
    cfg = dict(ot.SMALL, **over)
    p = ot.synth_params(100 + seed, cfg)
    m = TransformerTTS(cfg["idim"], cfg["odim"], device=DEV, **{k: v for k, v in cfg.items() if k not in ("idim", "odim")})
    m.set_state_dict(p)
    A, L = cfg["adim"], cfg["dlayers"]
    steps = steps or max(minlen, maxlen, 1)
    g = torch.Generator().manual_seed(200 + seed)
    hs = (torch.rand(1, t_enc, A, generator=g) * 2 - 1).to(DEV)              # fp32 values: the same input in both precisions
    p64 = {k: v.to(DEV, torch.float64) for k, v in p.items()}
    src = [f"decoder.decoders.{l}.src_attn.linear_" for l in range(L)]
    mem_kv = torch.cat([hs[0].double() @ p64[s + kv + ".weight"] + p64[s + kv + ".bias"] for s in src for kv in "kv"], 1)
    pe = (p["decoder.embed.1.alpha"] * ofs.positional_encoding(steps, A)[0]).to(DEV)    # the oracle's own fp32 alpha pe rows
    got = ops.tts_decode(m._pack()["dec"], mem_kv.float().contiguous(), pe, heads=cfg["aheads"], steps=steps, minlen=minlen,
                         maxlen=maxlen, threshold=threshold, seed=dseed)
    with torch.no_grad():
        r64 = ot.decode(p, cfg, hs.double(), minlen, maxlen, threshold, dseed)
        r32 = ot.decode(p, cfg, hs, minlen, maxlen, threshold, dseed, dtype=torch.float32)
    return got, r64, r32, cfg


def check(got, r64, r32, cfg, tag):
    outs, probs, att, frames = got
    r, odim = cfg["reduction_factor"], cfg["odim"]
    n = r64[1].numel() // r
    assert int(frames.item()) == n, (tag, int(frames.item()), n)
    assert r32[1].numel() == n * r                # no case sits near a stop decision: both oracles exit at the same step
    assert_drift(f"{tag} outs", outs[:n], r64[0].reshape(n, r * odim), r32[0].reshape(n, r * odim))
    assert_drift(f"{tag} probs", probs[:n], r64[1].reshape(n, r), r32[1].reshape(n, r))
    assert_drift(f"{tag} att_ws", att[:, :, :n], r64[2], r32[2])
    # each softmax row: the sum of the exponentials has depth ceil(T / 512) + 5 + 16 (thread, warp butterfly, warps) and each weight
    # is one division by it, so the weights sum to 1 within (depth + 2) u, here doubled for the unknown order of the check's sum
    T = att.shape[-1]
    depth = -(-T // THREADS) + 5 + 16
    s = att[:, :, :n].double().sum(-1)
    assert (s - 1).abs().max().item() <= 2 * (depth + 2) * U, (tag, (s - 1).abs().max().item())
    # rows past the stop are never written: exactly zero
    assert not outs[n:].any() and not probs[n:].any() and not att[:, :, n:].any(), tag


@pytest.mark.parametrize("heads", [1, 2, 4, 8])
@pytest.mark.parametrize("dk", [64, 128, 192])
def test_decoder_head_widths(dk, heads):
    """attend's context splits the keys into 512 / d_k = 8, 4 or 2 chunks per column; one CTA per head, heads at h d_k."""
    check(*decode_case(dk + heads, adim=dk * heads, aheads=heads), tag=f"dk={dk} H={heads}")


def test_decoder_rows_wrap_around_the_grid():
    """dunits = 64 x SMs + 20: ceil(dunits / 16) = 4 x SMs + 2 row blocks of w_1, more than any co-resident grid of 512-thread CTAs
    (at most 4 per SM) has CTAs, so CTA 0 owns two or more blocks; dunits % 16 = 4 leaves a partial last block."""
    sms = torch.cuda.get_device_properties(DEV).multi_processor_count
    dunits = 64 * sms + 20
    assert -(-dunits // 16) > 4 * sms and dunits % 16 and dunits % 4 == 0
    check(*decode_case(1, adim=64, aheads=1, dunits=dunits, dlayers=1, maxlen=6), tag=f"dunits={dunits}")


@pytest.mark.parametrize("n_pre", [1, 3])
def test_decoder_prenet_depth(n_pre):
    """the prenet layers ping-pong between two buffers by (i & 1); the input Linear reads the last layer's."""
    check(*decode_case(2 + n_pre, dprenet_layers=n_pre), tag=f"prenet layers={n_pre}")


def test_decoder_small_k():
    """odim 4 and 4 prenet units: the prenet and the input Linear have K / 4 = 1 float4 per row, fewer than the 32 lanes."""
    check(*decode_case(6, odim=4, dprenet_units=4), tag="odim=4 prenet=4")


def test_decoder_reduction_factor_16():
    """r = 16: the 16 stop rows and the first frame rows share CTA 0's first row block; the stop rule reads all 16."""
    check(*decode_case(7, reduction_factor=16, maxlen=5), tag="r=16")


@pytest.mark.parametrize("dlayers", [1, 6])
def test_decoder_depth(dlayers):
    """per-layer weight offsets and K / V cache offsets kc / vc = l x steps x adim."""
    check(*decode_case(8 + dlayers, dlayers=dlayers), tag=f"dlayers={dlayers}")


@pytest.mark.parametrize("t_enc,steps", [(1, 12), (511, 12), (512, 12), (513, 12), (4000, 6), (5, 600)])
def test_decoder_lengths(t_enc, steps):
    """attend's score and softmax loops stride by 16 warps and 512 threads over t_enc keys (source attention) and t + 1 keys
    (self-attention); the score buffer holds max(steps, t_enc).  600 steps over 5 encoder rows: the self-attention passes 512."""
    check(*decode_case(20 + t_enc, t_enc=t_enc, maxlen=steps, dlayers=1 if steps > 100 else 2), tag=f"t_enc={t_enc} steps={steps}")


@pytest.mark.parametrize("dseed", (0,) + BIG_SEEDS)
def test_decoder_prenet_dropout_seed(dseed):
    """the seed's high 32 bits key the Philox masks as much as the low ones."""
    check(*decode_case(30, dseed=dseed), tag=f"seed={dseed}")


N_STOP = 9


@pytest.mark.parametrize("minlen,maxlen", [(0, 0), (0, N_STOP), (5, 3), (N_STOP, N_STOP)])
@pytest.mark.parametrize("threshold", [-1.0, 2.0])
def test_decoder_stop_rule(threshold, minlen, maxlen):
    """threshold -1: every step's probabilities reach it; 2: none does.  So the exit is max(minlen, 1), or max(minlen, maxlen, 1),
    with no probability near the threshold.  The kernel gets 3 steps more than the exit needs, so a late stop shows."""
    want = max(minlen, 1) if threshold < 0 else max(minlen, maxlen, 1)
    got, r64, r32, cfg = decode_case(40, minlen=minlen, maxlen=maxlen, threshold=threshold, steps=max(minlen, maxlen, 1) + 3,
                                     dseed=BIG_SEEDS[1])
    assert r64[1].numel() == want * cfg["reduction_factor"]
    check(got, r64, r32, cfg, tag=f"threshold={threshold} minlen={minlen} maxlen={maxlen}")


# ---------------------------------------------------------------------------------------------------------------------------
# glue of the teacher-forced forward, bit for bit
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T", [0, 1, 13])
def test_text_eos(T):
    """lens 0, 1 and T (where T allows): eos at column lens[b], zeros after, ilens = lens + 1."""
    g = torch.Generator().manual_seed(T)
    lens = torch.tensor([0, min(1, T), T, T // 2], dtype=torch.int32)
    text = torch.randint(1, 50, (4, T), generator=g)                      # live ids also past lens: they must not appear
    xs, ilens = ops.tts_text_eos(text.to(DEV), lens.to(DEV), 77)
    want_xs, want_ilens, _, _ = ot.eos_and_labels(text, lens, torch.ones(4, dtype=torch.int64), 77, 1)
    for b, n in enumerate(lens.tolist()):
        want_xs[b, n + 1:] = 0
    assert torch.equal(xs.cpu(), want_xs) and torch.equal(ilens.cpu().long(), want_ilens)


@pytest.mark.parametrize("r,olens", [(1, [1, 7, 12]), (2, [2, 7, 12, 9]), (3, [3, 7, 12, 11, 5])])
def test_stop_labels(r, olens):
    """olens % r != 0, olens == r and olens == the width; the width is max(olens - olens % r) as the model cuts it."""
    sl = torch.tensor(olens)
    width = int((sl - sl % r).max())
    _, _, want, cut = ot.eos_and_labels(torch.zeros(len(olens), 1, dtype=torch.int64), torch.zeros(len(olens), dtype=torch.int64), sl, 1, r)
    assert int(cut.max()) == width
    got = ops.tts_stop_labels(sl.to(DEV, torch.int32), width)
    assert torch.equal(got.cpu(), want)


@pytest.mark.parametrize("L,r", [(1, 1), (12, 1), (3, 3), (12, 3), (13, 3), (14, 4), (17, 16)])
def test_shift_frames(L, r):
    """ys[:, r-1::r] with a zero first frame and its last frame dropped; L a multiple of r or not, and L = r."""
    g = torch.Generator().manual_seed(10 * L + r)
    ys = torch.randn(3, L, 20, generator=g)
    thin = ys[:, r - 1::r]
    want = torch.cat([torch.zeros_like(thin[:, :1]), thin[:, :-1]], 1)
    got = ops.tts_shift_frames(ys.to(DEV), r)
    assert got.shape == want.shape and torch.equal(got.cpu(), want)


@pytest.mark.parametrize("p", [0.5, 0.1])
@pytest.mark.parametrize("units", [256, 30])
@pytest.mark.parametrize("seed", BIG_SEEDS)
def test_prenet_dropout(seed, units, p):
    """B = 3, 1000 frame positions, sites 0-2 against ot.prenet_masks(batch=3): element b units + j, so with 30 units a Philox
    block of 4 elements straddles two items.  The kept share is 1 - p within 5 binomial standard deviations."""
    B, L, sites = 3, 1000, 3
    keep = ot.prenet_masks(seed, L, units, sites, batch=B, p=p)
    scale = np.float32(1.0) / (np.float32(1.0) - np.float32(p))         # the kernel's fp32 1 / (1 - p)
    g = torch.Generator().manual_seed(units)
    for site in range(sites):
        x = torch.randn(B, L, units, generator=g) + 3.0                    # no zeros: a dropped element is exactly 0
        got = ops.tts_prenet_dropout_(x.to(DEV), p, seed, site).cpu()
        assert torch.equal(got, x * keep[site] * torch.tensor(scale)), site
    n = keep.numel()
    assert abs(keep.mean().item() - (1 - p)) <= 5 * (p * (1 - p) / n) ** 0.5
