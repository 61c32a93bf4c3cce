"""The Tacotron2 kernels (csrc/tacotron2.cu) alone, each against a plain fp64 evaluation of the same operation on the same fp32
inputs: the persistent decoder `pk_taco2_decode` on synthetic encoder outputs (so no encoder or GEMM error enters its budget), in
both modes and at the batch, length, reduction-factor and location-kernel edges where its loops branch; the encoder glue and the
loss kernel.

The fp64 references are oracle/tacotron2.py, evaluated on the GPU in float64 (cuBLAS / cuDNN double, the oracle's own
arithmetic) so the long cases stay quick.  TF32 is switched off for this module, so the fp32 oracle runs used as the yardstick
of fp32 drift are true fp32.

Decoder bounds.  Every decoder quantity is a recurrence in fp32 FFMA.  One step's dot products are warp-strided sums of depth
K / 128 + 5 <= 27 (K <= 2816), each within 27 u of the sum of its terms' magnitudes (u = 2^-24, 27 u = 1.6e-6); for these
weights and inputs the terms' magnitudes add up to at most ~10x the result, so one step is within ~1.6e-5 of its row's scale,
and the recurrence carries and can grow that over the steps.  So, as in tests/test_gpu_tacotron2.py, the kernel's error against
fp64 is held to max(FLOOR, 10 x the error of the same computation in fp32 torch), both measured per row (every step of every
item) against fp64: the fp32 oracle shows how far plain fp32 drifts on this very input, and FLOOR = 2e-5, one step's worth,
covers a case whose fp32 oracle happens to round more favourably than the kernel's summation order."""
import pytest
import torch

import oracle.tacotron2 as ot
from parakeet_b200 import ops
from parakeet_b200.models import Tacotron2

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
U = 2.0 ** -24
FLOOR = 2e-5
THREADS = 512            # csrc/tacotron2.cu kThreads


@pytest.fixture(autouse=True, scope="module")
def _no_tf32(cuda):
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def row_rel(a, b, floor=1e-3):
    """worst over rows (the last axis; each element of a 2-D tensor) of max |a - b| / max |b| in the row, the denominator at least
    floor x the tensor's max |b| (a row of near-zeros is held to the tensor's scale, not to its own)."""
    a, b = a.double().cpu(), b.double().cpu()
    if b.dim() == 2:
        a, b = a.unsqueeze(-1), b.unsqueeze(-1)
    den = b.abs().amax(-1).clamp_min(floor * b.abs().max().item() + 1e-30)
    return ((a - b).abs().amax(-1) / den).max().item()


def assert_drift(name, got, r64, r32):
    e_k, e_32 = row_rel(got, r64), row_rel(r32, r64)
    print(f"{name}: kernel vs fp64 {e_k:.2e}, fp32 oracle vs fp64 {e_32:.2e}, bound {max(FLOOR, 10 * e_32):.2e}")
    assert e_k <= max(FLOOR, 10 * e_32), (name, e_k, e_32)


def make(cfg, seed, stop_bias=None):
    """-> (model, fp32 parameters on the device)."""
    p = ot.synth_params(seed, cfg, stop_bias=stop_bias)
    m = Tacotron2(device=DEV, **cfg)
    m.set_state_dict(p)
    return m, {k: v.to(DEV) for k, v in p.items()}


def synth_keys(seed, B, T, p):
    """Encoder-like keys in (-1, 1), non-zero also past text_lens (the mask alone must keep them out), and key_layer(keys)
    evaluated in fp64 and rounded once to fp32."""
    g = torch.Generator().manual_seed(seed)
    dk = p["decoder.attention_layer.key_layer.weight"].shape[0]
    keys = torch.tanh(torch.randn(B, T, dk, generator=g)).to(DEV)
    return keys, pkeys_of(keys, p)


def pkeys_of(keys, p):
    return (keys.double() @ p["decoder.attention_layer.key_layer.weight"].double()).float().contiguous()


def ragged(B, T, seed):
    g = torch.Generator().manual_seed(seed)
    lens = [T, 1] + [int(x) for x in torch.randint(1, T + 1, (max(B - 2, 0),), generator=g)]
    return torch.tensor(lens[:B], dtype=torch.int32)


def teacher_case(B, T, r=1, d_mels=80, loc_k=31, gc=False, stop=True, pdrop=0.0, steps=10, seed=0):
    cfg = ot.cfg_of(vocab_size=20, d_mels=d_mels, reduction_factor=r, attention_kernel_size=loc_k, use_stop_token=stop,
                    p_prenet_dropout=pdrop, d_global_condition=256 if gc else None)
    m, p = make(cfg, 40 + seed)
    keys, pkeys = synth_keys(50 + seed, B, T, p)
    lens = ragged(B, T, 60 + seed).to(DEV)
    g = torch.Generator().manual_seed(70 + seed)
    mels = (torch.randn(B, steps * r, d_mels, generator=g) * 0.5 - 1.0).to(DEV)
    got = ops.taco2_decode(m._packs()["dec"], keys, pkeys, steps, teacher=True, mels=mels, text_lens=lens, p_prenet=pdrop, seed=seed)
    with torch.no_grad():
        r64 = ot.decode(p, cfg, keys.double(), mels=mels, text_lens=lens, seed=seed)
        r32 = ot.decode(p, cfg, keys, mels=mels, text_lens=lens, seed=seed, dtype=torch.float32)
    return got, r64, r32, lens, steps


def check_teacher(got, r64, r32, lens, steps, tag):
    mel, align, stop, frames = got
    B, _, T = align.shape
    assert torch.all(frames == steps)
    assert_drift(f"{tag} mel", mel, r64[0], r32[0])
    assert_drift(f"{tag} alignment", align, r64[1], r32[1])
    assert (stop is None) == (r64[2] is None)
    if stop is not None:
        assert_drift(f"{tag} stop", stop, r64[2], r32[2])
    # each softmax row: the sum of the exponentials has depth ceil(T / 512) + 5 + 16 (thread, warp butterfly, warps) and each weight
    # is one division by it, so the weights sum to 1 within (depth + 2) u, here doubled for the unknown order of the check's sum
    depth = -(-T // THREADS) + 5 + 16
    s = align.double().sum(-1)
    assert (s - 1).abs().max().item() <= 2 * (depth + 2) * U, (tag, (s - 1).abs().max().item())
    # positions past text_lens get exactly zero weight (energy - 1e9 underflows exp)
    for b in range(B):
        assert torch.all(align[b, :, int(lens[b]):] == 0), (tag, b)


@pytest.mark.parametrize("B", [1, 2, 7, 8, 9, 31, 32])
def test_decoder_batch_chunks(B):
    """B = 1 runs the BC = 1 kernel; 2..7, 9 and 31 leave a partial last chunk of 8 in the matvec staging and the gate staging."""
    check_teacher(*teacher_case(B, 32, seed=B), tag=f"B={B}")


@pytest.mark.parametrize("T", [1, 15, 31, 32, 200, 513, 700])
def test_decoder_encoder_lengths(T):
    """T = 1, 15: every 31-tap location window padded on both sides; 31, 32: windows touching both ends; 200 and up: interior
    windows, more positions than the 16 warps (energy loop) and, from 513, than the 512 threads (softmax / argmax loops)."""
    check_teacher(*teacher_case(3, T, stop=False, steps=8, seed=T), tag=f"T={T}")


@pytest.mark.parametrize("r,d_mels", [(2, 80), (3, 80), (1, 8), (3, 8)])
def test_decoder_reduction_factor_and_mel_width(r, d_mels):
    """d_mels * r + stop crosses the 16-row projection blocks differently: 161, 241, 9, 25 rows."""
    check_teacher(*teacher_case(5, 40, r=r, d_mels=d_mels, seed=100 + 10 * r + d_mels), tag=f"r={r} d_mels={d_mels}")


@pytest.mark.parametrize("loc_k", [1, 3, 63])
def test_decoder_location_kernel(loc_k):
    check_teacher(*teacher_case(4, 70, loc_k=loc_k, seed=200 + loc_k), tag=f"loc_k={loc_k}")


def test_decoder_global_condition_d_enc_768():
    check_teacher(*teacher_case(6, 48, gc=True, steps=12, seed=300), tag="d_enc=768")


@pytest.mark.parametrize("B", [1, 9])
def test_decoder_prenet_dropout(B):
    """p = 0.5 with a fixed seed: the oracle restates the Philox mask of both prenet layers per step."""
    check_teacher(*teacher_case(B, 40, stop=B == 1, pdrop=0.5, steps=12, seed=400 + B), tag=f"dropout B={B}")


def test_decoder_long_teacher_forced_run():
    """Recipe-like lengths: T_enc = 180, 400 decoder steps, B = 9.  The cell states and the cumulative attention carry fp32
    rounding over all 400 steps; the drift bound measures how much plain fp32 accumulates on the same input."""
    check_teacher(*teacher_case(9, 180, pdrop=0.5, steps=400, seed=500), tag="long")


# ---------------------------------------------------------------------------------------------------------------------------
# infer mode: frames fed back, stop rules on the device
# ---------------------------------------------------------------------------------------------------------------------------
def infer_refs(p, cfg, keys, steps, seed):
    with torch.no_grad():
        return (ot.decode(p, cfg, keys.double(), max_decoder_steps=steps, seed=seed),
                ot.decode(p, cfg, keys, max_decoder_steps=steps, seed=seed, dtype=torch.float32))


def compare_prefix(got, r64, r32, n, tag):
    """kernel frames [:n] against fp64, with fp32 drift over the prefix both oracles share."""
    n32 = min(n, r32[0].shape[1])
    for i, name in enumerate(("mel", "alignment", "stop")):
        if r64[i] is None:
            continue
        e_k, e_32 = row_rel(got[i][:, :n], r64[i][:, :n]), row_rel(r32[i][:, :n32], r64[i][:, :n32])
        print(f"{tag} {name}: kernel vs fp64 {e_k:.2e}, fp32 oracle vs fp64 {e_32:.2e}")
        assert e_k <= max(FLOOR, 10 * e_32), (tag, name, e_k, e_32)


def test_infer_stop_token_frame_count():
    """B = 1, T_enc = 150: the stop bias is placed, from the fp64 trajectory, halfway between the largest stop logit before a
    chosen step and the logit at that step, so the reference stops there with a known margin."""
    cfg = dict(ot.LJSPEECH, use_stop_token=True)
    steps, seed = 200, 3
    _, p_free = make(cfg, 7, stop_bias=0.0)
    keys, pkeys = synth_keys(8, 1, 150, p_free)
    with torch.no_grad():
        free = ot.decode({**p_free, "decoder.stop_layer.bias": torch.full((1,), -1e4, dtype=torch.float64, device=DEV)}, cfg,
                         keys.double(), max_decoder_steps=steps, seed=seed)
    s = (free[2][0] + 1e4).cpu()                          # the logits without bias, for every step
    assert free[0].shape[1] == steps
    run = torch.cummax(s, 0).values
    gaps = [(float(s[t] - run[t - 1]), t) for t in range(30, steps) if s[t] > run[t - 1]]
    t_stop = max(gaps)[1] if gaps else int(torch.argmax(s[1:])) + 1     # the widest margin past step 30
    lo, hi = float(run[t_stop - 1]), float(s[t_stop])
    bias = -(lo + hi) / 2
    m, p = make(cfg, 7, stop_bias=bias)
    got = ops.taco2_decode(m._packs()["dec"], keys, pkeys, steps, teacher=False, p_prenet=0.5, seed=seed)
    r64, r32 = infer_refs(p, cfg, keys, steps, seed)
    assert r64[0].shape[1] == t_stop + 1
    # the stop decision is sigmoid(logit) > 0.5; the logits' error bound is the drift bound on the stop row
    n32 = min(t_stop + 1, r32[2].shape[1])
    bound = max(FLOOR, 10 * row_rel(r32[2][:, :n32], r64[2][:, :n32])) * float(r64[2].abs().max())
    if (hi - lo) / 2 <= bound:
        pytest.skip(f"the reference's stop decision is within the error bound of its threshold ({(hi - lo) / 2:.2e} <= {bound:.2e})")
    assert int(got[3][0]) == t_stop + 1
    compare_prefix(got, r64, r32, t_stop + 1, "infer stop token")


def argmax_ambiguous(align, n, bound):
    """Whether the end-of-text rule's decision (argmax of item 0's weights == T_enc - 1) at any step up to its first hit is within
    `bound` of flipping."""
    w = align[0, :n].double().cpu()
    last, others = w[:, -1], w[:, :-1].max(1).values if w.shape[1] > 1 else torch.full((n,), -1.0, dtype=torch.float64)
    hit = (last >= others).nonzero()
    upto = int(hit[0]) + 1 if len(hit) else n
    return bool(((last[:upto] - others[:upto]).abs() <= bound).any())


@pytest.mark.parametrize("B,T,steps", [(1, 150, 200), (4, 60, 50)])
def test_infer_end_of_text_rule(B, T, steps):
    """No stop token: the reference stops 21 steps after item 0's attention first peaks on the last position.  The last key is
    steered towards the attention vector so that the rule can fire; the frame count must equal the reference's."""
    cfg = dict(ot.LJSPEECH)
    m, p = make(cfg, 9)
    keys, _ = synth_keys(10, B, T, p)
    wk = p["decoder.attention_layer.key_layer.weight"].double()
    target = 0.8 * torch.sign(p["decoder.attention_layer.value.weight"][:, 0].double())
    keys[:, -1] = (wk @ torch.linalg.solve(wk.t() @ wk, target)).float().clamp(-3, 3)
    pkeys = pkeys_of(keys, p)
    got = ops.taco2_decode(m._packs()["dec"], keys, pkeys, steps, teacher=False, p_prenet=0.5, seed=4)
    r64, r32 = infer_refs(p, cfg, keys, steps, 4)
    n = r64[0].shape[1]
    n32 = min(n, r32[1].shape[1])
    bound = max(FLOOR, 10 * row_rel(r32[1][:, :n32], r64[1][:, :n32])) * float(r64[1].abs().max())
    if argmax_ambiguous(r64[1], n, bound):
        pytest.skip("the reference's end-of-text decision is within the error bound of an argmax tie")
    print(f"B={B} T={T}: reference stops after {n} of {steps} frames")
    assert torch.all(got[3] == n), (got[3].tolist(), n)
    compare_prefix(got, r64, r32, n, f"infer B={B}")


# ---------------------------------------------------------------------------------------------------------------------------
# encoder: the model's bidirectional LSTM and the glue kernels
# ---------------------------------------------------------------------------------------------------------------------------
def test_encoder_bilstm_ragged_against_fp64():
    """taco2_embed -> 3 x conv_gemm -> taco2_time_major (both directions) -> pk_lstm_fwd -> taco2_bilstm_merge -> key GEMM, at B = 9,
    T = 200, lengths ragged and including 1, against oracle.tacotron2.encoder in fp64 (CPU).  The GEMMs and the recurrence are
    split-bf16 wgmma: each product holds 2^-15 of |w x|, ~2^-15 sqrt(K) of a random-sign dot product at worst (1.5e-3 at the
    convs' K = 2560, 5e-4 in the recurrence), while independent roundings leave ~2^-15 of the output per GEMM.  The bound is 1e-3
    of each row's scale, the model tests' tolerance; rows past a length must be exactly zero."""
    cfg = dict(ot.LJSPEECH)
    m, p = make(cfg, 11)
    B, T = 9, 200
    text, _ = ot.synth_text(12, B, T, cfg["vocab_size"])
    lens = ragged(B, T, 13)
    keys, pkeys = m._encode(text.to(DEV), None, lens.to(DEV), None)
    p_cpu = {k: v.cpu() for k, v in p.items()}
    with torch.no_grad():
        ref = ot.encoder(p_cpu, cfg, text, None, lens, None)
    err = row_rel(keys, ref)
    print(f"encoder keys: row-relative error {err:.2e}")
    assert err < 1e-3
    for b in range(B):
        assert torch.all(keys[b, int(lens[b]):] == 0)


def test_taco2_embed_bit_exact():
    g = torch.Generator().manual_seed(1)
    vocab, n_tones, C = 37, 10, 512
    table, tone_table = torch.randn(vocab, C, generator=g), torch.randn(n_tones, C, generator=g)   # row 0 non-zero on purpose
    ids = torch.randint(0, vocab, (5, 23), generator=g)
    tones = torch.randint(0, n_tones, (5, 23), generator=g)
    ids[0, 0], ids[1, 3], tones[0, 0], tones[2, :] = vocab - 1, 0, 0, 0
    ref = table[ids] + torch.cat([torch.zeros(1, C), tone_table[1:]])[tones]       # tone 0 is padding: adds exactly zero
    got = ops.taco2_embed(ids.to(DEV), table.to(DEV), tones.to(DEV), tone_table.to(DEV))
    assert torch.equal(got.cpu(), ref)
    assert torch.equal(ops.taco2_embed(ids.to(DEV), table.to(DEV)).cpu(), table[ids])


@pytest.mark.parametrize("reverse", [False, True])
def test_taco2_time_major_bit_exact(reverse):
    g = torch.Generator().manual_seed(2)
    B, T, C = 5, 37, 1024
    x = torch.randn(B, T, C, generator=g)
    lens = torch.tensor([1, T, 17, 1, 36], dtype=torch.int32)
    ref = x.transpose(0, 1).clone()
    if reverse:
        for b in range(B):
            n = int(lens[b])
            ref[:n, b] = x[b, :n].flip(0)                  # rows past the length keep their place
    got = ops.taco2_time_major(x.to(DEV), lens.to(DEV), reverse=reverse)
    assert torch.equal(got.cpu(), ref)
    full = x.transpose(0, 1).flip(0) if reverse else x.transpose(0, 1)
    assert torch.equal(ops.taco2_time_major(x.to(DEV), None, reverse=reverse).cpu(), full)


@pytest.mark.parametrize("gc_dim", [0, 256])
def test_taco2_bilstm_merge_bit_exact(gc_dim):
    g = torch.Generator().manual_seed(3)
    T, B, H = 41, 6, 256
    hf, hb = torch.randn(T, B, H, generator=g), torch.randn(T, B, H, generator=g)
    gc = torch.randn(B, gc_dim, generator=g) if gc_dim else None
    lens = torch.tensor([T, 1, 20, 40, 1, 33], dtype=torch.int32)
    ref = torch.zeros(B, T, 2 * H + gc_dim)
    for b in range(B):
        n = int(lens[b])
        for t in range(n):
            ref[b, t, :H] = hf[t, b]
            ref[b, t, H:2 * H] = hb[n - 1 - t, b]          # the backward direction ran on the sequence reversed within n
            if gc_dim:
                ref[b, t, 2 * H:] = gc[b]
    got = ops.taco2_bilstm_merge(hf.to(DEV), hb.to(DEV), lens.to(DEV), gc.to(DEV) if gc_dim else None)
    assert torch.equal(got.cpu(), ref)


def test_taco2_loss_recipe_shape_against_fp64():
    """B = 32, T_mel = 800, t_enc = 200 (the guided-attention sum has 160 000 terms per item, 156 per thread of the block), ragged
    lengths including 1, stop logits of +-90.  The kernel sums in double (relative error < 2^-53 x 1e6 terms = 1e-10), then rounds
    each output once to fp32: within 2 u of each loss."""
    g = torch.Generator().manual_seed(4)
    B, T, C, Te = 32, 800, 80, 200
    mel, post, tgt = (torch.randn(B, T, C, generator=g) for _ in range(3))
    align = torch.softmax(torch.randn(B, T, Te, generator=g) * 3, -1)
    stop = torch.randn(B, T, generator=g) * 5
    slens = torch.randint(1, T + 1, (B,), generator=g)
    plens = torch.randint(1, Te + 1, (B,), generator=g)
    slens[0], slens[1], slens[2], plens[0], plens[3], plens[4] = 1, T, 2, Te, 1, 2
    stop[0, 0] = -90.0                                     # the positive label at a logit of -90
    stop[1, 5], stop[5, 10], stop[6, 3] = 95.0, -120.0, 90.0
    stop[7, int(slens[7]) - 1] = 100.0
    got = ops.taco2_loss(mel.to(DEV), post.to(DEV), tgt.to(DEV), align.to(DEV), slens.to(DEV), plens.to(DEV), 0.2, stop.to(DEV))
    ref = ot.loss(*(x.double() for x in (mel, post, tgt, align)), slens, plens, stop.double(), use_guided_attention_loss=True)
    for i, k in enumerate(("loss", "mel_loss", "post_mel_loss", "guided_attn_loss", "stop_loss")):
        r = float(ref[k])
        print(f"{k}: {float(got[i]):.9g} vs {r:.9g}, rel {abs(float(got[i]) - r) / abs(r):.2e}")
        assert abs(float(got[i]) - r) <= 2 * U * abs(r), k
