"""Parallel WaveGAN on the GPU where the model-level tests do not look.

Per layer: `pk_pwg_residual_layer_fc` (frame-rate conditioning, the default path) and `pk_pwg_residual_layer` (sample-rate
conditioning planes, the path of configs the band tables do not cover) are launched directly for ONE layer and compared with
`oracle.pwg.residual_block` in float64, run on each utterance alone.  The operands are built here: x as split planes, W1 / W2
packed by `PWGGenerator._pack`, P = W_aux conv_in(mel) and the upsampled conditioning in float64 on the host, the band table
from `compact_band_tables`, so neither `pk_pwg_upsample` nor the P GEMM is on the path under test, and the reference does not
use `_pwg_frame_cond` at all.

Generator: `PWGGenerator` against `oracle.pwg.generator_forward` at upsample configs the baker tests never run.
"""
import ctypes as C
import functools
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# max |kernel - fp64 reference| / max |reference| of one layer (y, skip written, skip accumulated), per utterance and over
# its first and last 256 rows.  Largest values over all cases on an H100 80GB HBM3 at a 400 W power limit (the per-case
# figures are recorded as test properties: pytest --junitxml=... -o junit_family=legacy):
#   pk_pwg_residual_layer_fc 9.0e-6, pk_pwg_residual_layer 9.0e-6; with saturated gates 2.4e-5 and 1.7e-5.
LAYER_TOL = 2e-5
SATURATED_TOL = 5e-5
# 9-layer generator against the float64 oracle, measured the same way: at most 2.6e-5 over the three configs below.  The
# frame-rate band tables at [2, 16, 8] (wrong within 136 samples of an end) gave 1.0e-3.
GEN_TOL = 1e-4
SCALES = {300: [4, 5, 3, 5], 256: [4, 4, 4, 4]}
SENTINEL = -3.25                    # y planes are filled with it before a launch: windows the kernel skips keep it
SATURATE = 8.0                      # W1 scale that drives the gate pre-activations to about +-50
BATCHES = {                         # frames per utterance; ragged batches pass lens, the others run without
    "one_frame": ((1,), False),     # T = hop: the last window holds fewer live rows than its first half tile
    "two_frames": ((2,), False),    # end_tile_start in the second half of a window
    "ragged": ((40, 0, 33, 1), True),        # an empty utterance; end tiles in the first and the second half of a window
    "idle_ctas": ((0, 0, 0, 40), True),      # every live tile lands on a subset of the CTAs: the others get none
    "many_tiles": ((40,) * 8, False),        # 8 x 40 frames: 640 (hop 256) / 752 (hop 300) half tiles on 132 SMs
}


@functools.lru_cache(maxsize=None)
def _layer_model(hop, saturate, device):
    """One-layer generator at the upsample config of `hop`: (packed layer, fp64 params, fp64 FIRs)."""
    from oracle import pwg as opwg
    from parakeet_b200.models import PWGGenerator
    cfg = dict(upsample_scales=SCALES[hop], layers=1, stacks=1)
    params = opwg.synth_params(7, cfg)
    if saturate:
        for k in ("conv_layers.0.conv.weight", "conv_layers.0.conv1x1_aux.weight"):
            params[k] = params[k] * SATURATE
    gen = PWGGenerator(**{**opwg.DEFAULT_GENERATOR_PARAMS, **cfg, "use_weight_norm": False}, device=device)
    gen.set_state_dict(params)
    p64 = {k: v.double() for k, v in params.items()}
    firs = [p64[f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"].reshape(-1) for i in range(len(SCALES[hop]))]
    return gen._pack()["layers"][0], p64, firs


@functools.lru_cache(maxsize=None)
def _band_base(hop, device):
    from parakeet_b200.models import _pwg_frame_cond as fc
    _, _, firs = _layer_model(hop, False, device)
    return fc.compact_band_tables(firs, SCALES[hop], [1])[2]     # the length-independent part, shared by every batch


@functools.lru_cache(maxsize=None)
def _inputs(hop, frames):
    """x (B, T, 64) fp32, zero past each utterance (as the model keeps it), and each utterance's mel (80, frames + 4) fp64."""
    g = torch.Generator().manual_seed(hop * 131 + sum(frames) * 7 + len(frames))
    T = max(frames) * hop
    x = torch.zeros(len(frames), T, 64)
    mels = []
    for b, nf in enumerate(frames):
        x[b, :nf * hop] = torch.randn(nf * hop, 64, generator=g)
        mels.append(torch.randn(80, nf + 4, generator=g, dtype=torch.float64))
    return x, mels


def _conv_in(p64, mel):
    return F.conv1d(mel[None], p64["upsample_net.conv_in.weight"])[0]                 # (80, frames)


def _operands(kind, hop, frames, x, mels, saturate, device):
    """Everything a launch reads, on the device: the x planes and the conditioning operands of `kind`."""
    from oracle import pwg as opwg
    from parakeet_b200.models import _pwg_frame_cond as fc
    from parakeet_b200.ops import Split
    _, p64, firs = _layer_model(hop, saturate, device)
    B, T = x.shape[:2]
    ops = dict(x=Split.from_f32(x.to(device)), B=B, T=T)
    if kind == "fc":
        w_aux = p64["conv_layers.0.conv1x1_aux.weight"][:, :, 0]                        # (128, 80)
        fp = max((max(frames) + 7) // 8 * 8, 64)
        P = torch.zeros(B, 128, fp, dtype=torch.float64)                               # frames past an utterance stay zero
        for b, nf in enumerate(frames):
            if nf:
                P[b, :, :nf] = w_aux @ _conv_in(p64, mels[b])
        tab, lay, _ = fc.compact_band_tables(firs, SCALES[hop], frames, _band_base(hop, device))
        wide = torch.zeros(tab.shape[0], 64)
        wide[:, :fc.KWIN] = tab.float()
        ops.update(P=Split.from_f32(P.float().to(device)), p_ld=fp, p_frames=max(frames),
                   U=Split.from_f32(wide.to(device)), lay=lay)
    else:
        c = torch.zeros(B, T, 80)
        for b, nf in enumerate(frames):
            if nf:
                c[b, :nf * hop] = opwg.upsample_net(p64, _conv_in(p64, mels[b])[None], SCALES[hop])[0].T.float()
        ops["c"] = Split.from_f32(c.to(device))
    return ops


def _launch(kind, hop, ops, lay, dil, lens, skip, skip_init):
    """One layer into fresh y planes filled with SENTINEL; `skip` is written (skip_init=1) or accumulated into."""
    from parakeet_b200 import _lib
    from parakeet_b200.ops import Split, _stream
    L = _lib.lib()
    B, T = ops["B"], ops["T"]
    y = Split.empty((B, T, 64), skip.device)
    y.hi.fill_(SENTINEL)
    y.lo.fill_(SENTINEL)
    a = _lib.PwgLayerFcArgs() if kind == "fc" else _lib.PwgLayerArgs()
    a.batch, a.t, a.dilation = B, T, dil
    a.lens = lens.data_ptr() if lens is not None else None
    a.x_hi, a.x_lo, a.y_hi, a.y_lo = ops["x"].hi.data_ptr(), ops["x"].lo.data_ptr(), y.hi.data_ptr(), y.lo.data_ptr()
    a.w1_hi, a.w1_lo = lay["w1"].hi.data_ptr(), lay["w1"].lo.data_ptr()
    a.w2_hi, a.w2_lo = lay["w2"].hi.data_ptr(), lay["w2"].lo.data_ptr()
    a.bias1, a.bias2 = lay["b1"].ctypes.data, lay["b2"].ctypes.data
    a.skip, a.skip_init = skip.data_ptr(), skip_init
    if kind == "fc":
        U, P, ul = ops["U"], ops["P"], ops["lay"]
        a.hop = hop
        a.u_hi, a.u_lo, a.u_rows = U.hi.data_ptr(), U.lo.data_ptr(), U.hi.shape[0]
        a.u_period, a.u_start_row, a.u_end_base = ul["period"], ul["start_row"], ul["end_base"]
        a.p_hi, a.p_lo, a.p_rows, a.p_ld, a.p_frames, a.p_row0 = P.hi.data_ptr(), P.lo.data_ptr(), 128, ops["p_ld"], ops["p_frames"], 0
        _lib.check(L.pk_pwg_residual_layer_fc(C.byref(a), _stream()), "pk_pwg_residual_layer_fc")
    else:
        a.aux_channels = 80
        a.c_hi, a.c_lo = ops["c"].hi.data_ptr(), ops["c"].lo.data_ptr()
        _lib.check(L.pk_pwg_residual_layer(C.byref(a), _stream()), "pk_pwg_residual_layer")
    torch.cuda.synchronize()
    return y


def _reference(hop, frames, saturate, dil, device):
    """Per utterance (None when empty): y (L, 64) and skip without its bias (the kernel leaves that to the tail), fp64,
    from x = hi + lo of the split planes the kernel reads, and the gate pre-activations' largest magnitude."""
    from oracle import pwg as opwg
    from parakeet_b200.ops import Split
    _, p64, _ = _layer_model(hop, saturate, device)
    x, mels = _inputs(hop, frames)
    xs = Split.from_f32(x.to(device)).float().double().cpu()
    pre = "conv_layers.0."
    out, hmax = [], 0.0
    for b, nf in enumerate(frames):
        if not nf:
            out.append(None)
            continue
        xb = xs[b, :nf * hop].T[None]
        c_up = opwg.upsample_net(p64, _conv_in(p64, mels[b])[None], SCALES[hop])
        y, s = opwg.residual_block(p64, pre, xb, c_up, dil)
        h = F.conv1d(xb, p64[pre + "conv.weight"], p64[pre + "conv.bias"], padding=dil, dilation=dil) \
            + F.conv1d(c_up, p64[pre + "conv1x1_aux.weight"])
        hmax = max(hmax, float(h.abs().max()))
        out.append((y[0].T, (s - p64[pre + "conv1x1_skip.bias"][None, :, None])[0].T))
    return out, hmax


def _edge_err(got, ref):
    """max |got - ref| / max |ref| over the utterance, over its first 256 rows and over its last 256 rows (an edge error
    cannot hide behind a larger interior maximum)."""
    got = got.double().cpu()
    return max(float((got[sl] - ref[sl]).abs().max() / ref[sl].abs().max().clamp_min(1e-30))
               for sl in (slice(None), slice(0, 256), slice(-256, None)))


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _check_layer(kind, hop, batch, dil, saturate, device, record_property):
    frames, ragged = BATCHES[batch]
    lay, _, _ = _layer_model(hop, saturate, device)
    x, mels = _inputs(hop, frames)
    ops = _operands(kind, hop, frames, x, mels, saturate, device)
    B, T = ops["B"], ops["T"]
    lens = torch.tensor([nf * hop for nf in frames], dtype=torch.int32, device=device) if ragged else None
    refs, hmax = _reference(hop, frames, saturate, dil, device)
    nan_skip = lambda: torch.full((B, T, 64), float("nan"), device=device)   # noqa: E731
    skip1 = nan_skip()
    y1 = _launch(kind, hop, ops, lay, dil, lens, skip1, 1)
    skip2 = nan_skip()
    y2 = _launch(kind, hop, ops, lay, dil, lens, skip2, 1)
    s0 = torch.randn(B, T, 64, generator=torch.Generator().manual_seed(dil)).to(device)
    skip3 = s0.clone()
    y3 = _launch(kind, hop, ops, lay, dil, lens, skip3, 0)

    # determinism: same launch twice, and y does not depend on skip_init
    for a, b in ((y1.hi, y2.hi), (y1.lo, y2.lo), (skip1, skip2), (y1.hi, y3.hi), (y1.lo, y3.lo)):
        assert torch.equal(_bits(a), _bits(b))
    errs = dict(y=0.0, skip=0.0, skip_acc=0.0)
    yf = y1.float()
    for b, nf in enumerate(frames):
        n = nf * hop
        if n:
            y_ref, s_ref = refs[b]
            errs["y"] = max(errs["y"], _edge_err(yf[b, :n], y_ref))
            errs["skip"] = max(errs["skip"], _edge_err(skip1[b, :n], s_ref))
            errs["skip_acc"] = max(errs["skip_acc"], _edge_err(skip3[b, :n].double() - s0[b, :n].double(), s_ref))
        # rows at or past the utterance's end: zero (live window) or untouched (window skipped), never anything else
        for plane in (y1.hi, y1.lo):
            dead = plane[b, n:]
            assert bool(((dead == 0) | (dead == SENTINEL)).all()), (b, nf)
    for k, v in errs.items():
        record_property(k, v)
    assert all(math.isfinite(v) for v in errs.values()), errs
    assert max(errs.values()) < (SATURATED_TOL if saturate else LAYER_TOL), errs

    # each utterance alone (B = 1, T = its own length, no lens): bit for bit the rows it has inside the batch
    if B > 1:
        for b, nf in enumerate(frames):
            if not nf:
                continue
            one = _operands(kind, hop, (nf,), x[b:b + 1, :nf * hop], mels[b:b + 1], saturate, device)
            s = torch.empty(1, nf * hop, 64, device=device)
            y = _launch(kind, hop, one, lay, dil, None, s, 1)
            assert torch.equal(_bits(y.hi[0]), _bits(y1.hi[b, :nf * hop])) and torch.equal(_bits(y.lo[0]), _bits(y1.lo[b, :nf * hop]))
            assert torch.equal(_bits(s[0]), _bits(skip1[b, :nf * hop])), (b, nf)
    return hmax


@pytest.mark.parametrize("batch", list(BATCHES))
@pytest.mark.parametrize("dil", [1, 2, 64, 256, 512])
@pytest.mark.parametrize("hop", [300, 256])
@pytest.mark.parametrize("kind", ["fc", "sr"])
def test_pwg_layer_vs_fp64(cuda, record_property, kind, hop, dil, batch):
    """One layer of either kernel: y and the skip sum (written over NaN, and accumulated onto random values) against the fp64
    block at every live row, zero or untouched rows past each length, two launches bit-identical, and each utterance of a
    batch bit-identical to running it alone."""
    _check_layer(kind, hop, batch, dil, False, cuda, record_property)


@pytest.mark.parametrize("hop", [300, 256])
@pytest.mark.parametrize("kind", ["fc", "sr"])
def test_pwg_layer_saturated_gates(cuda, record_property, kind, hop):
    """W1 scaled so that the gate pre-activations reach about +-50: the clamp of exp2's argument and the overflow of e2 to
    infinity are exercised; the output stays finite.  The bound is looser: a pre-activation's split-bf16 rounding grows
    with the magnitude of its terms, and near zero the gate passes it on undamped."""
    hmax = _check_layer(kind, hop, "ragged", 64, True, cuda, record_property)
    assert 40 < hmax < 100, hmax


# ----------------------------------------------------------------------------------------------------------------------
# Generator at upsample configs the baker tests do not run
# ----------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scales", [[4, 4, 4, 4], [2, 16, 8], [4, 4, 4]], ids=lambda s: "x".join(map(str, s)))
def test_pwg_generator_upsample_configs_vs_oracle(cuda, record_property, scales):
    """[4, 4, 4, 4] is the model's default and the reference's unit-test config (9 layers in 3 stacks, x [4, 1, 80 * 256],
    c [4, 80, 84]): it takes the frame-rate path.  [2, 16, 8] (the upsampler's padding reaches 136 samples into an
    utterance, past the band tables' 128 edge rows) and [4, 4, 4] (hop 64) take the sample-rate path.  Whole batch and a
    ragged batch with an empty utterance, against the oracle in float64, per utterance and over its first and last 256
    samples (the frame-rate tables' error at [2, 16, 8] sits next to the ends)."""
    from oracle import pwg as opwg
    from parakeet_b200.models import PWGGenerator
    cfg = {**opwg.DEFAULT_GENERATOR_PARAMS, "upsample_scales": scales, "layers": 9, "stacks": 3}
    hop = math.prod(scales)
    params = opwg.synth_params(3, cfg, weight_norm=True)
    folded = {k: v.double() for k, v in opwg.fold_weight_norm(params).items()}
    gen = PWGGenerator(**cfg, device=cuda)
    gen.set_state_dict(params)
    assert gen._uses_frame_cond() == (scales == [4, 4, 4, 4])

    def ref(x, c):
        with torch.no_grad():
            return opwg.generator_forward(folded, x.double(), c.double(), cfg)
    err = 0.0
    x, c = opwg.synth_inputs(3, batch=4, mel_frames=80, cfg=cfg)
    y, y_ref = gen(x.to(cuda), c.to(cuda)), ref(x, c)
    for i in range(4):
        err = max(err, _edge_err(y[i, 0], y_ref[i, 0]))
    frames = [80, 0, 37, 1]
    xs = torch.zeros(4, 1, 80 * hop)
    cs = torch.zeros(4, 80, 84)
    refs = {}
    for i, f in enumerate(frames):
        if f:
            xi, ci = opwg.synth_inputs(40 + i, batch=1, mel_frames=f, cfg=cfg)
            xs[i, :, :f * hop], cs[i, :, :f + 4] = xi[0], ci[0]
            refs[i] = ref(xi, ci)[0, 0]
    lens = torch.tensor([f * hop for f in frames], dtype=torch.int32, device=cuda)
    y = gen(xs.to(cuda), cs.to(cuda), lens=lens)
    for i, f in enumerate(frames):
        if f:
            err = max(err, _edge_err(y[i, 0, :f * hop], refs[i]))
        assert f == 80 or y[i, :, f * hop:].abs().max().item() == 0, (i, f)
    record_property("err", err)
    assert err < GEN_TOL, err


def test_pwg_generator_rejects_lens_off_the_frame_grid(cuda):
    """lens are samples of whole frames within T: anything else would give band tables whose end blocks do not match the
    rows the layer kernels treat as live, so it raises instead of returning wrong audio."""
    from parakeet_b200._lib import PkError
    from parakeet_b200.models import PWGGenerator
    gen = PWGGenerator(layers=3, stacks=1, upsample_scales=[4, 5, 3, 5], device=cuda)
    x = torch.zeros(2, 1, 10 * 300, device=cuda)
    c = torch.zeros(2, 80, 14, device=cuda)
    for bad in ([3000, 1501], [3300, 300], [-300, 300], [3000]):
        with pytest.raises(PkError, match="lens"):
            gen(x, c, lens=torch.tensor(bad, dtype=torch.int32, device=cuda))
    y = gen(x, c, lens=torch.tensor([3000, 0], dtype=torch.int32, device=cuda))
    assert y[1].abs().max().item() == 0
