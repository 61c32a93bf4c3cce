"""The two ends of the frame-rate Parallel WaveGAN residual stack, launched directly for one layer (`pk_pwg_residual_layer_fc`
with `noise` or `out` set) and compared with the float64 reference, run on each utterance alone.

  * first layer: first_conv(noise) is computed inside the layer kernel; against float64 first_conv + ResidualBlock 0;
  * last layer: the tail (last_conv_layers on the scaled skip sum) runs in the layer's epilogue; against float64
    tail((skip + conv1x1_skip(z)) * scale), and its y bit for bit the middle layer's y.

The operands are built here as in test_gpu_pwg_layer.py: W1 / W2 and the end vectors from `PWGGenerator._pack`, P = W_aux
conv_in(mel) in float64 on the host, the band table from `compact_band_tables`.
"""
import ctypes as C
import functools
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

# max |kernel - fp64 reference| / max |reference| per utterance and over its first and last 256 rows
LAYER_TOL = 2e-5
TAIL_TOL = 5e-5
SCALES = {300: [4, 5, 3, 5], 256: [4, 4, 4, 4]}
SENTINEL = -3.25                    # y planes and out are filled with it before a launch: windows the kernel skips keep it
TAIL_SCALE = math.sqrt(1.0 / 30)    # the model's scale at 30 layers, not 1 as a one-layer model would have it
BATCHES = {                         # frames per utterance; ragged batches pass lens, the others run without
    "one_frame": ((1,), False),
    "ragged": ((40, 0, 33, 1), True),
    "idle_ctas": ((0, 0, 0, 40), True),
    "many_tiles": ((40,) * 8, False),
}


@functools.lru_cache(maxsize=None)
def _model(hop, device):
    """One-layer generator at the upsample config of `hop`: (packed weights, fp64 params, fp64 FIRs)."""
    from oracle import pwg as opwg
    from parakeet_b200.models import PWGGenerator
    cfg = dict(upsample_scales=SCALES[hop], layers=1, stacks=1)
    params = opwg.synth_params(11, cfg)
    gen = PWGGenerator(**{**opwg.DEFAULT_GENERATOR_PARAMS, **cfg, "use_weight_norm": False}, device=device)
    gen.set_state_dict(params)
    p64 = {k: v.double() for k, v in params.items()}
    firs = [p64[f"upsample_net.upsample.up_layers.{2 * i + 1}.weight"].reshape(-1) for i in range(len(SCALES[hop]))]
    return gen._pack(), p64, firs


@functools.lru_cache(maxsize=None)
def _inputs(hop, frames):
    """noise (B, T) and x (B, T, 64), zero past each utterance, skip (B, T, 64), and each utterance's mel (80, frames + 4)."""
    g = torch.Generator().manual_seed(hop * 17 + sum(frames) * 5 + len(frames))
    T = max(frames) * hop
    noise, x = torch.zeros(len(frames), T), torch.zeros(len(frames), T, 64)
    mels = []
    for b, nf in enumerate(frames):
        noise[b, :nf * hop] = torch.randn(nf * hop, generator=g)
        x[b, :nf * hop] = torch.randn(nf * hop, 64, generator=g)
        mels.append(torch.randn(80, nf + 4, generator=g, dtype=torch.float64))
    skip = torch.randn(len(frames), T, 64, generator=g)
    return noise, x, skip, mels


def _conv_in(p64, mel):
    return F.conv1d(mel[None], p64["upsample_net.conv_in.weight"])[0]


def _operands(hop, frames, noise, x, mels, device):
    from parakeet_b200.models import _pwg_frame_cond as fc
    from parakeet_b200.ops import Split
    _, p64, firs = _model(hop, device)
    B, T = x.shape[:2]
    w_aux = p64["conv_layers.0.conv1x1_aux.weight"][:, :, 0]
    fp = max((max(frames) + 7) // 8 * 8, 64)
    P = torch.zeros(B, 128, fp, dtype=torch.float64)
    for b, nf in enumerate(frames):
        if nf:
            P[b, :, :nf] = w_aux @ _conv_in(p64, mels[b])
    tab, lay, _ = fc.compact_band_tables(firs, SCALES[hop], frames)
    wide = torch.zeros(tab.shape[0], 64)
    wide[:, :fc.KWIN] = tab.float()
    return dict(B=B, T=T, noise=noise.contiguous().to(device), x=Split.from_f32(x.to(device)), P=Split.from_f32(P.float().to(device)),
                p_ld=fp, p_frames=max(frames), U=Split.from_f32(wide.to(device)), lay=lay)


def _launch(mode, hop, ops, dil, lens, skip, skip_init=0):
    """One layer (mode "first", "middle" or "last") into fresh y planes (and out) filled with SENTINEL: (y, out or None)."""
    from parakeet_b200 import _lib
    from parakeet_b200.ops import Split, _stream
    L = _lib.lib()
    pk = _model(hop, skip.device)[0]
    lay, fh, th = pk["layers"][0], pk["first_host"], pk["tail_host"]
    B, T = ops["B"], ops["T"]
    y = Split.empty((B, T, 64), skip.device)
    y.hi.fill_(SENTINEL)
    y.lo.fill_(SENTINEL)
    out = torch.full((B, T), SENTINEL, device=skip.device) if mode == "last" else None
    a = _lib.PwgLayerFcArgs()
    a.batch, a.t, a.dilation, a.hop = B, T, dil, hop
    a.lens = lens.data_ptr() if lens is not None else None
    if mode == "first":
        a.noise = ops["noise"].data_ptr()
    else:
        a.x_hi, a.x_lo = ops["x"].hi.data_ptr(), ops["x"].lo.data_ptr()
    a.y_hi, a.y_lo = y.hi.data_ptr(), y.lo.data_ptr()
    a.w1_hi, a.w1_lo = lay["w1"].hi.data_ptr(), lay["w1"].lo.data_ptr()
    a.w2_hi, a.w2_lo = lay["w2"].hi.data_ptr(), lay["w2"].lo.data_ptr()
    a.bias1, a.bias2 = lay["b1"].ctypes.data, lay["b2"].ctypes.data
    a.skip, a.skip_init = skip.data_ptr(), skip_init
    U, P, ul = ops["U"], ops["P"], ops["lay"]
    a.u_hi, a.u_lo, a.u_rows = U.hi.data_ptr(), U.lo.data_ptr(), U.hi.shape[0]
    a.u_period, a.u_start_row, a.u_end_base = ul["period"], ul["start_row"], ul["end_base"]
    a.p_hi, a.p_lo, a.p_rows, a.p_ld, a.p_frames, a.p_row0 = P.hi.data_ptr(), P.lo.data_ptr(), 128, ops["p_ld"], ops["p_frames"], 0
    a.first_w, a.first_b, a.first_u, a.first_v = fh["w"].ctypes.data, fh["b"].ctypes.data, fh["u"].ctypes.data, fh["v"].ctypes.data
    a.tail_w1_hi, a.tail_w1_lo = th["w1"].hi.data_ptr(), th["w1"].lo.data_ptr()
    a.tail_b1, a.tail_w2, a.tail_b2, a.skip_bias = th["b1"].ctypes.data, th["w2"].ctypes.data, th["b2"].ctypes.data, th["skip_bias"].ctypes.data
    a.tail_scale = TAIL_SCALE
    if mode == "last":
        a.out = out.data_ptr()
    _lib.check(L.pk_pwg_residual_layer_fc(C.byref(a), _stream()), "pk_pwg_residual_layer_fc")
    torch.cuda.synchronize()
    return y, out


def _block(hop, x64, mel, dil, device):
    """float64 ResidualBlock 0 of one utterance: y (n, 64) and its skip branch with its bias, (64, n)."""
    from oracle import pwg as opwg
    _, p64, _ = _model(hop, device)
    c_up = opwg.upsample_net(p64, _conv_in(p64, mel)[None], SCALES[hop])
    y, s = opwg.residual_block(p64, "conv_layers.0.", x64, c_up, dil)
    return y[0].T, s[0]


def _edge_err(got, ref):
    got = got.double().cpu()
    return max(float((got[sl] - ref[sl]).abs().max() / ref[sl].abs().max().clamp_min(1e-30))
               for sl in (slice(None), slice(0, 256), slice(-256, None)))


def _bits(t):
    return t.view(torch.int16) if t.dtype == torch.bfloat16 else t.view(torch.int32)


def _dead_rows_ok(t, n):
    dead = t[n:]
    return bool(((dead == 0) | (dead == SENTINEL)).all())


@pytest.mark.parametrize("batch", list(BATCHES))
@pytest.mark.parametrize("dil", [1, 64])
@pytest.mark.parametrize("hop", [300, 256])
def test_pwg_first_layer_vs_fp64(cuda, record_property, hop, dil, batch):
    """first_conv inside layer 0: y and the skip sum (written over NaN, without its bias) against float64 first_conv +
    ResidualBlock 0 at every live row, zero or untouched y past each length, two launches bit-identical, and each utterance of
    a batch bit-identical to running it alone."""
    frames, ragged = BATCHES[batch]
    _, p64, _ = _model(hop, cuda)
    noise, x, _, mels = _inputs(hop, frames)
    ops = _operands(hop, frames, noise, x, mels, cuda)
    B, T = ops["B"], ops["T"]
    lens = torch.tensor([nf * hop for nf in frames], dtype=torch.int32, device=cuda) if ragged else None
    skip1 = torch.full((B, T, 64), float("nan"), device=cuda)
    y1, _ = _launch("first", hop, ops, dil, lens, skip1, 1)
    skip2 = torch.full((B, T, 64), float("nan"), device=cuda)
    y2, _ = _launch("first", hop, ops, dil, lens, skip2, 1)
    for a, b in ((y1.hi, y2.hi), (y1.lo, y2.lo), (skip1, skip2)):
        assert torch.equal(_bits(a), _bits(b))
    errs = dict(y=0.0, skip=0.0)
    yf = y1.float()
    sb = p64["conv_layers.0.conv1x1_skip.bias"]
    for b, nf in enumerate(frames):
        n = nf * hop
        if n:
            x0 = F.conv1d(noise[b, :n].double()[None, None], p64["first_conv.weight"], p64["first_conv.bias"])
            y_ref, s_ref = _block(hop, x0, mels[b], dil, cuda)
            errs["y"] = max(errs["y"], _edge_err(yf[b, :n], y_ref))
            errs["skip"] = max(errs["skip"], _edge_err(skip1[b, :n], (s_ref - sb[:, None]).T))
        for plane in (y1.hi, y1.lo):
            assert _dead_rows_ok(plane[b], n), (b, nf)
    for k, v in errs.items():
        record_property(k, v)
    assert all(math.isfinite(v) for v in errs.values()) and max(errs.values()) < LAYER_TOL, errs

    if B > 1:
        for b, nf in enumerate(frames):
            if not nf:
                continue
            n = nf * hop
            one = _operands(hop, (nf,), noise[b:b + 1, :n], x[b:b + 1, :n], mels[b:b + 1], cuda)
            s = torch.empty(1, n, 64, device=cuda)
            y, _ = _launch("first", hop, one, dil, None, s, 1)
            assert torch.equal(_bits(y.hi[0]), _bits(y1.hi[b, :n])) and torch.equal(_bits(y.lo[0]), _bits(y1.lo[b, :n]))
            assert torch.equal(_bits(s[0]), _bits(skip1[b, :n])), (b, nf)


@pytest.mark.parametrize("batch", ["ragged", "many_tiles"])
@pytest.mark.parametrize("hop", [300, 256])
def test_pwg_last_layer_tail_vs_fp64(cuda, record_property, hop, batch):
    """The tail in the last layer's epilogue: out against float64 tail((skip + conv1x1_skip(z) + the other layers' skip biases)
    * scale) at every live row, zero or untouched past each length; the skip buffer is read, not written; y bit for bit the
    middle layer's y; two launches bit-identical."""
    frames, ragged = BATCHES[batch]
    dil = 2
    pk, p64, _ = _model(hop, cuda)
    noise, x, skip0, mels = _inputs(hop, frames)
    ops = _operands(hop, frames, noise, x, mels, cuda)
    lens = torch.tensor([nf * hop for nf in frames], dtype=torch.int32, device=cuda) if ragged else None
    skip = skip0.to(cuda)
    y1, out1 = _launch("last", hop, ops, dil, lens, skip)
    assert torch.equal(_bits(skip), _bits(skip0.to(cuda)))
    y2, out2 = _launch("last", hop, ops, dil, lens, skip)
    assert torch.equal(_bits(out1), _bits(out2))
    y_mid, _ = _launch("middle", hop, ops, dil, lens, skip0.clone().to(cuda))
    for a, b in ((y1.hi, y_mid.hi), (y1.lo, y_mid.lo), (y1.hi, y2.hi), (y1.lo, y2.lo)):
        assert torch.equal(_bits(a), _bits(b))
    # this one-layer model's skip-bias sum is its own conv1x1_skip bias, which the float64 block includes
    xs = ops["x"].float().double().cpu()
    err = 0.0
    for b, nf in enumerate(frames):
        n = nf * hop
        if n:
            _, s_ref = _block(hop, xs[b, :n].T[None], mels[b], dil, cuda)
            h = F.relu((skip0[b, :n].double().T + s_ref) * TAIL_SCALE)[None]
            h = F.relu(F.conv1d(h, p64["last_conv_layers.1.weight"], p64["last_conv_layers.1.bias"]))
            ref = F.conv1d(h, p64["last_conv_layers.3.weight"], p64["last_conv_layers.3.bias"])[0, 0]
            err = max(err, _edge_err(out1[b, :n], ref))
        assert _dead_rows_ok(out1[b], n), (b, nf)
    record_property("out", err)
    assert math.isfinite(err) and err < TAIL_TOL, err


def test_pwg_layer_fc_rejects_mixed_ends(cuda):
    """noise and out together, and x planes with noise, are argument errors."""
    from parakeet_b200._lib import PkError
    frames = (2,)
    noise, x, skip0, mels = _inputs(300, frames)
    ops = _operands(300, frames, noise, x, mels, cuda)
    from parakeet_b200 import _lib
    from parakeet_b200.ops import _stream
    a = _lib.PwgLayerFcArgs()
    a.batch, a.t, a.dilation, a.hop = 1, 600, 1, 300
    a.noise, a.out = ops["noise"].data_ptr(), skip0.data_ptr()
    with pytest.raises(PkError, match="exclusive"):
        _lib.check(_lib.lib().pk_pwg_residual_layer_fc(C.byref(a), _stream()), "pk_pwg_residual_layer_fc")
    a.out = None
    a.x_hi = a.x_lo = ops["x"].hi.data_ptr()
    with pytest.raises(PkError, match="x planes"):
        _lib.check(_lib.lib().pk_pwg_residual_layer_fc(C.byref(a), _stream()), "pk_pwg_residual_layer_fc")
