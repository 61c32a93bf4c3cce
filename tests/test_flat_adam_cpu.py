"""FlatAdam's checkpoint entries on the CPU (training/flat.py): only its update needs the CUDA library."""
from collections import OrderedDict

import torch

from parakeet_b200.training import FlatAdam


def _make(seed):
    g = torch.Generator().manual_seed(seed)
    params = OrderedDict((k, torch.randn(shape, generator=g)) for k, shape in (("a.weight", (3, 5)), ("a.bias", (3,)), ("b.weight", (2, 3, 3))))
    opt = FlatAdam(params, list(params), "cpu", clip_norm=1.0)
    return params, opt


def test_moments_round_trip_shapes_suffixes_and_gaps():
    params, src = _make(0)
    assert src.buffers.offsets == [0, 16, 20] and src.buffers.total == 40            # 15 -> 16, 3 -> 4, 18 -> 20: gaps at 15, 19, 38, 39
    assert src.steps == 0 and src.sq.dtype == torch.float64 and FlatAdam(OrderedDict(w=torch.ones(2)), ["w"], "cpu").sq is None
    g = torch.Generator().manual_seed(1)
    src.m.copy_(torch.randn(40, generator=g))
    src.v.copy_(torch.rand(40, generator=g))
    opt = src.moments()
    assert set(opt) == {k + s for k in params for s in ("_moment1_0", "_moment2_0")}
    for k, p in params.items():
        assert opt[k + "_moment1_0"].shape == p.shape and opt[k + "_moment2_0"].shape == p.shape
    assert torch.equal(opt["a.bias_moment2_0"], src.v[16:19])
    opt["a.bias_moment1_0"][0] = 7.0
    assert src.m[16] != 7.0                                                          # clones, not views
    _, dst = _make(2)
    dst.m.fill_(-1.0)
    dst.v.fill_(-2.0)
    dst.load_moments(opt)
    gaps = torch.tensor([15, 19, 38, 39])
    keep = torch.ones(40, dtype=torch.bool)
    keep[gaps] = False
    want_m = src.m.clone()
    want_m[16] = 7.0
    assert torch.equal(dst.m[keep], want_m[keep]) and torch.equal(dst.v[keep], src.v[keep])
    assert dst.m[gaps].eq(-1.0).all() and dst.v[gaps].eq(-2.0).all()                # the padding between aligned views is not touched


def test_load_moments_skips_absent_keys_and_takes_arrays():
    _, opt = _make(3)
    opt.m.fill_(0.5)
    opt.v.fill_(0.25)
    opt.load_moments({"a.bias_moment1_0": torch.arange(3.0).numpy(), "b.weight_moment2_0": torch.full((18,), 9.0), "step_count": 4})
    assert torch.equal(opt.m[16:19], torch.arange(3.0)) and opt.m[:16].eq(0.5).all() and opt.m[19:].eq(0.5).all()
    assert opt.v[20:38].eq(9.0).all() and opt.v[:20].eq(0.25).all() and opt.v[38:].eq(0.25).all()
    assert opt.steps == 0
