"""Channels-last Conv1D / Linear layers of the training steps through pk_conv_gemm: the packed weight operands, the forward, the
data gradient (the conv with flipped taps) and the split-K weight gradient (wgrad.splitk_wgrad), for every step alike.

A Paddle Linear weight is [in, out], a Conv1D weight [out, in, k]; `linear` names the parameter's layout, and the operand
packs, tap shifts and result layout follow from it.  `pad` is the forward's left padding in taps (None: (k - 1) // 2, 'same' for
odd k).  pack_dev pads K to a multiple of 64 and pk_conv_gemm uses k only as ceil(k / 64) chunks, so an input whose channel axis
is wider than the weight's (a 1-channel signal carried 8 wide for the TMA row pitch) multiplies against the plain weight's pack."""
from .. import ops
from ..ops import pack_dev
from . import wgrad


def _dims(w, linear):
    """-> (cout, cin, taps)."""
    return (w.shape[1], w.shape[0], 1) if linear else tuple(w.shape)


class ConvOps:
    def __init__(self, zp):
        self.zp = zp                    # the step's ZeroPlanes (operand planes of the weight gradients)
        self.packs = {}

    def reset(self):
        """Forget the packed weights: called at the start of every forward + backward, which packs the weights of its own step
        (inside a captured graph the pack kernels are part of the graph)."""
        self.packs = {}

    def _packed(self, key, fn):
        v = self.packs.get(key)
        if v is None:
            v = self.packs[key] = fn()
        return v

    def fwd(self, x, key, w, *, linear=False, bias=None, dil=1, pad=None, act=None, residual=None, out_f32=True, out_split=False):
        """x Split (B, T, >= Cin) -> pk_conv_gemm's (y fp32, y Split), each (B, T, Cout).  `key` names the weight's pack."""
        cout, cin, taps = _dims(w, linear)
        wp = self._packed(("f", key), lambda: pack_dev(w.t() if linear else w))
        return ops.conv_gemm(x, wp, n=cout, k=cin, taps=taps, dil=dil, pad=pad, bias=bias, act=act, residual=residual, out_f32=out_f32,
                             out_split=out_split)

    def dgrad(self, dys, key, w, *, linear=False, dil=1, pad=None, residual=None):
        """dys Split (B, T, >= Cout) -> dx fp32 (B, T, Cin) (+ residual): the conv with flipped taps, which pads k - 1 - pad."""
        cout, cin, taps = _dims(w, linear)
        left = (taps - 1) // 2 if pad is None else pad
        wb = self._packed(("b", key), lambda: pack_dev(w if linear else w.flip(-1).permute(1, 0, 2)))
        return ops.conv_gemm(dys, wb, n=cin, k=cout, taps=taps, dil=dil, pad=taps - 1 - left, residual=residual)[0]

    def wgrad(self, x, dys, w, *, linear=False, dil=1, pad=None, out=None):
        """x Split (B, T, >= Cin) saved input, dys Split (B, T, >= Cout) -> dW fp32 in w's layout (written into `out` if given):
        tap j pairs dY[t] with X[t + (j - pad) * dil] over the flattened (batch, time) axis."""
        cout, cin, taps = _dims(w, linear)
        if linear:
            return wgrad.splitk_wgrad(self.zp, x, dys, cout, cin, [0], x_first=True, out=out)
        left = (taps - 1) // 2 if pad is None else pad
        g = wgrad.splitk_wgrad(self.zp, x, dys, cout, cin, [(tap - left) * dil for tap in range(taps)]).permute(1, 2, 0)
        return g if out is None else out.copy_(g)
