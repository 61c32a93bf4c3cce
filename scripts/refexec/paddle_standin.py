"""A torch-backed stand-in for the slice of the PaddlePaddle API that the reference's hot-path model code calls, so that the
REFERENCE'S OWN PYTHON (module wiring, masks, transposes, scalings, residuals, dilation rules ...) can be executed in this
container, where Paddle cannot be installed.  Used only by scripts/make_golden_ref.py to write tests/golden/ref_executed*.npz.

What this pins and what it does not: every line of the reference's model code runs as written; each Paddle primitive it calls
is mapped to the torch primitive of the same mathematical definition.  The handful of Paddle semantics that differ from torch
or are not obvious are implemented the way oracle/README.md records them (Linear weight [in, out]; Embedding(padding_idx)
returns zeros; round half away from zero; BatchNorm eval with _mean / _variance, eps 1e-5; transpose takes a permutation) -
those remain restated decisions, everything else becomes executed reference code.
"""
import math
import sys
import types

import torch
import torch.nn.functional as TF


class Tensor(torch.Tensor):
    """torch.Tensor with Paddle's method spellings (results of torch ops on it stay of this class)."""

    def cast(self, dtype=None):
        return self.to(_dt(dtype))

    def astype(self, dtype):
        return self.to(_dt(dtype))

    def transpose(self, *perm):
        if len(perm) == 1 and isinstance(perm[0], (list, tuple)):
            return self.permute(*perm[0])
        return torch.Tensor.transpose(self, *perm)

    def numpy(self):
        return self.detach().as_subclass(torch.Tensor).numpy()

    def sum(self, axis=None, keepdim=False, dtype=None, **kw):
        if "dim" in kw:
            axis = kw["dim"]
        return torch.sum(self, dim=axis, keepdim=keepdim) if axis is not None else torch.sum(self)

    def mean(self, axis=None, keepdim=False, **kw):
        if "dim" in kw:
            axis = kw["dim"]
        return torch.mean(self, dim=axis, keepdim=keepdim) if axis is not None else torch.mean(self)

    def max(self, axis=None, keepdim=False, **kw):
        if axis is None and not kw:
            return torch.max(self)
        return torch.max(self, dim=kw.get("dim", axis), keepdim=keepdim).values

    def expand(self, *shape, **kw):                      # paddle: Tensor.expand(shape=[...]) (-1 keeps a dimension)
        if "shape" in kw:
            shape = kw["shape"]
        if len(shape) == 1 and isinstance(shape[0], (list, tuple)):
            shape = shape[0]
        return torch.Tensor.expand(self, *shape)

    def tile(self, reps):
        return torch.Tensor.repeat(self, *reps)

    def unsqueeze(self, axis):
        if isinstance(axis, (list, tuple)):                 # paddle accepts a list of axes, applied in order
            out = self
            for a in axis:
                out = torch.Tensor.unsqueeze(out, a)
            return out
        return torch.Tensor.unsqueeze(self, axis)

    @property
    def size(self):
        """paddle: Tensor.size is the element count (an int); torch: Tensor.size(dim) is a method.  Both spellings work."""
        return _Size(self)

    def squeeze(self, axis=None):
        return torch.Tensor.squeeze(self) if axis is None else torch.Tensor.squeeze(self, axis)

    def flatten(self, start_axis=0, stop_axis=-1):
        return torch.Tensor.flatten(self, start_axis, stop_axis)

    @property
    def place(self):
        return "cpu"

    def real(self):
        return torch.real(self)

    def imag(self):
        return torch.imag(self)

    @property
    def name(self):                                  # paddle tensors carry auto-generated unique names
        n = getattr(self, "_pk_name", None)
        if n is None:
            Tensor._counter += 1
            n = f"generated_tensor_{Tensor._counter}"
            self._pk_name = n
        return n

    @property
    def stop_gradient(self):
        return not self.requires_grad

    @stop_gradient.setter
    def stop_gradient(self, v):
        pass


Tensor._counter = 0


class Parameter(torch.nn.Parameter):
    def _grad_ivar(self):                                # the gradient tensor itself (written in place by do_gradient_ops)
        return self.grad


class _Size(int):
    def __new__(cls, t):
        obj = super().__new__(cls, t.numel())
        obj._shape = t.shape
        return obj

    def __call__(self, dim=None):
        return self._shape if dim is None else self._shape[dim]


def T(x):
    return x.as_subclass(Tensor) if isinstance(x, torch.Tensor) else x


_DT = {"float32": torch.float32, "float64": torch.float64, "int64": torch.int64, "int32": torch.int32, "bool": torch.bool,
       "float": torch.float32, "int": torch.int64, "uint8": torch.uint8}


def _dt(d):
    if d is None or isinstance(d, torch.dtype):
        return d
    return _DT[str(d)]


def build():
    P = types.ModuleType("paddle")
    P.Tensor = Tensor
    P.float32, P.float64, P.int64, P.int32, P.bool, P.uint8 = torch.float32, torch.float64, torch.int64, torch.int32, torch.bool, torch.uint8
    P.dtype = torch.dtype
    def to_tensor(x, dtype=None, place=None, stop_gradient=True):
        t = torch.as_tensor(x)
        if t.dim() == 0:
            t = t.reshape(1)                       # Paddle 2.1 has no 0-D tensors: a python scalar becomes shape [1]
        if t.dtype == torch.float64 and dtype is None and not isinstance(x, torch.Tensor):
            t = t.float()                          # python floats / float64 numpy default to the default dtype only for python floats
            if hasattr(x, "dtype"):
                t = torch.as_tensor(x)             # numpy arrays keep their dtype
        return T(t.to(_dt(dtype)) if dtype is not None else t)
    P.to_tensor = to_tensor
    P.cast = lambda x, dtype: T(x.to(_dt(dtype)))
    P.concat = lambda xs, axis=0: T(torch.cat(list(xs), dim=axis))
    P.stack = lambda xs, axis=0: T(torch.stack(list(xs), dim=axis))
    P.ones = lambda shape, dtype=None: T(torch.ones(tuple(shape), dtype=_dt(dtype) or torch.float32))
    P.zeros = lambda shape, dtype=None: T(torch.zeros(tuple(shape), dtype=_dt(dtype) or torch.float32))
    P.full = lambda shape, v, dtype=None: T(torch.full(tuple(shape), v, dtype=_dt(dtype) or torch.float32))
    P.ones_like = lambda x, dtype=None: T(torch.ones_like(x, dtype=_dt(dtype)))
    P.zeros_like = lambda x, dtype=None: T(torch.zeros_like(x, dtype=_dt(dtype)))
    P.meshgrid = lambda *xs: [T(t) for t in torch.meshgrid(*xs, indexing="ij")]       # paddle.meshgrid: 'ij' indexing
    P.arange = lambda start, end=None, step=1, dtype=None: T(torch.arange(start, end, step, dtype=_dt(dtype)) if end is not None else torch.arange(start, dtype=_dt(dtype)))
    P.reshape = lambda x, shape: T(x.reshape(tuple(shape)))
    P.transpose = lambda x, perm: T(x.permute(*perm))
    P.matmul = lambda a, b, transpose_x=False, transpose_y=False: T(torch.matmul(a.transpose(-1, -2) if transpose_x else a, torch.Tensor.transpose(b, -1, -2) if transpose_y else b))
    P.round = lambda x: T(torch.sign(x) * torch.floor(torch.abs(x) + 0.5))          # C round(): half away from zero
    P.logical_not = lambda x: T(torch.logical_not(x))
    P.logical_and = lambda x, y: T(torch.logical_and(x, y))
    P.where = lambda c, a, b: T(torch.where(c, a, b))
    P.tril = lambda x, diagonal=0: T(torch.tril(x, diagonal))
    P.sin, P.cos, P.exp, P.log, P.sqrt, P.abs, P.tanh = (lambda f: (lambda x: T(f(x))))(torch.sin), None, None, None, None, None, None
    for name, f in (("sin", torch.sin), ("cos", torch.cos), ("exp", torch.exp), ("log", torch.log), ("sqrt", torch.sqrt),
                    ("abs", torch.abs), ("tanh", torch.tanh)):
        setattr(P, name, (lambda f: (lambda x: T(f(x))))(f))
    P.clip = lambda x, min=None, max=None: T(torch.clamp(x, min=min, max=max))
    P.expand = lambda x, shape: T(torch.Tensor.expand(x, *shape))
    P.broadcast_shape = lambda a, b: list(torch.broadcast_shapes(tuple(a), tuple(b)))
    P.sum = lambda x, axis=None, keepdim=False: T(torch.sum(x, dim=axis, keepdim=keepdim) if axis is not None else torch.sum(x))
    P.mean = lambda x, axis=None, keepdim=False: T(torch.mean(x, dim=axis, keepdim=keepdim) if axis is not None else torch.mean(x))
    P.randn = lambda shape, dtype=None: T(torch.randn(tuple(shape)))
    P.no_grad = torch.no_grad
    P.chunk = lambda x, chunks, axis=0: [T(t) for t in torch.chunk(x, chunks, dim=axis)]
    P.split = lambda x, n, axis=0: [T(t) for t in (torch.chunk(x, n, dim=axis) if isinstance(n, int) else torch.split(x, list(n), dim=axis))]
    P.unsqueeze = lambda x, axis: T(x).unsqueeze(axis)                           # an int or a list of axes
    P.argmax = lambda x, axis=None: T(torch.argmax(x) if axis is None else torch.argmax(x, dim=axis))   # first index on ties
    P.exp = lambda x: T(torch.exp(x))
    P.tanh = lambda x: T(torch.tanh(x))
    P.squeeze = lambda x, axis=None: T(torch.squeeze(x) if axis is None else torch.squeeze(x, axis))
    P.shape = lambda x: list(x.shape)
    P.divide = lambda a, b: T(a / b)
    P.norm = lambda x, p="fro", axis=None, keepdim=False: T(torch.linalg.norm(x.reshape(-1)) if (axis is None and p == "fro") else torch.norm(x, p=p, dim=axis, keepdim=keepdim))
    sig = types.ModuleType("paddle.signal")

    def p_stft(x, n_fft, hop_length=None, win_length=None, window=None, center=True, pad_mode="reflect", normalized=False, onesided=True):
        # paddle.signal.stft is a Paddle kernel: mapped to torch.stft of the same definition (window centre-padded to n_fft)
        w = window.to(x.dtype) if window is not None else None
        return T(torch.stft(x, n_fft, hop_length, win_length, window=w, center=center, pad_mode=pad_mode, normalized=normalized,
                            onesided=onesided, return_complex=True))
    sig.stft = p_stft
    P.signal = sig
    P.subtract = lambda a, b: T(a - b)
    P.maximum = lambda a, b: T(torch.maximum(a, b))
    P.get_default_dtype = lambda: "float32"
    P.multiply = lambda a, b: T(a * b)
    P.bmm = lambda a, b: T(torch.bmm(a, b))
    P.broadcast_to = lambda x, shape: T(torch.Tensor.expand(x, *shape))

    def scatter(x, index, updates, overwrite=True):
        """paddle.scatter along axis 0; overwrite=True: rows of `index` take the rows of `updates` (unique indices here)."""
        assert overwrite
        return T(x.index_put((index.reshape(-1).to(torch.int64),), updates))
    P.scatter = scatter
    P.add = lambda a, b: T(a + b)

    def create_parameter(shape, dtype="float32", default_initializer=None, attr=None, is_bias=False):
        p = Parameter(torch.zeros(tuple(shape), dtype=_dt(dtype) or torch.float32))
        if default_initializer is not None:
            default_initializer(p)
        return p
    P.create_parameter = create_parameter

    # ---------------------------------------------------------------- nn
    nn = types.ModuleType("paddle.nn")

    class Layer(torch.nn.Module):
        def __call__(self, *a, **k):
            out = super().__call__(*[T(x) for x in a], **{key: T(v) for key, v in k.items()})
            return out

        def create_parameter(self, shape, attr=None, dtype="float32", is_bias=False, default_initializer=None):
            return create_parameter(shape, dtype, default_initializer)

        def add_sublayer(self, name, layer):
            self.add_module(str(name), layer)
            return layer

        def add_parameter(self, name, p):
            self.register_parameter(name, p)
            return p

        def named_sublayers(self, prefix="", include_self=False):
            return [(n, m) for n, m in self.named_modules(prefix=prefix) if include_self or m is not self]

        def sublayers(self, include_self=False):
            return [m for m in self.modules() if include_self or m is not self]

        def set_state_dict(self, sd):
            own = dict(self.named_parameters())
            own.update(dict(self.named_buffers()))
            missing = [k for k in own if k not in sd and "generated_tensor_" not in k]      # auto-named index buffers
            extra = [k for k in sd if k not in own]
            if missing or extra:
                raise KeyError(f"state dict mismatch: missing {missing[:6]} unexpected {extra[:6]}")
            with torch.no_grad():
                for k, v in own.items():
                    if k in sd:
                        v.copy_(torch.as_tensor(sd[k]).reshape(v.shape))

        def apply(self, fn):
            for m in self.children():
                m.apply(fn) if isinstance(m, Layer) else torch.nn.Module.apply(m, fn)
            fn(self)
            return self
    nn.Layer = Layer

    class Linear(Layer):
        def __init__(self, in_features, out_features, weight_attr=None, bias_attr=None, name=None):
            super().__init__()
            self.weight = torch.nn.Parameter(torch.zeros(in_features, out_features))          # paddle: [in, out]
            self.bias = torch.nn.Parameter(torch.zeros(out_features)) if bias_attr is not False else None

        def forward(self, x):
            y = torch.matmul(x, self.weight)
            return y + self.bias if self.bias is not None else y
    nn.Linear = Linear

    def _pad(p, k, d):
        """-> (dilation, left, right).  padding="same" is Paddle's rule (models/speedyspeech.py `paddle_same_conv`): undilated,
        the extra row of an even kernel on the right."""
        if isinstance(p, str):
            assert p.lower() == "same"
            from parakeet_b200.models.speedyspeech import paddle_same_conv
            return paddle_same_conv(k, d)
        if isinstance(p, (list, tuple)):
            assert len(p) == 1 or p[0] == p[1]
            return d, int(p[0]), int(p[0])
        return d, int(p), int(p)

    class Conv1D(Layer):
        def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, padding_mode="zeros",
                     weight_attr=None, bias_attr=None, data_format="NCL"):
            super().__init__()
            assert data_format in ("NCL", "NLC") and padding_mode == "zeros"
            self.weight = torch.nn.Parameter(torch.zeros(out_channels, in_channels // groups, kernel_size))
            self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias_attr is not False else None
            d, left, right = _pad(padding, kernel_size, dilation)
            self.args = (stride, (left, right), d, groups)
            self._nlc = data_format == "NLC"

        def forward(self, x):
            s, (left, right), d, g = self.args
            if self._nlc:
                x = x.transpose(1, 2)
            if left == right:
                y = TF.conv1d(x, self.weight, self.bias, s, left, d, g)
            else:
                y = TF.conv1d(TF.pad(x, (left, right)), self.weight, self.bias, s, 0, d, g)
            return y.transpose(1, 2) if self._nlc else y
    nn.Conv1D = Conv1D

    class Conv2D(Layer):
        def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, padding_mode="zeros",
                     weight_attr=None, bias_attr=None, data_format="NCHW"):
            super().__init__()
            ks = tuple(kernel_size) if isinstance(kernel_size, (list, tuple)) else (kernel_size, kernel_size)
            self.weight = torch.nn.Parameter(torch.zeros(out_channels, in_channels // groups, *ks))
            self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias_attr is not False else None
            self.args = (stride, tuple(padding) if isinstance(padding, (list, tuple)) else padding, dilation, groups)

        def forward(self, x):
            s, p, d, g = self.args
            if isinstance(p, tuple) and len(p) == 4:            # paddle: [top, bottom, left, right] (asymmetric, e.g. causal)
                x = TF.pad(x, (p[2], p[3], p[0], p[1]))
                p = 0
            return TF.conv2d(x, self.weight, self.bias, s, p, d, g)
    nn.Conv2D = Conv2D

    class Conv2DTranspose(Layer):
        def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, output_padding=0, groups=1, dilation=1,
                     weight_attr=None, bias_attr=None, data_format="NCHW"):
            super().__init__()
            ks = tuple(kernel_size) if isinstance(kernel_size, (list, tuple)) else (kernel_size, kernel_size)
            self._kernel_size = list(ks)
            self._stride = list(stride) if isinstance(stride, (list, tuple)) else [stride, stride]
            self.weight = torch.nn.Parameter(torch.zeros(in_channels, out_channels // groups, *ks))     # paddle: [in, out, kh, kw]
            self.bias = torch.nn.Parameter(torch.zeros(out_channels)) if bias_attr is not False else None
            self.args = (tuple(stride) if isinstance(stride, (list, tuple)) else stride,
                         tuple(padding) if isinstance(padding, (list, tuple)) else padding, output_padding, groups, dilation)

        def forward(self, x):
            s, p, op, g, d = self.args
            return TF.conv_transpose2d(x, self.weight, self.bias, s, p, op, g, d)
    nn.Conv2DTranspose = Conv2DTranspose

    class LayerNorm(Layer):
        def __init__(self, normalized_shape, epsilon=1e-5, weight_attr=None, bias_attr=None, name=None):
            super().__init__()
            shape = (normalized_shape,) if isinstance(normalized_shape, int) else tuple(normalized_shape)
            self.weight = torch.nn.Parameter(torch.ones(shape))
            self.bias = torch.nn.Parameter(torch.zeros(shape))
            self._shape, self._eps = shape, epsilon

        def forward(self, x):
            return TF.layer_norm(x, self._shape, self.weight, self.bias, self._eps)
    nn.LayerNorm = LayerNorm

    class BatchNorm1D(Layer):
        def __init__(self, num_features, momentum=0.9, epsilon=1e-5, weight_attr=None, bias_attr=None, data_format="NCL", name=None):
            super().__init__()
            self.weight = torch.nn.Parameter(torch.ones(num_features))
            self.bias = torch.nn.Parameter(torch.zeros(num_features))
            self.register_buffer("_mean", torch.zeros(num_features))
            self.register_buffer("_variance", torch.ones(num_features))
            self._eps, self._momentum = epsilon, momentum
            self._nlc = data_format == "NLC"

        def forward(self, x):
            if self._nlc:
                return self._ncl(x.transpose(1, 2)).transpose(1, 2)
            return self._ncl(x)

        def _ncl(self, x):
            if self.training:
                # restated Paddle semantics (oracle/README.md): normalise with the biased batch variance; running statistics
                # move by (1 - momentum) with momentum 0.9 and keep the BIASED variance
                mean = x.mean(dim=(0, 2))
                var = x.var(dim=(0, 2), unbiased=False)
                with torch.no_grad():
                    self._mean.mul_(self._momentum).add_((1 - self._momentum) * mean)
                    self._variance.mul_(self._momentum).add_((1 - self._momentum) * var)
                return (x - mean[None, :, None]) / torch.sqrt(var[None, :, None] + self._eps) * self.weight[None, :, None] \
                    + self.bias[None, :, None]
            return TF.batch_norm(x, self._mean, self._variance, self.weight, self.bias, False, 0.0, self._eps)
    nn.BatchNorm1D = BatchNorm1D

    class Embedding(Layer):
        def __init__(self, num_embeddings, embedding_dim, padding_idx=None, sparse=False, weight_attr=None, name=None):
            super().__init__()
            self.weight = torch.nn.Parameter(torch.zeros(num_embeddings, embedding_dim))
            self._padding_idx = padding_idx

        def forward(self, ids):
            y = TF.embedding(ids, self.weight)
            if self._padding_idx is not None:
                y = y * (ids != self._padding_idx).unsqueeze(-1).to(y.dtype)                    # paddle: padding_idx -> zeros
            return y
    nn.Embedding = Embedding

    class Dropout(Layer):
        def __init__(self, p=0.5, axis=None, mode="upscale_in_train", name=None):
            super().__init__()
            self.p = p

        def forward(self, x):
            assert not self.training or self.p == 0.0, "dropout is only executed with p = 0 or in eval mode (RNG streams differ)"
            return x
    nn.Dropout = Dropout

    class _Act(Layer):
        fn = None

        def __init__(self, *a, **k):
            super().__init__()
            self.a, self.k = a, k

        def forward(self, x):
            return type(self).fn(x, *self.a, **self.k)
    nn.ReLU = type("ReLU", (_Act,), {"fn": staticmethod(lambda x: torch.relu(x))})
    nn.Tanh = type("Tanh", (_Act,), {"fn": staticmethod(lambda x: torch.tanh(x))})
    nn.Sigmoid = type("Sigmoid", (_Act,), {"fn": staticmethod(lambda x: torch.sigmoid(x))})
    nn.LeakyReLU = type("LeakyReLU", (_Act,), {"fn": staticmethod(lambda x, negative_slope=0.01: TF.leaky_relu(x, negative_slope))})
    nn.Softmax = type("Softmax", (_Act,), {"fn": staticmethod(lambda x, axis=-1: torch.softmax(x, dim=axis))})

    class Pad1D(Layer):
        def __init__(self, padding, mode="constant", value=0.0, data_format="NCL"):
            super().__init__()
            self.pad = (padding, padding) if isinstance(padding, int) else tuple(padding)
            self.mode, self.value = mode, value

        def forward(self, x):
            return TF.pad(x, self.pad, mode=self.mode, value=self.value) if self.mode == "constant" else TF.pad(x, self.pad, mode=self.mode)
    nn.Pad1D = Pad1D

    class Sequential(Layer):
        def __init__(self, *layers):
            super().__init__()
            for i, l in enumerate(layers):
                if isinstance(l, (tuple, list)):
                    self.add_module(str(l[0]), l[1])
                else:
                    self.add_module(str(i), l)

        def forward(self, x):
            for m in self.children():
                x = m(x)
            return x

        def __getitem__(self, i):
            return list(self.children())[i]

        def __len__(self):
            return len(list(self.children()))
    nn.Sequential = Sequential

    class LayerList(Layer):
        def __init__(self, layers=None):
            super().__init__()
            for i, l in enumerate(layers or []):
                self.add_module(str(i), l)

        def append(self, l):
            self.add_module(str(len(self)), l)
            return self

        def extend(self, layers):
            for l in layers:
                self.append(l)
            return self

        def __iter__(self):
            return iter(self.children())

        def __len__(self):
            return len(list(self.children()))

        def __getitem__(self, i):
            return list(self.children())[i]
    nn.LayerList = LayerList

    class LSTMCell(Layer):
        def __init__(self, input_size, hidden_size):
            super().__init__()
            self.weight_ih = torch.nn.Parameter(torch.zeros(4 * hidden_size, input_size))
            self.weight_hh = torch.nn.Parameter(torch.zeros(4 * hidden_size, hidden_size))
            self.bias_ih = torch.nn.Parameter(torch.zeros(4 * hidden_size))
            self.bias_hh = torch.nn.Parameter(torch.zeros(4 * hidden_size))

        def forward(self, inputs, states=None):
            """paddle.nn.LSTMCell: -> (h, (h, c)); states default to zeros."""
            if states is None:
                z = torch.zeros(inputs.shape[0], self.weight_hh.shape[1], dtype=inputs.dtype)
                states = (z, z)
            h, c = torch._VF.lstm_cell(inputs, tuple(states), self.weight_ih, self.weight_hh, self.bias_ih, self.bias_hh)
            return T(h), (T(h), T(c))

    class BiRNN(Layer):
        """paddle.nn.BiRNN (2.1): keys `cell_fw.*`, `cell_bw.*`."""
        def __init__(self, cell_fw, cell_bw):
            super().__init__()
            self.cell_fw, self.cell_bw = cell_fw, cell_bw

    def _run(cell, x, lens, reverse):
        """Paddle 2.1's dynamic-graph RNN loop (rnn.py `_rnn_dynamic_graph`): the reverse direction runs over the whole padded
        sequence flipped in time; with sequence_length, a step past a sequence's length keeps the previous state (the mask), and
        every step's output is kept as computed."""
        B, L = x.shape[0], x.shape[1]
        H = cell.weight_hh.shape[1]
        h = c = torch.zeros(B, H, dtype=x.dtype)
        order = range(L - 1, -1, -1) if reverse else range(L)
        outs = [None] * L
        for t in order:
            hn, cn = torch._VF.lstm_cell(x[:, t], (h, c), cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)
            outs[t] = hn
            if lens is not None:
                m = (t < lens).to(x.dtype).unsqueeze(-1)
                hn, cn = m * hn + (1 - m) * h, m * cn + (1 - m) * c
            h, c = hn, cn
        return torch.stack(outs, 1), h, c

    class RNN(Layer):
        def __init__(self, cell):
            super().__init__()
            self.cell = cell

    class LSTM(Layer):
        """paddle.nn.LSTM (2.1): a LayerList of RNN(LSTMCell), so the keys are `{l}.cell.weight_ih` ...; input (B, T, I)
        (time_major=False), returns (out, (h, c)) with h, c [num_layers, B, H].  The cell is torch's lstm_cell (gates i, f, g, o,
        both biases added)."""
        def __init__(self, input_size, hidden_size, num_layers=1, direction="forward", time_major=False, dropout=0.0):
            super().__init__()
            assert direction in ("forward", "bidirectional", "bidirect") and not time_major and dropout == 0.0
            self.bidirectional = direction != "forward"
            for l in range(num_layers):
                if self.bidirectional:
                    assert num_layers == 1
                    self.add_module(str(l), BiRNN(LSTMCell(input_size, hidden_size), LSTMCell(input_size, hidden_size)))
                else:
                    self.add_module(str(l), RNN(LSTMCell(input_size if l == 0 else hidden_size, hidden_size)))
            self.num_layers, self.hidden_size = num_layers, hidden_size

        def forward(self, inputs, initial_states=None, sequence_length=None):
            if self.bidirectional:
                assert initial_states is None
                birnn = getattr(self, "0")
                lens = None if sequence_length is None else torch.as_tensor(sequence_length).reshape(-1, 1).to(torch.int64).reshape(-1)
                of, hf, cf = _run(birnn.cell_fw, inputs, lens, False)
                ob, hb, cb = _run(birnn.cell_bw, inputs, lens, True)
                return T(torch.cat([of, ob], -1)), (T(torch.stack([hf, hb])), T(torch.stack([cf, cb])))
            assert sequence_length is None
            B = inputs.shape[0]
            x, hs, cs = inputs, [], []
            for l, rnn in enumerate(self.children()):
                if initial_states is None:
                    h = c = torch.zeros(B, self.hidden_size, dtype=inputs.dtype)
                else:
                    h, c = initial_states[0][l], initial_states[1][l]
                outs = []
                for t in range(x.shape[1]):
                    cell = rnn.cell
                    h, c = torch._VF.lstm_cell(x[:, t], (h, c), cell.weight_ih, cell.weight_hh, cell.bias_ih, cell.bias_hh)
                    outs.append(h)
                x = torch.stack(outs, 1)
                hs.append(h)
                cs.append(c)
            return T(x), (T(torch.stack(hs)), T(torch.stack(cs)))
    nn.LSTMCell, nn.RNN, nn.LSTM = LSTMCell, RNN, LSTM

    def cross_entropy_loss(weight=None, ignore_index=-100, reduction="mean", soft_label=False, axis=-1):
        assert weight is None and not soft_label and axis == -1
        return lambda x, label: T(TF.cross_entropy(x, label.reshape(-1), ignore_index=ignore_index, reduction=reduction))
    nn.CrossEntropyLoss = cross_entropy_loss
    nn.MSELoss = lambda reduction="mean": (lambda a, b: T(TF.mse_loss(a, b, reduction=reduction)))
    nn.L1Loss = lambda reduction="mean": (lambda a, b: T(TF.l1_loss(a, b, reduction=reduction)))
    nn.BCEWithLogitsLoss = lambda weight=None, reduction="mean", pos_weight=None: \
        (lambda a, b: T(TF.binary_cross_entropy_with_logits(a, b.to(a.dtype), reduction=reduction, weight=weight,
                                                            pos_weight=None if pos_weight is None else torch.as_tensor(pos_weight).to(a.dtype))))

    init = types.ModuleType("paddle.nn.initializer")
    for name in ("XavierUniform", "XavierNormal", "KaimingUniform", "KaimingNormal", "Uniform", "Normal"):
        setattr(init, name, lambda *a, **k: None)                                            # weights are loaded afterwards
    init.Constant = lambda value=0.0: (lambda p: torch.nn.init.constant_(p, value))
    init.Assign = lambda value: (lambda p: p.data.copy_(torch.as_tensor(value).reshape(p.shape)))
    init.set_global_initializer = lambda *a, **k: None
    nn.initializer = init

    F = types.ModuleType("paddle.nn.functional")
    F.softmax = lambda x, axis=-1: T(torch.softmax(x, dim=axis))
    F.log_softmax = lambda x, axis=-1: T(torch.log_softmax(x, dim=axis))
    def f_dropout(x, p=0.5, training=True, **k):
        assert (not training) or p == 0.0, "F.dropout is only executed with p = 0 or training=False"
        return x
    F.dropout = f_dropout
    F.relu = lambda x: T(torch.relu(x))
    F.l1_loss = lambda a, b, reduction="mean": T(TF.l1_loss(a, b, reduction=reduction))
    F.mse_loss = lambda a, b, reduction="mean": T(TF.mse_loss(a, b, reduction=reduction))
    F.leaky_relu = lambda x, negative_slope=0.01: T(TF.leaky_relu(x, negative_slope))
    F.sigmoid = lambda x: T(torch.sigmoid(x))
    F.one_hot = lambda x, num_classes: T(TF.one_hot(torch.as_tensor(x).to(torch.int64), num_classes).to(torch.float32))
    F.tanh = lambda x: T(torch.tanh(x))
    F.conv1d = lambda x, w, bias=None, stride=1, padding=0, dilation=1, groups=1: T(TF.conv1d(x, w, bias, stride, padding, dilation, groups))
    def conv2d(x, w, bias=None, stride=1, padding=0, dilation=1, groups=1, data_format="NCHW"):
        if isinstance(padding, (list, tuple)) and len(padding) == 4:            # paddle: [top, bottom, left, right]
            top, bottom, left, right = padding
            x = TF.pad(x, (left, right, top, bottom))
            padding = 0
        return T(TF.conv2d(x, w, bias, stride, tuple(padding) if isinstance(padding, (list, tuple)) else padding,
                           tuple(dilation) if isinstance(dilation, (list, tuple)) else dilation, groups))
    F.conv2d = conv2d
    F.normalize = lambda x, p=2, axis=1, epsilon=1e-12: T(TF.normalize(x, p=p, dim=axis, eps=epsilon))
    F.pad = lambda x, pad, mode="constant", value=0.0, data_format="NCL": T(TF.pad(x, tuple(pad), mode=mode, value=value) if mode == "constant" else TF.pad(x, tuple(pad), mode=mode))
    F.interpolate = lambda x, size=None, scale_factor=None, mode="nearest", **k: T(TF.interpolate(x, size=size, scale_factor=scale_factor, mode=mode))
    def sequence_mask(x, maxlen=None, dtype="int64", name=None):
        """fluid.layers.sequence_mask / F.sequence_mask: mask[..., j] = j < x[...], maxlen defaults to max(x)."""
        n = int(x.max()) if maxlen is None else int(maxlen)
        return T((torch.arange(n) < torch.as_tensor(x).unsqueeze(-1)).to(_dt(dtype)))
    F.sequence_mask = sequence_mask

    def huber_loss(input, label, delta):
        """fluid.layers.huber_loss (huber_loss_op.h): r = label - input; 0.5 r^2 where |r| <= delta, else delta (|r| - 0.5 delta)."""
        r = label - input
        return T(torch.where(r.abs() <= delta, 0.5 * r * r, delta * (r.abs() - 0.5 * delta)))
    fluid = types.ModuleType("paddle.fluid")
    fluid.layers = types.ModuleType("paddle.fluid.layers")
    fluid.layers.sequence_mask, fluid.layers.huber_loss = sequence_mask, huber_loss
    P.fluid = fluid
    nn.functional = F

    utils = types.ModuleType("paddle.nn.utils")

    def weight_norm(layer, name="weight", dim=0):
        """paddle.nn.utils.weight_norm: w = g * v / ||v||, the norm over every axis but `dim`; weight_g is 1-D [w.shape[dim]]."""
        w = getattr(layer, name)
        del layer._parameters[name]
        axes = [a for a in range(w.dim()) if a != dim]
        g = torch.sqrt((w.detach() ** 2).sum(dim=axes))
        layer.register_parameter(name + "_g", torch.nn.Parameter(g.clone()))
        layer.register_parameter(name + "_v", torch.nn.Parameter(w.detach().clone()))
        shape = [1] * w.dim()
        shape[dim] = -1

        def hook(mod, inputs):
            v, gg = getattr(mod, name + "_v"), getattr(mod, name + "_g")
            norm = torch.sqrt((v ** 2).sum(dim=axes, keepdim=True))
            object.__setattr__(mod, name, gg.reshape(shape) * v / norm)
        layer.register_forward_pre_hook(hook)
        hook(layer, None)
        return layer
    utils.weight_norm = weight_norm
    utils.remove_weight_norm = lambda layer: layer
    nn.utils = utils
    P.nn = nn
    dist = types.ModuleType("paddle.distributed")          # imported by parakeet/utils/checkpoint.py (not on the executed path)
    dist.get_rank = lambda: 0
    dist.get_world_size = lambda: 1
    P.distributed = dist
    P.gather = lambda x, index, axis=0: T(torch.index_select(x, axis, index.reshape(-1).to(torch.int64)))
    P.index_select = lambda x, index, axis=0: T(torch.index_select(x, axis, index.reshape(-1).to(torch.int64)))
    # librosa is not installed; modules/audio.py imports it at module level.  pad_center (centre zero-padding of the window to
    # n_fft) is restated; filters.mel is NOT provided - MelScale is checked against torchaudio elsewhere, not executed here.
    import numpy as _np
    librosa = types.ModuleType("librosa")
    librosa.util = types.ModuleType("librosa.util")

    def pad_center(data, size, axis=-1, mode="constant"):
        n = data.shape[axis]
        lpad = (size - n) // 2
        widths = [(0, 0)] * data.ndim
        widths[axis] = (lpad, size - n - lpad)
        return _np.pad(data, widths, mode=mode)
    librosa.util.pad_center = pad_center
    tg = types.ModuleType("typeguard")                 # the installed typeguard rejects the reference's `x: int = None` defaults
    tg.check_argument_types = lambda *a, **k: True
    return {"paddle.fluid": fluid, "paddle.fluid.layers": fluid.layers, "typeguard": tg, "librosa": librosa, "librosa.util": librosa.util, "paddle": P, "paddle.distributed": dist, "paddle.signal": sig, "paddle.nn": nn, "paddle.nn.functional": F, "paddle.nn.initializer": init, "paddle.nn.utils": utils}
