"""Light-weight layer library (H100-native re-design of the reference's
``theanompi/models/layers2.py``).

What is kept from the reference: the weight-initialiser classes
(``layers2.py:22-166``), the ``Layer`` base with ``input_layer`` chaining and
``input_shape``/``output_shape``/``print_shape`` (``:169-221``), the layer set
(``Subtract :223``, ``Crop :249``, ``Conv :349``, ``Pool :402``, ``ConvPoolLRN :430``,
``ConvPoolLRN_bc01 :680``, ``BatchNormal :748``, ``CrossChannelNormalization :753``,
``LRN :811``, ``Dimshuffle :825``, ``Flatten :844``, ``Dropout :864``, ``FC :912``,
``Softmax :937``) and the graph helpers (``get_layers/get_params/count_params/
extract_weight_types :1000-1056``).

What is different: there is no symbolic graph.  A layer is an eager callable
(``layer.forward(x)``) whose math is one fused op from :mod:`theanompi_b200.ops`
(hand-written sm_90a kernels on CUDA, torch reference on CPU).  Activations are
NHWC ``(B, H, W, C)`` (bf16 on GPU) instead of c01b; conv filters are stored
OHWI; FC weights ``[n_out, n_in]``.  ``filter_shape`` arguments keep the
reference's ``(C_in, kh, kw, C_out)`` order for API parity.

The module RNG is seeded 23455 exactly like the reference (``layers2.py:14-17``) so
every rank starts from identical weights.
"""
from __future__ import annotations

import os

import numpy as np
import torch

from .. import ops

rng = np.random.RandomState(23455)


def reseed(seed=23455):
    global rng
    rng = np.random.RandomState(seed)


# =========================================================================== initialisers
class Weight(object):
    """Base initialiser: holds ``val`` (a torch fp32 tensor; after the model
    binds its :class:`FlatArena` this tensor aliases the arena)."""

    def __init__(self):
        self.val = None
        self.shape = None
        self.name = None

    def _set(self, np_values, name=None):
        self.np_values = np.asarray(np_values, dtype=np.float32)
        self.val = torch.from_numpy(self.np_values.copy())
        self.shape = tuple(self.np_values.shape)
        self.val.pname = name
        self.name = name

    def save_weight(self, dir, name):
        os.makedirs(dir, exist_ok=True)
        np.save(os.path.join(dir, name + ".npy"), self.val.detach().float().cpu().numpy())

    def load_weight(self, dir, name):
        arr = np.load(os.path.join(dir, name + ".npy"))
        if tuple(arr.shape) != tuple(self.val.shape):
            raise ValueError("shape mismatch loading %s: file %s vs param %s"
                             % (name, arr.shape, tuple(self.val.shape)))
        with torch.no_grad():
            self.val.copy_(torch.from_numpy(arr).to(self.val.device))
            sh = getattr(self.val, "shadow", None)
            if sh is not None:
                sh.copy_(self.val)


class Constant(Weight):
    def __init__(self, shape, val=0):
        super().__init__()
        shape = (int(shape),) if np.isscalar(shape) else tuple(int(s) for s in shape)
        self._set(np.full(shape, val, dtype=np.float32))


class Normal(Weight):
    def __init__(self, shape, mean=0, std=0.01):
        super().__init__()
        self._set(rng.normal(mean, std, tuple(int(s) for s in shape)))


class Uniform(Weight):
    def __init__(self, shape, low, high):
        super().__init__()
        self._set(rng.uniform(low, high, tuple(int(s) for s in shape)))


def _fans(shape):
    """fan_in/fan_out for our storage layouts: FC ``[out,in]``, conv OHWI."""
    shape = tuple(int(s) for s in shape)
    if len(shape) == 2:
        return shape[1], shape[0]
    if len(shape) == 4:
        rf = shape[1] * shape[2]
        return shape[3] * rf, shape[0] * rf
    n = int(np.prod(shape))
    return n, n


class GlorotNormal(Weight):
    def __init__(self, shape, gain=np.sqrt(2)):
        super().__init__()
        fi, fo = _fans(shape)
        std = gain * np.sqrt(2.0 / (fi + fo))
        self._set(rng.normal(0.0, std, tuple(int(s) for s in shape)))


class GlorotUniform(Weight):
    def __init__(self, shape, gain=np.sqrt(2)):
        super().__init__()
        fi, fo = _fans(shape)
        a = gain * np.sqrt(6.0 / (fi + fo))
        self._set(rng.uniform(-a, a, tuple(int(s) for s in shape)))


class HeUniform(Weight):
    def __init__(self, shape, gain=np.sqrt(2)):
        super().__init__()
        fi, _ = _fans(shape)
        a = gain * np.sqrt(3.0 / fi)
        self._set(rng.uniform(-a, a, tuple(int(s) for s in shape)))


class HeNormal(Weight):
    def __init__(self, shape, gain=np.sqrt(2)):
        super().__init__()
        fi, _ = _fans(shape)
        self._set(rng.normal(0.0, gain * np.sqrt(1.0 / fi), tuple(int(s) for s in shape)))


def _tag(t, name, wtype):
    t.pname = name
    t.weight_type = wtype
    t.requires_grad_(True)
    return t


# =========================================================================== base
class Layer(object):
    """Eager layer with reference-style chaining."""

    name = "Layer\t"

    def __init__(self):
        self.params = []
        self.weight_type = []

    def get_input_shape(self, input, input_shape):
        if isinstance(input, Layer):
            self.input_layer = input
            self.input_shape = tuple(input.output_shape)
        else:
            if input_shape is None:
                raise ValueError("first layer needs input_shape")
            self.input_shape = tuple(input_shape)
        return self.input_shape

    def get_output_shape(self, input_shape):
        """Analytic shape inference (the reference evaluated the symbolic graph)."""
        return tuple(input_shape)

    def print_shape(self):
        print("%s\tin %s --> out %s" % (self.name, tuple(self.input_shape), tuple(self.output_shape)))

    def forward(self, x):
        raise NotImplementedError

    __call__ = lambda self, x: self.forward(x)  # noqa: E731


def _conv_out(n, k, s, p):
    return (n + 2 * p - k) // s + 1


# =========================================================================== data layers
class Subtract(Layer):
    """Mean subtraction (ref ``layers2.py:223-247``)."""

    def __init__(self, input, subtract_arr, printinfo=True, input_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.subtract_arr = torch.as_tensor(np.asarray(subtract_arr, dtype=np.float32))
        self.output_shape = self.input_shape
        self.name = "Subtract"
        if printinfo:
            self.print_shape()

    def forward(self, x):
        if self.subtract_arr.device != x.device:
            self.subtract_arr = self.subtract_arr.to(x.device)
        return x - self.subtract_arr.to(x.dtype)


class Crop(Layer):
    """Random crop + mirror inside the step (ref ``layers2.py:249-347``); one
    fused device kernel on CUDA.  ``flag_batch=True`` draws one offset/flip per
    batch, else per image."""

    layers = []

    def __init__(self, input, output_shape, input_shape=None, flag_batch=True, printinfo=True):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.output_shape = tuple(output_shape)
        self.flag_batch = flag_batch
        self.flag_rand = True
        self._rs = np.random.RandomState(1234)
        Crop.layers.append(self)
        self.name = "Crop\t"
        if printinfo:
            self.print_shape()

    def forward(self, x):
        B, H, W, C = x.shape
        ch, cw = self.output_shape[1], self.output_shape[2]
        if self.flag_rand:
            if self.flag_batch:
                oy = np.full(B, self._rs.randint(0, H - ch + 1))
                ox = np.full(B, self._rs.randint(0, W - cw + 1))
                fl = np.full(B, self._rs.randint(0, 2))
            else:
                oy = self._rs.randint(0, H - ch + 1, B)
                ox = self._rs.randint(0, W - cw + 1, B)
                fl = self._rs.randint(0, 2, B)
        else:
            oy = np.full(B, (H - ch) // 2)
            ox = np.full(B, (W - cw) // 2)
            fl = np.zeros(B, dtype=np.int64)
        offs = torch.as_tensor(np.stack([oy, ox], 1).astype(np.int32)).to(x.device, non_blocking=True)
        flips = torch.as_tensor(fl.astype(np.uint8)).to(x.device, non_blocking=True)
        zero = torch.zeros(1, device=x.device)
        return ops.crop_mirror_normalize(x, zero, 1.0, (ch, cw), offs, flips, out_dtype=x.dtype)

    @staticmethod
    def SetRandCropOn():
        for l in Crop.layers:
            l.flag_rand = True

    @staticmethod
    def SetRandCropOff():
        for l in Crop.layers:
            l.flag_rand = False


# =========================================================================== conv / pool
def _ohwi_from_ref(filter_shape):
    cin, kh, kw, cout = (int(s) for s in filter_shape)
    return (cout, kh, kw, cin)


class Conv(Layer):
    """conv + bias + ReLU as ONE fused op (ref ``layers2.py:349-400``)."""

    def __init__(self, input, convstride, padsize, W=None, b=None, filter_shape=None,
                 lib_conv="native", printinfo=True, input_shape=None, output_shape=None,
                 relu=True, group=1):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.convstride, self.padsize, self.relu, self.group = convstride, padsize, relu, group
        if W is None:
            assert filter_shape is not None
            W = Normal(_ohwi_from_ref(filter_shape), mean=0, std=0.01)
        if b is False:                                   # bias-free convolution (a BatchNormal follows)
            b = None
        elif b is None:
            b = Constant((W.shape[0],), val=0.0)
        elif np.isscalar(b):
            b = Constant((W.shape[0],), val=b)
        self.W, self.b = W, b
        _tag(self.W.val, "W", "W")
        self.params, self.weight_type = [self.W.val], ["W"]
        if b is not None:
            _tag(self.b.val, "b", "b")
            self.params.append(self.b.val)
            self.weight_type.append("b")
        self.output_shape = tuple(output_shape) if output_shape else self.get_output_shape(self.input_shape)
        self.name = "Conv (%s)" % lib_conv
        if printinfo:
            self.print_shape()

    def get_output_shape(self, s):
        B, H, W_, C = s
        O, kh, kw, _ = self.W.shape
        return (B, _conv_out(H, kh, self.convstride, self.padsize),
                _conv_out(W_, kw, self.convstride, self.padsize), O)

    def forward(self, x):
        return ops.conv2d_bias_act(x, self.W.val, None if self.b is None else self.b.val, self.convstride, self.padsize,
                                   self.group, self.relu)


class Pool(Layer):
    """max / average pooling (ref ``layers2.py:402-428``)."""

    def __init__(self, input, poolsize, poolstride, poolpad=0, mode="max", printinfo=True,
                 input_shape=None, output_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.poolsize, self.poolstride, self.poolpad, self.mode = poolsize, poolstride, poolpad, mode
        self.output_shape = tuple(output_shape) if output_shape else self.get_output_shape(self.input_shape)
        self.name = "Pool\t"
        if printinfo:
            self.print_shape()

    def get_output_shape(self, s):
        B, H, W_, C = s
        return (B, _conv_out(H, self.poolsize, self.poolstride, self.poolpad),
                _conv_out(W_, self.poolsize, self.poolstride, self.poolpad), C)

    def forward(self, x):
        return ops.pool2d(x, self.poolsize, self.poolstride, self.poolpad,
                          "max" if self.mode == "max" else "avg")


class CrossChannelNormalization(object):
    """LRN functor, ``x / (k + alpha * sum_{window n} x^2) ** beta``
    (ref ``layers2.py:753-809``) — one fused forward and one fused backward kernel."""

    def __init__(self, alpha=1e-4, k=2, beta=0.75, n=5):
        if n % 2 == 0:
            raise NotImplementedError("Only works with odd n for now")
        self.alpha, self.k, self.beta, self.n = alpha, k, beta, n

    def __call__(self, x):
        return ops.lrn(x, self.n, float(self.k), self.alpha, self.beta)


class LRN(Layer):
    def __init__(self, input, input_shape=None, printinfo=True):
        super().__init__()
        self.lrn_func = CrossChannelNormalization()
        self.get_input_shape(input, input_shape)
        self.output_shape = self.input_shape
        self.name = "LRN\t"
        if printinfo:
            self.print_shape()

    def forward(self, x):
        return self.lrn_func(x)


class ConvPoolLRN(Layer):
    """AlexNet block: conv(+bias+ReLU) → max-pool → LRN, with the reference's
    2-group split into two independent parameter sets ``W0,b0,W1,b1``
    (ref ``layers2.py:430-678``)."""

    def __init__(self, input, convstride, padsize, poolsize, poolstride, group, b, W=None,
                 filter_shape=None, poolpad=0, mode="max", lrn=False, lib_conv="native",
                 printinfo=True, input_shape=None, output_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        assert group in (1, 2)
        self.convstride, self.padsize, self.group = convstride, padsize, group
        self.poolsize, self.poolstride, self.poolpad, self.mode = poolsize, poolstride, poolpad, mode
        self.lrn = lrn
        if lrn:
            self.lrn_func = CrossChannelNormalization()
        cin, kh, kw, cout = (int(s) for s in filter_shape)
        self.filter_shape = (cin, kh, kw, cout)
        if group == 1:
            self.W = W if W is not None else Normal((cout, kh, kw, cin), mean=0, std=0.01)
            self.b = Constant((cout,), val=b)
            _tag(self.W.val, "W", "W"); _tag(self.b.val, "b", "b")
            self.params = [self.W.val, self.b.val]
            self.weight_type = ["W", "b"]
        else:
            self.W0 = Normal((cout // 2, kh, kw, cin // 2), mean=0, std=0.01)
            self.b0 = Constant((cout // 2,), val=b)
            self.W1 = Normal((cout // 2, kh, kw, cin // 2), mean=0, std=0.01)
            self.b1 = Constant((cout // 2,), val=b)
            for t, n_, wt in ((self.W0, "W0", "W"), (self.b0, "b0", "b"),
                              (self.W1, "W1", "W"), (self.b1, "b1", "b")):
                _tag(t.val, n_, wt)
            self.params = [self.W0.val, self.b0.val, self.W1.val, self.b1.val]
            self.weight_type = ["W", "b", "W", "b"]
        self.output_shape = tuple(output_shape) if output_shape else self.get_output_shape(self.input_shape)
        self.name = "ConvPoolLRN(%s)" % lib_conv
        if printinfo:
            self.print_shape()

    def get_output_shape(self, s):
        B, H, W_, C = s
        _, kh, kw, cout = self.filter_shape
        h = _conv_out(H, kh, self.convstride, self.padsize)
        w = _conv_out(W_, kw, self.convstride, self.padsize)
        if self.poolsize != 1:
            h = _conv_out(h, self.poolsize, self.poolstride, self.poolpad)
            w = _conv_out(w, self.poolsize, self.poolstride, self.poolpad)
        return (B, h, w, cout)

    def forward(self, x):
        # the pooling layer runs inside the conv's autograd node: its backward is one fused kernel
        # (pool scatter + ReLU mask + bias gradient) instead of three passes over the conv output
        pool = None
        if self.poolsize != 1:
            pool = (self.poolsize, self.poolstride, self.poolpad, "max" if self.mode == "max" else "avg")
        if self.group == 1:
            y = ops.conv2d_bias_act(x, self.W.val, self.b.val, self.convstride, self.padsize, 1, True, pool)
        else:
            y = ops.conv2d_group2_bias_act(x, self.W0.val, self.b0.val, self.W1.val, self.b1.val,
                                           self.convstride, self.padsize, True, pool)
        if self.lrn:
            y = self.lrn_func(y)
        return y


class ConvPoolLRN_bc01(ConvPoolLRN):
    """The reference had a second copy for bc01 inputs (``layers2.py:680-746``).
    With a single NHWC layout the two coincide; kept for API parity."""


class BatchNormal(Layer):
    """Batch normalisation with ``gamma`` / ``beta`` parameters, optionally fused with a residual add and a ReLU
    (``forward(x, residual=None)``) — hand-written forward / backward kernels (``csrc/bn_kernels.cu``).

    The reference's class is an empty stub (``layers2.py:748-751``) while its optimizer and exchanger special-case
    parameters *named* gamma / beta (``opt.py:207-226``, ``exchanger.py:35-43``) and its ResNet50 / Wide-ResNet take
    batch norm from Lasagne / Keras; this layer is what those models are built from here.  Gradients of gamma / beta are
    written straight into the arena's G views; train / eval mode is a global switch like ``Dropout``'s."""

    layers = []

    def __init__(self, input, input_shape=None, eps=1e-5, momentum=0.1, relu=False, gamma=1.0, printinfo=True):
        super().__init__()
        self.get_input_shape(input, input_shape)
        C = self.input_shape[-1]
        self.gamma, self.beta = Constant((C,), float(gamma)), Constant((C,), 0.0)
        _tag(self.gamma.val, "gamma", "b"); _tag(self.beta.val, "beta", "b")
        self.params = [self.gamma.val, self.beta.val]
        self.weight_type = ["b", "b"]
        self.running_mean = torch.zeros(C)
        self.running_var = torch.ones(C)
        self.eps, self.momentum, self.relu = eps, momentum, relu
        self.training = True
        self.update_stats = True       # False: training mode without a running-statistics update (ModelBase.bn_stats_frozen)
        BatchNormal.layers.append(self)
        self.output_shape = self.input_shape
        self.name = "BatchNorm"
        if printinfo:
            self.print_shape()

    def forward(self, x, residual=None, drop=None):
        """``drop``: a drop-path row of the training step (ops/drop_path.py) that scales this layer's output per sample before the
        residual add."""
        if self.running_mean.device != x.device:
            self.running_mean = self.running_mean.to(x.device)
            self.running_var = self.running_var.to(x.device)
        keep = self.update_stats or not self.training
        return ops.batch_norm(x, self.gamma.val, self.beta.val, self.running_mean if keep else None, self.running_var if keep else None,
                              self.training, self.momentum, self.eps, self.relu, residual, drop=drop)

    @staticmethod
    def SetTrainOn():
        for l in BatchNormal.layers:
            l.training = True

    @staticmethod
    def SetTrainOff():
        for l in BatchNormal.layers:
            l.training = False


# =========================================================================== shape layers
class Dimshuffle(Layer):
    def __init__(self, input, new_axis_order, printinfo=True, input_shape=None, output_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.new_axis_order = tuple(new_axis_order)
        self.output_shape = tuple(output_shape) if output_shape else \
            tuple(self.input_shape[i] for i in self.new_axis_order)
        self.name = "Dimshuffle    "
        if printinfo:
            self.print_shape()

    def forward(self, x):
        return x.permute(*self.new_axis_order).contiguous()


class Flatten(Layer):
    """Flatten to ``axis`` dims (ref ``layers2.py:844-862``)."""

    def __init__(self, input, axis=2, printinfo=True, input_shape=None, output_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.axis = axis
        keep = self.input_shape[:axis - 1]
        self.output_shape = tuple(output_shape) if output_shape else \
            tuple(keep) + (int(np.prod(self.input_shape[axis - 1:])),)
        self.name = "Flatten\t"
        if printinfo:
            self.print_shape()

    def forward(self, x):
        return x.reshape(x.shape[:self.axis - 1] + (-1,))


class Dropout(Layer):
    """Dropout with a global on/off switch (ref ``layers2.py:864-908``).
    Train: ``mask * x``; eval: ``(1-p) * x`` — the reference does not use inverted
    scaling.  On CUDA the mask comes from a Philox stream keyed by
    (seed, layer id, device step counter) inside the kernel."""

    layers = []

    def __init__(self, input, n_out=None, prob_drop=0.5, printinfo=True, input_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        self.prob_drop = prob_drop
        self.prob_keep = 1.0 - prob_drop
        self.flag_on = True
        self.layer_id = len(Dropout.layers)
        Dropout.layers.append(self)
        self.output_shape = self.input_shape
        self.name = "Dropout" + str(self.prob_drop)
        if printinfo:
            self.print_shape()

    def forward(self, x):
        return ops.dropout(x, self.prob_drop, self.flag_on, self.layer_id)

    @staticmethod
    def SetDropoutOn():
        for l in Dropout.layers:
            l.flag_on = True

    @staticmethod
    def SetDropoutOff():
        for l in Dropout.layers:
            l.flag_on = False


# =========================================================================== dense / loss
class FC(Layer):
    """FC + bias + ReLU fused (ref ``layers2.py:912-935``).  ``W`` may be given in
    the reference's ``(n_in, n_out)`` shape; it is stored ``[n_out, n_in]``."""

    def __init__(self, input, n_out, W=None, b=None, printinfo=True, input_shape=None, relu=True):
        super().__init__()
        self.get_input_shape(input, input_shape)
        n_in = int(self.input_shape[-1])
        if W is not None and b is not None:
            if tuple(W.shape) == (n_in, n_out) and n_in != n_out:
                W._set(W.np_values.T.copy())
            self.W, self.b = W, b
        else:
            self.W = Normal((n_out, n_in), std=0.005)
            self.b = Constant((n_out,), val=0.1)
        _tag(self.W.val, "W", "W"); _tag(self.b.val, "b", "b")
        self.W.val.rs_ok = True      # dW comes from ONE fp32 GEMM straight into gbuf: eligible for the fused reduce-scatter
        self.relu = relu
        self.params = [self.W.val, self.b.val]
        self.weight_type = ["W", "b"]
        self.output_shape = tuple(self.input_shape[:-1]) + (n_out,)
        self.name = "FC\t"
        if printinfo:
            self.print_shape()

    def forward(self, x):
        return ops.linear_bias_act(x, self.W.val, self.b.val, self.relu)


class Softmax(Layer):
    """Linear + softmax classifier head (ref ``layers2.py:937-997``).  ``forward``
    returns logits; ``negative_log_likelihood / errors / errors_top_x`` come from one
    fused softmax-xent kernel and are cached per forward."""

    def __init__(self, input, n_out, W=None, b=None, printinfo=True, input_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        n_in = int(self.input_shape[-1])
        if W is not None and b is not None:
            if tuple(W.shape) == (n_in, n_out) and n_in != n_out:
                W._set(W.np_values.T.copy())
            self.W, self.b = W, b
        else:
            self.W = Normal((n_out, n_in))
            self.b = Constant((n_out,), val=0)
        _tag(self.W.val, "W", "W"); _tag(self.b.val, "b", "b")
        self.W.val.rs_ok = True      # as FC: the logits' weight gradient is one fp32 GEMM into gbuf
        self.params = [self.W.val, self.b.val]
        self.weight_type = ["W", "b"]
        self.output_shape = tuple(self.input_shape[:-1]) + (n_out,)
        self.name = "Softmax\t"
        self._cache = None
        if printinfo:
            self.print_shape()

    def forward(self, x):
        self.logits = ops.linear_bias_act(x, self.W.val, self.b.val, False)
        self._cache = None
        return self.logits

    def _eval(self, y, label_smoothing=None, mix=None, kd=None):
        """(y, ε, mix, kd, loss, err1, err5) of one launch on this forward's logits, cached per (y, ε, mix record, kd);
        ``label_smoothing`` None takes the cached launch whatever its ε, mix and kd (the errors of a training step are those of its
        loss launch), else ε = 0, no mix and no distillation."""
        c = self._cache
        if c is None or c[0] is not y or (label_smoothing is not None and (c[1] != label_smoothing or c[2] is not mix or c[3] is not kd)):
            eps = label_smoothing or 0.0
            if kd is None:
                out = ops.softmax_xent(self.logits, y, eps, mix)
            else:
                out = ops.softmax_xent_kd(self.logits, y, kd.logits, kd.alpha, kd.temperature, eps, mix)
            self._cache = (y, eps, mix, kd) + tuple(out)
        return self._cache

    @property
    def p_y_given_x(self):
        return torch.softmax(self.logits.float(), dim=1)

    @property
    def y_pred(self):
        return self.logits.argmax(1)

    def negative_log_likelihood(self, y, label_smoothing=0.0, mix=None, kd=None):
        """Mean NLL of ``y``; ``label_smoothing`` ε > 0 gives the cross-entropy against (1 − ε)·onehot + ε / C instead, and a Mixup /
        CutMix record ``mix`` the cross-entropy against its mixed target (ops/mixup.py).  ``kd`` (ops/distill.py: a teacher's logits
        with α and T) makes it the distillation loss (1 − α)·CE + α·T²·KL of ops.softmax_xent_kd."""
        return self._eval(y, label_smoothing, mix, kd)[4]

    def errors(self, y):
        return self._eval(y)[5]

    def errors_top_x(self, y, num_top=5):
        if num_top != 5:
            lg = self.logits.float()
            topk = lg.topk(num_top, dim=1).indices
            return 1.0 - (topk == y[:, None]).any(1).float().mean()
        return self._eval(y)[6]


# =========================================================================== graph helpers
def get_layers(lastlayer):
    """Walk the ``input_layer`` chain back to the first layer (ref ``:1000-1015``)."""
    layers = [lastlayer]
    while hasattr(lastlayer, "input_layer"):
        lastlayer = lastlayer.input_layer
        layers.append(lastlayer)
    return layers[::-1]


def get_params(layers):
    params, weight_types = [], []
    for layer in layers:
        if getattr(layer, "params", None):
            params += layer.params
            weight_types += layer.weight_type
    return params, weight_types


def count_params(params, verbose):
    model_size = 0
    for p in params:
        model_size += p.numel()
        if verbose:
            print(tuple(p.shape))
    if verbose:
        print("model size %.3f M floats" % (float(model_size) / (1024 * 1024)))
    return model_size


def extract_weight_types(params):
    return ["W" if p.dim() > 1 else "b" for p in params]


def forward_chain(layers, x):
    for l in layers:
        x = l.forward(x)
    return x
