"""GoogLeNet / Inception-v1 (ref ``theanompi/models/googlenet.py``): ``Incept`` module
(``:46-181``), ``Aux_tower`` (``:183-273``), network (``:399-648``), loss = main + 0.3·aux1 +
0.3·aux2 (``:640-642``); batch 32 out of 128-image files (``n_subb = 4``), lr 0.005 poly
decay, μ 0.9, wd 2e-4, 90 epochs (``:9-20``).  128 parameter tensors / 13.4 M weights.

Every conv is the fused wgmma conv+bias+ReLU op; 1×1 convolutions skip im2col entirely
(the NHWC activation already is the GEMM operand)."""
from __future__ import annotations

import torch

from .base import ModelBase
from .layers2 import (FC, LRN, Constant, Conv, ConvPoolLRN, Dropout, Flatten, Layer, Normal, Pool, Softmax,
                      get_params)

n_epochs = 90
momentum = 0.90
weight_decay = 0.0002
batch_size = 32
file_batch_size = 128
learning_rate = 0.005
lr_policy = "poly"
use_momentum = True
use_nesterov_momentum = False
input_width = 224
input_height = 224
batch_crop_mirror = False
rand_crop = True
lib_conv = "native"
monitor_grad = False


class Incept(Layer):
    """Four parallel branches concatenated on the channel axis (ref ``googlenet.py:46-181``)."""

    def __init__(self, input, n1x1=64, nr3x3=96, n3x3=128, nr5x5=16, n5x5=32, npj=32, lib_conv="native",
                 printinfo=False, input_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        C = self.input_shape[-1]
        mk = lambda inp, o, c, k, pad, std: Conv(input=inp, convstride=1, padsize=pad, W=Normal((o, k, k, c), mean=0.0, std=std),  # noqa: E731
                                                 b=Constant((o,), val=0.2), printinfo=False,
                                                 input_shape=None if isinstance(inp, Layer) else self.input_shape)
        self.conv_1x1 = mk(None, n1x1, C, 1, 0, 0.03)
        self.conv_r3x3 = mk(None, nr3x3, C, 1, 0, 0.09)
        self.conv_3x3 = mk(self.conv_r3x3, n3x3, nr3x3, 3, 1, 0.03)
        self.conv_r5x5 = mk(None, nr5x5, C, 1, 0, 0.2)
        self.conv_5x5 = mk(self.conv_r5x5, n5x5, nr5x5, 5, 2, 0.03)
        self.pool_3x3 = Pool(input=None, input_shape=self.input_shape, poolsize=3, poolstride=1, poolpad=1, mode="max", printinfo=False)
        self.conv_pj = mk(self.pool_3x3, npj, C, 1, 0, 0.1)
        self.branches = [self.conv_1x1, self.conv_r3x3, self.conv_3x3, self.conv_r5x5, self.conv_5x5, self.conv_pj]
        for l in self.branches:
            self.params += l.params
            self.weight_type += l.weight_type
        B, H, W_, _ = self.input_shape
        self.output_shape = (B, H, W_, n1x1 + n3x3 + n5x5 + npj)
        self.name = "Inception ( %s )" % lib_conv
        if printinfo:
            self.print_shape()

    def forward(self, x):
        # one autograd node for the whole module: branch outputs land in their channel slice of the concatenated tensor, the
        # four branches run on four streams, the four input gradients are merged by one kernel (ops/inception.py)
        from ..ops.inception import inception
        ps = []
        for l in (self.conv_1x1, self.conv_r3x3, self.conv_3x3, self.conv_r5x5, self.conv_5x5, self.conv_pj):
            ps += [l.W.val, l.b.val]
        return inception(x, tuple(ps))


class Aux_tower(Layer):
    """Auxiliary classifier: avg-pool 5/3 → 1×1 conv 128 → FC 1024 → Dropout 0.7 → Softmax
    (ref ``googlenet.py:183-273``)."""

    def __init__(self, input, n_softmax_out, lib_conv="native", printinfo=False, input_shape=None):
        super().__init__()
        self.get_input_shape(input, input_shape)
        C = self.input_shape[-1]
        self.pool = Pool(input=None, input_shape=self.input_shape, poolsize=5, poolstride=3, poolpad=0, mode="average", printinfo=False)
        self.conv1x1 = Conv(input=self.pool, convstride=1, padsize=0, W=Normal((128, 1, 1, C), mean=0.0, std=0.1),
                            b=Constant((128,), val=0.2), printinfo=False)
        self.flat = Flatten(input=self.conv1x1, axis=2, printinfo=False)
        self.fc = FC(input=self.flat, n_out=1024, W=Normal((1024, self.flat.output_shape[1]), mean=0, std=0.01),
                     b=Constant((1024,), val=0), printinfo=False)
        self.drp = Dropout(input=self.fc, n_out=1024, prob_drop=0.7, printinfo=False)
        self.softmax_layer = Softmax(input=self.drp, n_out=n_softmax_out, W=Normal((n_softmax_out, 1024), mean=0, std=0.01),
                                     b=Constant((n_softmax_out,), val=0), printinfo=False)
        self.chain = [self.pool, self.conv1x1, self.flat, self.fc, self.drp, self.softmax_layer]
        for l in self.chain:
            self.params += l.params
            self.weight_type += l.weight_type
        self.output_shape = self.softmax_layer.output_shape
        self.name = "AuxTower ( %s )" % lib_conv
        if printinfo:
            self.print_shape()

    def forward(self, x):
        for l in self.chain:
            x = l.forward(x)
        return x

    def negative_log_likelihood(self, y, label_smoothing=0.0, mix=None):
        return self.softmax_layer.negative_log_likelihood(y, label_smoothing, mix)


class GoogLeNet(ModelBase):
    supports_resized_crop = True
    supports_distill = True
    n_epochs, momentum, weight_decay = n_epochs, momentum, weight_decay
    batch_size, file_batch_size, learning_rate = batch_size, file_batch_size, learning_rate
    lr_policy = lr_policy
    use_momentum, use_nesterov_momentum = use_momentum, use_nesterov_momentum
    input_width, input_height = input_width, input_height
    batch_crop_mirror, rand_crop, monitor_grad = batch_crop_mirror, rand_crop, monitor_grad
    lr_power = 0.5

    def __init__(self, config):
        super().__init__(config)
        self.name = "GoogLeNet"
        for k in ("batch_size", "file_batch_size", "n_epochs"):
            if k in config:
                setattr(self, k, config[k])
        from .data.imagenet import ImageNet_data
        dk = dict(config.get("data_kwargs", {}))
        if "n_class" in config:
            dk.setdefault("n_class", config["n_class"])
        self.data = ImageNet_data(verbose=False, file_batch_size=self.file_batch_size, **dk)
        self.channels = self.data.channels
        self.n_softmax_out = config.get("n_class", self.data.n_class)
        self.setup_data_parallel(self.data)
        self.build_model()
        params, weight_types = get_params(self.layers)
        self.finalize(params, weight_types, (self.batch_size, self.input_height, self.input_width, self.channels))
        if self.data.para_load and not self.no_paraload:
            self.data.spawn_load()
            self.data.para_load_init(self.device, self.input_width, self.input_height, self.rand_crop,
                                     self.batch_crop_mirror, out_dtype=self.act_dtype,
                                     resized_crop=self.resized_crop, rank=self.rank,
                                     color_jitter=self.color_jitter, random_erasing=self.random_erasing,
                                     auto_augment=self.auto_augment, val_crops=self.val_crops)

    def build_model(self):
        v, B = self.verbose, self.batch_size
        if v:
            print(self.name)
        c1 = ConvPoolLRN(input=None, input_shape=(B, self.input_height, self.input_width, self.channels),
                         filter_shape=(self.channels, 7, 7, 64), convstride=2, padsize=3, group=1, poolsize=3, poolstride=2,
                         poolpad=1, b=0.2, W=Normal((64, 7, 7, self.channels), mean=0.0, std=0.1), lrn=True, printinfo=v)
        r3 = Conv(input=c1, convstride=1, padsize=0, W=Normal((64, 1, 1, 64), mean=0.0, std=0.1), b=Constant((64,), val=0.2), printinfo=v)
        c3 = ConvPoolLRN(input=r3, filter_shape=(64, 3, 3, 192), convstride=1, padsize=1, group=1, poolsize=3, poolstride=2,
                         poolpad=1, b=0.2, W=Normal((192, 3, 3, 64), mean=0.0, std=0.03), lrn=True, printinfo=v)
        i3a = Incept(c3, 64, 96, 128, 16, 32, 32, printinfo=v)
        i3b = Incept(i3a, 128, 128, 192, 32, 96, 64, printinfo=v)
        p3 = Pool(input=i3b, poolsize=3, poolstride=2, poolpad=1, mode="max", printinfo=v)
        i4a = Incept(p3, 192, 96, 208, 16, 48, 64, printinfo=v)
        i4b = Incept(i4a, 160, 112, 224, 24, 64, 64, printinfo=v)
        i4c = Incept(i4b, 128, 128, 256, 24, 64, 64, printinfo=v)
        i4d = Incept(i4c, 112, 144, 288, 32, 64, 64, printinfo=v)
        i4e = Incept(i4d, 256, 160, 320, 32, 128, 128, printinfo=v)
        lrn4 = LRN(input=i4e, printinfo=v)
        p4 = Pool(input=lrn4, poolsize=3, poolstride=2, poolpad=1, mode="max", printinfo=v)
        i5a = Incept(p4, 256, 160, 320, 32, 128, 128, printinfo=v)
        i5b = Incept(i5a, 384, 192, 384, 48, 128, 128, printinfo=v)
        px = Pool(input=i5b, poolsize=7, poolstride=1, poolpad=0, mode="average", printinfo=v)
        fl = Flatten(input=px, axis=2, printinfo=v)
        dr = Dropout(input=fl, n_out=fl.output_shape[1], prob_drop=0.4, printinfo=v)
        sm = Softmax(input=dr, n_out=self.n_softmax_out, W=Normal((self.n_softmax_out, fl.output_shape[1]), mean=0.0, std=0.01),
                     b=Constant((self.n_softmax_out,), val=0), printinfo=v)
        self.aux1 = Aux_tower(input=i4a, n_softmax_out=self.n_softmax_out, printinfo=v)
        self.aux2 = Aux_tower(input=i4d, n_softmax_out=self.n_softmax_out, printinfo=v)
        self.trunk = [c1, r3, c3, i3a, i3b, p3, i4a, i4b, i4c, i4d, i4e, lrn4, p4, i5a, i5b, px, fl, dr, sm]
        self._tap1, self._tap2 = i4a, i4d
        self.output_layer = sm
        self.layers = self.trunk + [self.aux1, self.aux2]

    def forward(self, x):
        taps = {}
        for l in self.trunk:
            x = l.forward(x)
            if l is self._tap1 or l is self._tap2:
                taps[id(l)] = x
        self._taps = taps
        return x

    def loss(self, x, y, label_smoothing=0.0, mix=None, kd=None):
        # config['distill'] (kd): only the main head distils; the auxiliary towers keep their hard loss
        self.forward(x)
        sm = self.output_layer
        cost = sm.negative_log_likelihood(y, label_smoothing, mix, kd)
        if Dropout.layers and Dropout.layers[0].flag_on:          # aux towers only contribute while training
            self.aux1.forward(self._taps[id(self._tap1)])
            self.aux2.forward(self._taps[id(self._tap2)])
            cost = (cost + 0.3 * self.aux1.negative_log_likelihood(y, label_smoothing, mix)
                    + 0.3 * self.aux2.negative_log_likelihood(y, label_smoothing, mix))
        return cost, sm.errors(y), sm.errors_top_x(y)
