"""Cifar10 CNN (ref ``theanompi/models/cifar10.py:120-252``): Subtract → Crop(28×28,
mirror) → Conv5×5(64) → Pool2 → Conv5×5(128) → Pool2 → Conv3×3(64) → FC256 → Dropout →
Softmax10; batch 256, lr 0.01 ÷10 at {50,60,65}, μ 0.9, wd 1e-4 (``cifar10.py:5-29``).
The model the EASGD / GOSGD examples train."""
from __future__ import annotations

from .. import ops
from .base import ModelBase
from .layers2 import (FC, Constant, Conv, Crop, Dropout, Flatten, Normal, Pool, Softmax, Subtract,
                      forward_chain, get_layers, get_params)

n_epochs = 70
momentum = 0.90
weight_decay = 0.0001
file_batch_size = 256
batch_size = 256
learning_rate = 0.01
lr_policy = "step"
lr_step = [50, 60, 65]
use_momentum = True
use_nesterov_momentum = False
input_width = 28
input_height = 28
batch_crop_mirror = True
rand_crop = True
monitor_grad = False


class Cifar10_model(ModelBase):
    graph_safe = False            # the in-graph Crop layer draws offsets / mirrors from the host RNG every step
    supports_sam = False          # that Crop draws at every forward: a second forward of the step would see another crop
    n_epochs, momentum, weight_decay = n_epochs, momentum, weight_decay
    batch_size, file_batch_size, learning_rate = batch_size, file_batch_size, learning_rate
    lr_policy, lr_step = lr_policy, lr_step
    use_momentum, use_nesterov_momentum = use_momentum, use_nesterov_momentum
    input_width, input_height = input_width, input_height
    batch_crop_mirror, rand_crop, monitor_grad = batch_crop_mirror, rand_crop, monitor_grad

    def __init__(self, config):
        super().__init__(config)
        self.name = "Cifar10_model"
        for k in ("batch_size", "file_batch_size", "n_epochs", "learning_rate"):
            if k in config:
                setattr(self, k, config[k])
        self.base_lr = self.learning_rate
        from .data.cifar10 import Cifar10_data
        self.data = Cifar10_data(verbose=False, **config.get("data_kwargs", {}))
        self.channels = self.data.channels
        self.n_softmax_out = self.data.n_class
        self.setup_data_parallel(self.data)
        self.build_model()
        self.layers = get_layers(lastlayer=self.output_layer)
        params, weight_types = get_params(self.layers)
        self.finalize(params, weight_types, (self.batch_size, self.data.height, self.data.width, self.channels))

    def build_model(self):
        v, B, C = self.verbose, self.batch_size, self.channels
        sub = Subtract(input=None, input_shape=(B, self.data.height, self.data.width, C),
                       subtract_arr=self.data.rawdata[4], printinfo=v)
        crop = self.crop = Crop(input=sub, output_shape=(B, self.input_height, self.input_width, C),
                                flag_batch=self.batch_crop_mirror, printinfo=v)
        c1 = Conv(input=crop, convstride=1, padsize=0, W=Normal((64, 5, 5, C), std=0.05), b=Constant((64,), val=0), printinfo=v)
        p1 = Pool(input=c1, poolsize=2, poolstride=2, poolpad=0, mode="max", printinfo=v)
        c2 = Conv(input=p1, convstride=1, padsize=0, W=Normal((128, 5, 5, 64), std=0.05), b=Constant((128,), val=0), printinfo=v)
        p2 = Pool(input=c2, poolsize=2, poolstride=2, poolpad=0, mode="max", printinfo=v)
        c3 = Conv(input=p2, convstride=1, padsize=0, W=Normal((64, 3, 3, 128), std=0.05), b=Constant((64,), val=0), printinfo=v)
        flat = Flatten(input=c3, axis=2, printinfo=v)
        fc = FC(input=flat, n_out=256, W=Normal((256, flat.output_shape[1]), std=0.001), b=Constant((256,), val=0), printinfo=v)
        drop = Dropout(input=fc, n_out=256, prob_drop=0.5, printinfo=v)
        sm = Softmax(input=drop, n_out=self.n_softmax_out, W=Normal((self.n_softmax_out, 256), std=0.005),
                     b=Constant((self.n_softmax_out,), val=0), printinfo=v)
        self.output_layer = sm

    def forward(self, x):
        rec, self._mix_rec = getattr(self, "_mix_rec", None), None
        if rec is None:
            return forward_chain(self.layers, x)
        k = self.layers.index(self.crop) + 1
        return forward_chain(self.layers[k:], ops.mix_batch(forward_chain(self.layers[:k], x), rec))

    # Mixup / CutMix mix the output of the in-graph Crop, the tensor that enters the first convolution: the CutMix box and λ refer
    # to the 28×28 crop
    @property
    def mix_hw(self):
        return (self.input_height, self.input_width)

    def mix_input(self, rec):
        self._mix_rec = rec                      # taken by the forward that follows
