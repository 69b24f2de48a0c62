"""AlexNet (ref ``theanompi/models/alex_net.py``).

Architecture and hyper-parameters as the reference: five ``ConvPoolLRN`` blocks
(11×11/4 3→96 +LRN+pool; 5×5 p2 96→256 g2 +LRN+pool; 3×3 256→384; 3×3 384→384 g2;
3×3 384→256 g2 +pool) → FC 9216→4096 → Dropout → FC 4096→4096 → Dropout → Softmax
1000 (``alex_net.py:186-290``); lr 0.01 ÷10 at epochs {20,40,60}, 70 epochs, μ = 0.9,
weight decay 5e-4, batch = file batch = 128 (``:10-41``).  22 parameter tensors /
60,965,224 weights.

Input is NHWC ``(128, 227, 227, 3)`` bf16 produced on the device by the loader's fused
normalise/crop/mirror kernel; every block is one or two fused sm_90a kernels.
"""
from __future__ import annotations

from .base import ModelBase
from .layers2 import (FC, Constant, ConvPoolLRN, Dropout, Flatten, Normal, Softmax,
                      get_layers, get_params, forward_chain)

# model hyperparams (module-level like the reference, ``alex_net.py:10-41``)
n_epochs = 70
momentum = 0.90
weight_decay = 0.0005
batch_size = 128
file_batch_size = 128
learning_rate = 0.01
lr_policy = "step"
lr_step = [20, 40, 60]
use_momentum = True
use_nesterov_momentum = False
input_width = 227
input_height = 227
batch_crop_mirror = False
rand_crop = True
image_mean = "img_mean"
dataname = "imagenet"
lib_conv = "native"
monitor_grad = False
seed_weight_on_pid = False


class AlexNet(ModelBase):
    supports_resized_crop = True
    supports_distill = True
    n_epochs, momentum, weight_decay = n_epochs, momentum, weight_decay
    batch_size, file_batch_size, learning_rate = batch_size, file_batch_size, learning_rate
    lr_policy, lr_step = lr_policy, lr_step
    use_momentum, use_nesterov_momentum = use_momentum, use_nesterov_momentum
    input_width, input_height = input_width, input_height
    batch_crop_mirror, rand_crop, monitor_grad = batch_crop_mirror, rand_crop, monitor_grad

    def __init__(self, config):
        super().__init__(config)
        self.name = "AlexNet"
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

        if seed_weight_on_pid:
            import os
            from . import layers2
            layers2.reseed(os.getpid())
        self.build_model()
        self.layers = get_layers(lastlayer=self.output_layer)
        params, weight_types = get_params(self.layers)
        self.finalize(params, weight_types,
                      (self.batch_size, self.input_height, self.input_width, self.channels))

        if self.data.para_load and not self.no_paraload:
            self.data.spawn_load()
            self.data.para_load_init(self.device, self.input_width, self.input_height,
                                     self.rand_crop, self.batch_crop_mirror, out_dtype=self.act_dtype,
                                     resized_crop=self.resized_crop, rank=self.rank,
                                     color_jitter=self.color_jitter, random_erasing=self.random_erasing,
                                     auto_augment=self.auto_augment, val_crops=self.val_crops)

    def build_model(self):
        if self.verbose:
            print(self.name)
        v = self.verbose
        B = self.batch_size
        c1 = ConvPoolLRN(input=None, input_shape=(B, self.input_height, self.input_width, self.channels),
                         filter_shape=(3, 11, 11, 96), convstride=4, padsize=0, group=1,
                         poolsize=3, poolstride=2, b=0.0, lrn=True, lib_conv=lib_conv, printinfo=v)
        c2 = ConvPoolLRN(input=c1, filter_shape=(96, 5, 5, 256), convstride=1, padsize=2, group=2,
                         poolsize=3, poolstride=2, b=0.1, lrn=True, lib_conv=lib_conv, printinfo=v)
        c3 = ConvPoolLRN(input=c2, filter_shape=(256, 3, 3, 384), convstride=1, padsize=1, group=1,
                         poolsize=1, poolstride=0, b=0.0, lrn=False, lib_conv=lib_conv, printinfo=v)
        c4 = ConvPoolLRN(input=c3, filter_shape=(384, 3, 3, 384), convstride=1, padsize=1, group=2,
                         poolsize=1, poolstride=0, b=0.1, lrn=False, lib_conv=lib_conv, printinfo=v)
        c5 = ConvPoolLRN(input=c4, filter_shape=(384, 3, 3, 256), convstride=1, padsize=1, group=2,
                         poolsize=3, poolstride=2, b=0.0, lrn=False, lib_conv=lib_conv, printinfo=v)
        flat = Flatten(input=c5, axis=2, printinfo=v)
        n_in = flat.output_shape[1]
        fc6 = FC(input=flat, n_out=4096, W=Normal((4096, n_in), std=0.005),
                 b=Constant((4096,), val=0.1), printinfo=v)
        d6 = Dropout(input=fc6, n_out=4096, prob_drop=0.5, printinfo=v)
        fc7 = FC(input=d6, n_out=4096, W=Normal((4096, 4096), std=0.005),
                 b=Constant((4096,), val=0.1), printinfo=v)
        d7 = Dropout(input=fc7, n_out=4096, prob_drop=0.5, printinfo=v)
        sm8 = Softmax(input=d7, n_out=self.n_softmax_out,
                      W=Normal((self.n_softmax_out, 4096), mean=0, std=0.01),
                      b=Constant((self.n_softmax_out,), val=0), printinfo=v)
        self.output_layer = sm8

    def forward(self, x):
        return forward_chain(self.layers, x)


if __name__ == "__main__":
    raise RuntimeError("to be tested using test_model.py:\n$ python -m theanompi_b200.models.test_model "
                       "theanompi_b200.models.alex_net AlexNet")
