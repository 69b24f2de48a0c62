"""ResNet-50 (ref ``theanompi/models/lasagne_model_zoo/resnet50.py``): bottleneck blocks
[3,4,6,3], the last BatchNorm gamma of every residual branch initialised to 0 (``:62-65``),
batch 32 (the published table uses 64), lr 0.1·b/256, μ 0.9, wd 1e-4, momentum-SGD through
the framework's ``pre_model_iter_fn`` path.  BN gamma/beta are updated locally and never
exchanged (``opt.py:207-226``, ``exchanger.py:35-43``).

``ResNet50`` runs entirely on the hand-written sm_90a kernels: every convolution is the wgmma implicit-GEMM kernel
(bias-free, linear), every ``batch_norm (+ shortcut) + rectify`` is one fused BatchNormal forward / backward pair
(``csrc/bn_kernels.cu``), the step is CUDA-graph captured.  ``ResNet50Torch`` is the same network on torch modules
(cuDNN / cuBLAS) — kept as the library yardstick and as the numerical reference of the tests."""
from __future__ import annotations

import torch.nn as nn

from ..base import ModelBase
from ..layers2 import BatchNormal, Conv, Flatten, HeNormal, Normal, Constant, Pool, Softmax, get_params
from ..torch_base import TorchModelBase

n_epochs = 90
momentum = 0.9
weight_decay = 1e-4
batch_size = 32
file_batch_size = 128
learning_rate = 0.1 * batch_size / 256.0
lr_policy = "step"
lr_step = [30, 60, 80]
input_width = input_height = 224


class Bottleneck(nn.Module):
    def __init__(self, cin, mid, stride):
        super().__init__()
        cout = mid * 4
        self.a = nn.Sequential(nn.Conv2d(cin, mid, 1, bias=False), nn.BatchNorm2d(mid), nn.ReLU(inplace=True),
                               nn.Conv2d(mid, mid, 3, stride, 1, bias=False), nn.BatchNorm2d(mid), nn.ReLU(inplace=True),
                               nn.Conv2d(mid, cout, 1, bias=False), nn.BatchNorm2d(cout))
        nn.init.zeros_(self.a[-1].weight)                  # 2c branch gamma = 0 (ref :62-65)
        self.proj = None
        if stride != 1 or cin != cout:
            self.proj = nn.Sequential(nn.Conv2d(cin, cout, 1, stride, bias=False), nn.BatchNorm2d(cout))
        self.relu = nn.ReLU(inplace=True)

    def forward(self, x):
        return self.relu(self.a(x) + (x if self.proj is None else self.proj(x)))


class ResNet50Net(nn.Module):
    def __init__(self, n_class=1000, blocks=(3, 4, 6, 3)):
        super().__init__()
        self.stem = nn.Sequential(nn.Conv2d(3, 64, 7, 2, 3, bias=False), nn.BatchNorm2d(64), nn.ReLU(inplace=True),
                                  nn.MaxPool2d(3, 2, 1))
        layers, cin = [], 64
        for i, n in enumerate(blocks):
            mid = 64 * 2 ** i
            for j in range(n):
                layers.append(Bottleneck(cin, mid, 2 if (j == 0 and i > 0) else 1))
                cin = mid * 4
        self.body = nn.Sequential(*layers)
        self.head = nn.Linear(cin, n_class)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out", nonlinearity="relu")

    def forward(self, x):
        return self.head(self.body(self.stem(x)).mean((2, 3)))


class ResNet50(ModelBase):
    supports_drop_path = True      # one drop-path block per bottleneck
    supports_resized_crop = True
    supports_distill = True
    n_epochs, momentum, weight_decay = n_epochs, momentum, weight_decay
    batch_size, file_batch_size, learning_rate = batch_size, file_batch_size, learning_rate
    lr_policy, lr_step = lr_policy, lr_step
    input_width, input_height = input_width, input_height
    blocks = (3, 4, 6, 3)

    def __init__(self, config):
        super().__init__(config)
        self.name = "ResNet50"
        for k in ("batch_size", "file_batch_size", "n_epochs"):
            if k in config:
                setattr(self, k, config[k])
        from ..data.imagenet import ImageNet_data
        from .. import layers2
        dk = dict(config.get("data_kwargs", {}))
        if "n_class" in config:
            dk.setdefault("n_class", config["n_class"])
        self.data = ImageNet_data(verbose=False, file_batch_size=self.file_batch_size, **dk)
        self.channels = self.data.channels
        self.n_softmax_out = config.get("n_class", self.data.n_class)
        self.setup_data_parallel(self.data)
        layers2.reseed()
        self.blocks = tuple(config.get("blocks", self.blocks))
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

    # ---- construction: every conv is bias-free and linear; BatchNormal carries the ReLU (and the shortcut add)
    def _conv(self, inp, cout, k, stride, pad, input_shape=None):
        cin = (inp.output_shape if inp is not None else input_shape)[-1]
        c = Conv(inp, stride, pad, W=HeNormal((cout, k, k, cin)), b=False, relu=False, printinfo=False, input_shape=input_shape)
        self.layers.append(c)
        return c

    def _bn(self, inp, relu, gamma=1.0):
        b = BatchNormal(inp, relu=relu, gamma=gamma, printinfo=False)
        self.layers.append(b)
        return b

    def build_model(self):
        B = self.batch_size
        self.layers = []
        c = self._conv(None, 64, 7, 2, 3, input_shape=(B, self.input_height, self.input_width, self.channels))
        b = self._bn(c, True)
        pool = Pool(b, 3, 2, 1, "max", printinfo=False)
        self.layers.append(pool)
        self.stem = (c, b, pool)
        self.body = []
        cur = pool
        for i, n in enumerate(self.blocks):
            mid = 64 * 2 ** i
            for j in range(n):
                stride = 2 if (j == 0 and i > 0) else 1
                cin, cout = cur.output_shape[-1], mid * 4
                c1 = self._conv(cur, mid, 1, 1, 0); b1 = self._bn(c1, True)
                c2 = self._conv(b1, mid, 3, stride, 1); b2 = self._bn(c2, True)
                c3 = self._conv(b2, cout, 1, 1, 0)
                proj = None
                if stride != 1 or cin != cout:
                    pc = self._conv(cur, cout, 1, stride, 0)
                    proj = (pc, self._bn(pc, False))
                b3 = self._bn(c3, True, gamma=0.0)               # 2c branch gamma = 0 (ref :62-65); ReLU after the shortcut add
                self.body.append((c1, b1, c2, b2, c3, b3, proj))
                cur = b3
        gap = Pool(cur, cur.output_shape[1], 1, 0, "avg", printinfo=False)
        flat = Flatten(gap, axis=2, printinfo=False)
        n_in = flat.output_shape[1]
        sm = Softmax(flat, self.n_softmax_out, W=Normal((self.n_softmax_out, n_in), std=0.01), b=Constant((self.n_softmax_out,), 0.0),
                     printinfo=False)
        self.layers += [gap, flat, sm]
        self.head = (gap, flat, sm)
        self.output_layer = sm

    def forward(self, x):
        c, b, pool = self.stem
        x = pool.forward(b.forward(c.forward(x)))
        from ... import ops
        for l, (c1, b1, c2, b2, c3, b3, proj) in enumerate(self.body):
            x, xs = ops.fork2(x)                                  # two consumers: the branch and the shortcut
            short = xs if proj is None else proj[1].forward(proj[0].forward(xs))
            y = b1.forward(c1.forward(x))
            y = b2.forward(c2.forward(y))
            # relu(s·bn(conv) + shortcut) in one kernel; s is block l's drop-path row (None: no drop)
            x = b3.forward(c3.forward(y), residual=short, drop=self.drop_row(l))
        gap, flat, sm = self.head
        return sm.forward(flat.forward(gap.forward(x)))


class ResNet50Torch(TorchModelBase):
    supports_resized_crop = True   # the same ImageNet loader as ResNet50
    n_epochs, momentum, weight_decay = n_epochs, momentum, weight_decay
    batch_size, file_batch_size, learning_rate = batch_size, file_batch_size, learning_rate
    lr_policy, lr_step = lr_policy, lr_step
    input_width, input_height = input_width, input_height
    blocks = (3, 4, 6, 3)

    def __init__(self, config):
        super().__init__(config)
        self.name = "ResNet50Torch"
        for k in ("batch_size", "file_batch_size", "n_epochs"):
            if k in config:
                setattr(self, k, config[k])
        import torch
        torch.manual_seed(23455)
        from ..data.imagenet import ImageNet_data
        dk = dict(config.get("data_kwargs", {}))
        if "n_class" in config:
            dk.setdefault("n_class", config["n_class"])
        self.data = ImageNet_data(verbose=False, file_batch_size=self.file_batch_size, **dk)
        self.channels = self.data.channels
        self.setup_data_parallel(self.data)
        net = ResNet50Net(config.get("n_class", self.data.n_class), config.get("blocks", self.blocks))
        self.finalize_torch(net, (self.batch_size, self.input_height, self.input_width, self.channels))
        if self.data.para_load and not self.no_paraload:
            self.data.spawn_load()
            self.data.para_load_init(self.device, self.input_width, self.input_height, self.rand_crop,
                                     self.batch_crop_mirror, out_dtype=self.act_dtype,
                                     resized_crop=self.resized_crop, rank=self.rank,
                                     color_jitter=self.color_jitter, random_erasing=self.random_erasing,
                                     auto_augment=self.auto_augment, val_crops=self.val_crops)
