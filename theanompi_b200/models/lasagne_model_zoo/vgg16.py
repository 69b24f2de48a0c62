"""VGG16 (ref ``theanompi/models/lasagne_model_zoo/vgg16.py:13-67,103-128``): thirteen 3×3
pad-1 convolutions (64,64 | 128,128 | 256×3 | 512×3 | 512×3) with 2×2 max-pools, FC
25088→4096→4096→1000 with dropout; batch 32 from 128-image files, lr 0.002, μ 0.9,
wd 5e-4.  32 parameter tensors / 138,357,544 weights (527.8 MiB exchanged per iteration —
the reference's most communication-bound model, ``README.md:116-117``).

The reference builds it from Lasagne layers; here it uses the framework's own fused layers
(the directory name is kept for import-path parity)."""
from __future__ import annotations

from ..base import ModelBase
from ..layers2 import FC, Constant, Conv, Dropout, Flatten, HeNormal, Normal, Pool, Softmax, forward_chain, get_layers, get_params

n_epochs = 70
momentum = 0.90
weight_decay = 0.0005
batch_size = 32
file_batch_size = 128
learning_rate = 0.002
lr_policy = "step"
lr_step = [20, 40, 60]
use_momentum = True
use_nesterov_momentum = False
input_width = 224
input_height = 224
batch_crop_mirror = False
rand_crop = True

CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512, "M"]


class VGG16(ModelBase):
    supports_resized_crop = True
    supports_distill = True
    n_epochs, momentum, weight_decay = n_epochs, momentum, weight_decay
    batch_size, file_batch_size, learning_rate = batch_size, file_batch_size, learning_rate
    lr_policy, lr_step = lr_policy, lr_step
    use_momentum, use_nesterov_momentum = use_momentum, use_nesterov_momentum
    input_width, input_height = input_width, input_height
    batch_crop_mirror, rand_crop = batch_crop_mirror, rand_crop

    def __init__(self, config):
        super().__init__(config)
        self.name = "VGG16"
        for k in ("batch_size", "file_batch_size", "n_epochs"):
            if k in config:
                setattr(self, k, config[k])
        from ..data.imagenet import ImageNet_data
        dk = dict(config.get("data_kwargs", {}))
        if "n_class" in config:
            dk.setdefault("n_class", config["n_class"])
        self.data = ImageNet_data(verbose=False, file_batch_size=self.file_batch_size, **dk)
        self.channels = self.data.channels
        self.n_softmax_out = config.get("n_class", self.data.n_class)
        self.setup_data_parallel(self.data)
        self.build_model()
        self.layers = get_layers(lastlayer=self.output_layer)
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
        prev, cin, first = None, self.channels, True
        for item in CFG:
            if item == "M":
                prev = Pool(input=prev, poolsize=2, poolstride=2, poolpad=0, mode="max", printinfo=v)
            else:
                kw = dict(input_shape=(B, self.input_height, self.input_width, cin)) if first else {}
                prev = Conv(input=prev, convstride=1, padsize=1, W=HeNormal((item, 3, 3, cin)), b=Constant((item,), val=0.0),
                            printinfo=v, **kw)
                cin, first = item, False
        flat = Flatten(input=prev, axis=2, printinfo=v)
        fc6 = FC(input=flat, n_out=4096, W=Normal((4096, flat.output_shape[1]), std=0.005), b=Constant((4096,), val=0.1), printinfo=v)
        d6 = Dropout(input=fc6, n_out=4096, prob_drop=0.5, printinfo=v)
        fc7 = FC(input=d6, n_out=4096, W=Normal((4096, 4096), std=0.005), b=Constant((4096,), val=0.1), printinfo=v)
        d7 = Dropout(input=fc7, n_out=4096, prob_drop=0.5, printinfo=v)
        self.output_layer = Softmax(input=d7, n_out=self.n_softmax_out, W=Normal((self.n_softmax_out, 4096), std=0.01),
                                    b=Constant((self.n_softmax_out,), val=0), printinfo=v)

    def forward(self, x):
        return forward_chain(self.layers, x)

    def save(self, path):
        from ...utils.helper_funcs import save_weights
        save_weights(self.layers, path, self.epoch)

    def load(self, path, epoch):
        """Load pretrained / snapshot weights (the reference loads a Lasagne pkl, ``vgg16.py:560-572``)."""
        from ...utils.helper_funcs import load_weights
        load_weights(self.layers, path, epoch)
        self.arena.refresh_shadow()
