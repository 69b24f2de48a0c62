"""Functional op surface of the framework.

GPU: hand-written sm_90a kernels (``csrc/``) — wgmma/TMA GEMM with fused
bias/ReLU epilogues for FC and conv (implicit-GEMM via an NHWC im2col gather),
fused LRN / pool / dropout / softmax-xent / crop-mirror-normalise and the flat-arena
optimizer + collective kernels.  CPU: plain-torch reference (``reference.py``).
"""
from . import accum, cifar_augment, drop_path, mixup, native, reference
from .functional import (add, advance_rng_step, batch_norm, compute_weight, conv2d_bias_act,
                         conv2d_group2_bias_act, crop_mirror_normalize, dropout, fork2,
                         linear_bias_act, lrn, mix_batch, mix_draw, pool2d, random_erase, resized_crop_mirror_normalize,
                         rng_state, seed_dropout, softmax_xent, softmax_xent_kd)

__all__ = [
    "accum", "cifar_augment", "drop_path", "mixup", "native", "reference", "conv2d_bias_act", "conv2d_group2_bias_act", "linear_bias_act",
    "pool2d", "lrn", "dropout", "softmax_xent", "softmax_xent_kd", "crop_mirror_normalize", "resized_crop_mirror_normalize", "compute_weight",
    "seed_dropout", "advance_rng_step", "rng_state", "batch_norm", "add", "fork2", "mix_draw", "mix_batch", "random_erase",
]
