"""LSGAN on CIFAR-10 (ref ``lasagne_model_zoo/lsgan_cifar10.py``) — the model of the "GAP"
swap session (``examples/bsp/session_gap.cfg``): 32×32×3 images, same contract."""
import numpy as np

from .wgan import WGAN, NativeWGAN


class _CifarIter(object):
    def __init__(self, data, batch_size):
        self.data, self.batch_size = data, batch_size
        self.n_batch_train = self.n_batch_val = 1

    def iterate(self, mode="train", shuffle=True, seed=None, forever=True):
        x = self.data.rawdata[0] if mode == "train" else self.data.rawdata[2]
        y = self.data.rawdata[1] if mode == "train" else self.data.rawdata[3]
        rs = np.random.RandomState(seed)
        B = self.batch_size
        while True:
            idx = rs.permutation(len(x)) if shuffle else np.arange(len(x))
            if len(idx) < B:                        # tiny (synthetic / test) sets: tile up to one batch
                idx = np.resize(idx, B)
            for s in range(0, len(idx) - B + 1, B):
                sel = idx[s:s + B]
                yield x[sel] / 255.0, y[sel]


class LSGAN(WGAN):
    loss_kind = "lsgan"
    learning_rate = 1e-4
    image_size, image_ch = 32, 3

    def make_data(self, config):
        from ..data.cifar10 import Cifar10_data
        return _CifarIter(Cifar10_data(verbose=False, **config.get("data_kwargs", {})), self.batch_size)


class NativeLSGAN(NativeWGAN):
    """:class:`LSGAN` (CIFAR-10) on the native kernels (see :class:`NativeWGAN`)."""
    loss_kind = "lsgan"
    learning_rate = 1e-4
    image_size, image_ch = 32, 3
    make_data = LSGAN.make_data
