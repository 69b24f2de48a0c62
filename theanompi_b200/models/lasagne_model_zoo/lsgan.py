"""Least-squares GAN on MNIST (ref ``lasagne_model_zoo/lsgan.py``): same generator / critic
and contract as :class:`WGAN`, least-squares losses, one critic step per generator step,
no weight clipping."""
from .wgan import WGAN, NativeWGAN


class LSGAN(WGAN):
    loss_kind = "lsgan"
    learning_rate = 1e-4


class NativeLSGAN(NativeWGAN):
    """:class:`LSGAN` on the native kernels (see :class:`NativeWGAN`)."""
    loss_kind = "lsgan"
    learning_rate = 1e-4
