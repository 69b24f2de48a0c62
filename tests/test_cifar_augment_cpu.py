"""CIFAR augmentation (config['cifar_augment']) on the CPU path: the validation of the key and the models that refuse it, the
statistics and independence of the reference draw, the reference zero-filled crop, flip and Cutout against torchvision's pad / crop /
horizontal_flip and DeVries & Taylor's mask, and a tiny Wide_ResNet that trains with it, feeds its stem the reference-augmented batch
and validates exactly as a model without the key."""
import os
import sys

import numpy as np
import pytest
import torch
from scipy import stats

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import cifar_augment as ca  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402

IMG = dict(no_paraload=True, n_class=8, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))


def _reseed():
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)


def _wrn(**kw):
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    _reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=8, file_batch_size=16, depth=10, widen=1,
               data_kwargs=dict(n_synthetic=256, synthetic=True))
    cfg.update(kw)
    return Wide_ResNet(cfg)


# --------------------------------------------------------------------------- configuration
@pytest.mark.parametrize("bad,key", [([4], None), ("pad", None), (dict(crop=4), "crop"), (dict(pad=True), "pad"), (dict(pad=4.0), "pad"),
                                     (dict(pad=-1), "pad"), (dict(pad=32), "pad"), (dict(cutout=33), "cutout"),
                                     (dict(cutout=-1), "cutout"), (dict(cutout=16.0), "cutout"), (dict(cutout=False), "cutout"),
                                     (dict(seed=1.5), "seed"), (dict(seed="1"), "seed"), (dict(seed=True), "seed")])
def test_malformed_values_name_the_key(bad, key):
    with pytest.raises(ValueError, match="cifar_augment") as e:
        ca.check_config(bad)
    if key is not None:
        assert repr(key) in str(e.value)
    m = _wrn(cifar_augment=bad)
    with pytest.raises(ValueError, match="cifar_augment"):
        m.compile_iter_fns("avg")


def test_defaults_are_filled_in():
    assert ca.check_config(None) is None
    assert ca.check_config({}) == dict(pad=4, cutout=0, seed=0)
    assert ca.check_config(dict(cutout=16, seed=-1)) == dict(pad=4, cutout=16, seed=2 ** 64 - 1)
    assert ca.check_config(dict(pad=np.int64(0), cutout=32)) == dict(pad=0, cutout=32, seed=0)
    m = _wrn()
    m.compile_iter_fns("avg")
    assert m.cifar_aug is None and m.train_augment() is None
    m = _wrn(cifar_augment=dict(cutout=16))
    m.compile_iter_fns("avg")
    aug = m.cifar_aug
    assert aug.cfg == dict(pad=4, cutout=16, seed=0) and aug.B == 8
    assert (aug.offs.dtype, tuple(aug.offs.shape)) == (torch.int32, (8, 2))
    assert (aug.flips.dtype, tuple(aug.flips.shape)) == (torch.uint8, (8,))
    assert (aug.boxes.dtype, tuple(aug.boxes.shape)) == (torch.int32, (8, 4))
    assert m.train_augment() is None                                # only the training forward reads the draw


def _refused():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNetTorch
    from theanompi_b200.models.lasagne_model_zoo.lsgan import LSGAN, NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50, ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    img = dict(batch_size=4, file_batch_size=4, **IMG)
    return [(AlexNet, img), (GoogLeNet, img), (ResNet50, dict(img, blocks=(1, 1, 1, 1))),
            (Cifar10_model, dict(batch_size=4, file_batch_size=8, data_kwargs=dict(n_synthetic=64, synthetic=True))),
            (NativeWGAN, dict(data_kwargs=dict(n_synthetic=128))), (NativeLSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (WGAN, dict(data_kwargs=dict(n_synthetic=128))), (LSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (LSTM, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (LSTMTorch, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (ResNet50Torch, dict(img, blocks=(1, 1, 1, 1))),
            (Wide_ResNetTorch, dict(batch_size=8, file_batch_size=8, depth=10, widen=1, data_kwargs=dict(n_synthetic=64, synthetic=True)))]


def test_every_other_model_refuses_it():
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    assert Wide_ResNet.supports_cifar_augment is True and VGG16.supports_cifar_augment is False
    for cls, kw in _refused():
        assert cls.supports_cifar_augment is False, cls
        _reseed()
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", cifar_augment={}, **kw))
        with pytest.raises(ValueError, match="cifar_augment is not supported.*Wide_ResNet"):
            m.compile_iter_fns("avg")


# --------------------------------------------------------------------------- the reference draw
def _draws(cfg, steps, B=512, seed=0, rank=0):
    outs = [ref.cifar_augment_draw(cfg, seed, rank, s, B) for s in steps]
    return [torch.cat(t).numpy() for t in zip(*outs)]


def _chi2_uniform(v, k):
    counts = np.bincount(np.asarray(v).reshape(-1), minlength=k)
    assert counts.shape[0] == k
    return stats.chisquare(counts).pvalue


@pytest.mark.parametrize("pad", [1, 4, 31])
def test_offsets_centres_and_flips_are_uniform(pad):
    cfg = ca.check_config(dict(pad=pad, cutout=1, seed=77))        # L = 1: the box is the empty hole at (cy, cx), read back below
    offs, flips, boxes = _draws(cfg, range(40))
    assert offs.min() >= -pad and offs.max() <= pad
    assert _chi2_uniform(offs[:, 0] + pad, 2 * pad + 1) > 1e-4 and _chi2_uniform(offs[:, 1] + pad, 2 * pad + 1) > 1e-4
    assert _chi2_uniform(boxes[:, 0], 32) > 1e-4 and _chi2_uniform(boxes[:, 1], 32) > 1e-4
    assert (boxes[:, 2:] == 0).all()
    n = flips.shape[0]
    assert set(np.unique(flips)) <= {0, 1}
    assert stats.binomtest(int(flips.sum()), n, 0.5).pvalue > 1e-4
    # the five values of an image are not correlated with each other
    v = np.stack([offs[:, 0], offs[:, 1], flips, boxes[:, 0], boxes[:, 1]]).astype(np.float64)
    c = np.corrcoef(v)
    assert np.abs(c - np.eye(5)).max() < 4.5 / np.sqrt(n)


def test_pad_zero_never_shifts():
    offs, flips, _ = _draws(ca.check_config(dict(pad=0)), range(4))
    assert (offs == 0).all() and 0 < flips.mean() < 1


def test_ranks_seeds_and_steps_give_different_streams():
    cfg = ca.check_config(dict(cutout=16, seed=5))
    base = ref.cifar_augment_draw(cfg, 5, 0, 3, 256)
    for other in (ref.cifar_augment_draw(cfg, 5, 1, 3, 256), ref.cifar_augment_draw(cfg, 6, 0, 3, 256),
                  ref.cifar_augment_draw(cfg, 5 + 2 ** 32, 0, 3, 256), ref.cifar_augment_draw(cfg, 5, 0, 4, 256),
                  ref.cifar_augment_draw(cfg, 5, 0, 3 + 2 ** 32, 256)):
        assert not torch.equal(base[0], other[0]) and not torch.equal(base[2], other[2])
    big = ref.cifar_augment_draw(cfg, 5, 0, 2 ** 40 + 7, 256)
    assert big[0].abs().max() <= 4 and big[2][:, 2:].max() <= 16
    again = ref.cifar_augment_draw(cfg, 5, 0, 3, 256)
    assert all(torch.equal(a, b) for a, b in zip(base, again))
    # image n's draw does not depend on the batch size
    assert all(torch.equal(a[:100], b) for a, b in zip(base, ref.cifar_augment_draw(cfg, 5, 0, 3, 100)))


def test_tags_are_disjoint_from_the_other_device_streams():
    from theanompi_b200.ops import drop_path
    for t in (ca.TAG, ca.TAG + 1):
        assert t > 0x7FFFFFFF and t != 0xFFFFFFFF and not drop_path.TAG <= t <= drop_path.TAG + drop_path.MAX_BLOCKS


def _train_draws(steps, **kw):
    """The cifar_augment buffers of every training step of a tiny Wide_ResNet on the CPU path."""
    ops.seed_dropout(0)
    m = _wrn(**kw)
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "t", False, device="cpu")
    out = []
    for i in range(steps):
        m.train_iter(i, rec)
        out.append(tuple(t.clone() for t in (m.cifar_aug.offs, m.cifar_aug.flips, m.cifar_aug.boxes)))
    return m, out, [float(c) for c in rec.train_info["cost"]]


def test_mixup_and_drop_path_do_not_change_the_draw():
    aug = dict(cutout=16, seed=3)
    _, plain, _ = _train_draws(3, cifar_augment=aug)
    _, both, _ = _train_draws(3, cifar_augment=aug, mixup=dict(alpha=1.0, cutmix_alpha=1.0, seed=3), drop_path_rate=0.3)
    for s, (a, b) in enumerate(zip(plain, both)):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        assert all(torch.equal(x, y) for x, y in zip(a, ref.cifar_augment_draw(ca.check_config(aug), 3, 0, s, 8)))
    assert not torch.equal(plain[0][0], plain[1][0])


# --------------------------------------------------------------------------- the reference apply against torchvision
def _devries(img, cy, cx, L):
    """DeVries & Taylor's Cutout (their util/cutout.py) on a CHW tensor with a given centre."""
    h, w = img.shape[1], img.shape[2]
    mask = np.ones((h, w), np.float32)
    y1, y2 = np.clip(cy - L // 2, 0, h), np.clip(cy + L // 2, 0, h)
    x1, x2 = np.clip(cx - L // 2, 0, w), np.clip(cx + L // 2, 0, w)
    mask[y1:y2, x1:x2] = 0.0
    return img * torch.from_numpy(mask).expand_as(img)


@pytest.mark.parametrize("pad", [0, 1, 4, 31])
@pytest.mark.parametrize("L", [0, 1, 16, 17, 32])
def test_reference_apply_matches_torchvision(pad, L):
    from torchvision.transforms.v2 import functional as TF
    g = torch.Generator().manual_seed(pad * 100 + L)
    N = 12
    x = torch.randint(0, 256, (N, 32, 32, 3), generator=g).float()
    mean = torch.rand((32, 32, 3), generator=g) * 255
    k = 2 * pad + 1
    oy = torch.randint(0, k, (N,), generator=g)
    ox = torch.randint(0, k, (N,), generator=g)
    oy[:4] = torch.tensor([0, 2 * pad, 0, 2 * pad]); ox[:4] = torch.tensor([0, 2 * pad, 2 * pad, 0])   # offsets at ±pad
    flips = (torch.arange(N) % 2).to(torch.uint8)
    cy = torch.randint(0, 32, (N,), generator=g).numpy()
    cx = torch.randint(0, 32, (N,), generator=g).numpy()
    cy[:4], cx[:4] = [0, 31, 0, 31], [0, 31, 31, 0]                 # centres at the corners
    offs = torch.stack([oy - pad, ox - pad], 1).to(torch.int32)
    boxes = torch.from_numpy(ca.cutout_boxes(cy, cx, L))
    got = ref.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), offs, flips, torch.float32, zero_fill=True)
    if L > 0:
        got = ref.random_erase(got, boxes)
    z = ((x - mean) * (1.0 / 64.0)).permute(0, 3, 1, 2)
    want = []
    for n in range(N):
        t = TF.pad(z[n], [pad], fill=0)
        t = TF.crop(t, int(oy[n]), int(ox[n]), 32, 32)
        if flips[n]:
            t = TF.horizontal_flip(t)
        want.append(_devries(t, int(cy[n]), int(cx[n]), L) if L > 0 else t)
    want = torch.stack(want).permute(0, 2, 3, 1)
    assert torch.equal(got, want)
    assert torch.equal(got.bfloat16(), want.bfloat16())
    got16 = ref.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), offs, flips, torch.bfloat16, zero_fill=True)
    if L > 0:
        got16 = ref.random_erase(got16, boxes)
    assert torch.equal(got16, want.bfloat16())
    if L % 2 == 1 and L > 1:                                       # an odd L cuts an (L − 1)-wide hole, as DeVries' code does
        assert int(boxes[4:, 2].max()) == L - 1


def test_zero_fill_whole_image_outside_and_zero_offsets_unchanged():
    g = torch.Generator().manual_seed(1)
    x = torch.randint(0, 256, (3, 32, 32, 3), generator=g).float()
    mean = torch.rand((32, 32, 3), generator=g) * 255
    offs = torch.tensor([[40, 0], [0, -32], [0, 0]], dtype=torch.int32)
    flips = torch.tensor([0, 1, 0], dtype=torch.uint8)
    out = ref.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), offs, flips, zero_fill=True)
    assert (out[:2] == 0).all()
    plain = ref.crop_mirror_normalize(x[2:], mean, 1.0 / 64.0, (32, 32), offs[2:], flips[2:])
    assert torch.equal(out[2:], plain) and torch.equal(plain[0], (x[2] - mean) / 64.0)


# --------------------------------------------------------------------------- models on the CPU
def test_wide_resnet_trains_and_its_stem_sees_the_reference_augmented_batch():
    m = _wrn(cifar_augment=dict(pad=4, cutout=16, seed=9), mixup=dict(alpha=1.0, seed=2), label_smoothing=0.1)
    m.compile_iter_fns("avg")
    w0 = m.arena.W.clone()
    seen = []
    fwd = m.stem.forward
    m.stem.forward = lambda x: (seen.append(x.detach().clone()), fwd(x))[1]
    ops.seed_dropout(0)
    rec = Recorder(None, 10 ** 6, "t", False, device="cpu")
    for i in range(3):
        m.train_iter(i, rec)
        x_in = m.x_in.clone()
        aug = m.cifar_aug
        want = ref.crop_mirror_normalize(x_in, m._mean, 1.0 / 64.0, (32, 32), aug.offs, aug.flips, torch.float32, zero_fill=True)
        want = ref.mix_batch(ref.random_erase(want, aug.boxes), m.mixer.rec)
        assert torch.equal(seen[-1], want), i
        assert (seen[-1] == 0).any()
    costs = [float(c) for c in rec.train_info["cost"]]
    assert all(np.isfinite(costs)) and not torch.equal(w0, m.arena.W)


def test_validation_equals_a_model_without_the_key():
    m, _, _ = _train_draws(2, cifar_augment=dict(cutout=8))
    plain = _wrn()
    plain.compile_iter_fns("avg")
    plain.arena.W.copy_(m.arena.W)
    plain.shared_x.copy_(m.shared_x); plain.shared_y.copy_(m.shared_y)
    stats_ = [(b.running_mean.clone(), b.running_var.clone()) for b in m._bn_layers()]

    def val(model):
        for b, (rm, rv) in zip(model._bn_layers(), stats_):
            b.running_mean = rm.clone(); b.running_var = rv.clone()
        return [float(v) for v in model.val_fn(0)]
    assert val(m) == val(plain)
    m.compile_inference(); plain.compile_inference()
    assert torch.equal(m.inf_fn(m.shared_x[:8]), plain.inf_fn(m.shared_x[:8]))


def test_grad_accum_micro_steps_draw_anew():
    m, draws, costs = _train_draws(4, cifar_augment=dict(cutout=16), grad_accum=2, optimizer="sgd", learning_rate=0.01)
    assert m.n_updates == 2 and all(np.isfinite(costs))
    for a, b in zip(draws, draws[1:]):
        assert not torch.equal(a[0], b[0])
