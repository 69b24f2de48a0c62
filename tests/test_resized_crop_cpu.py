"""Random-resized crop (config['random_resized_crop']) on the CPU: the validation of the key and the models that refuse it, the
vectorised box draw against torchvision's RandomResizedCrop.get_params, the reference resample against torchvision's resized_crop, and
the CPU ParaLoader and the serial load_batch path with the key."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.data.utils import (RRC_KEY, check_resized_crop, draw_crops, draw_resized_crops,  # noqa: E402
                                              resized_crop_rng)
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

IMG = dict(no_paraload=True, n_class=8, batch_size=4, file_batch_size=4,
           data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))


def _reseed():
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)


def _build(cls, **kw):
    _reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu")
    cfg.update(kw)
    return cls(cfg)


# --------------------------------------------------------------------------- configuration
def test_defaults_and_json_forms():
    assert check_resized_crop(None) is None
    assert check_resized_crop({}) == {"scale": (0.08, 1.0), "ratio": (0.75, 4.0 / 3.0), "seed": 0}
    cfg = check_resized_crop({"scale": [0.25, 1], "ratio": (1, 2), "seed": np.int64(-1)})
    assert cfg == {"scale": (0.25, 1.0), "ratio": (1.0, 2.0), "seed": 2 ** 64 - 1}


@pytest.mark.parametrize("bad", [
    [0.08, 1.0], "scale", {"size": 3}, {"scale": True}, {"scale": [True, 1.0]}, {"scale": [0.1]}, {"scale": [0.1, 0.5, 1.0]},
    {"scale": [0.0, 1.0]}, {"scale": [0.5, 1.5]}, {"scale": [0.6, 0.5]}, {"scale": [float("nan"), 1.0]}, {"scale": ["0.1", 1.0]},
    {"ratio": [0.0, 1.0]}, {"ratio": [-1.0, 1.0]}, {"ratio": [2.0, 1.0]}, {"ratio": [1.0, float("inf")]}, {"ratio": 1.0},
    {"seed": 1.0}, {"seed": True}, {"seed": "0"}, {"seed": None}])
def test_malformed_config_is_a_value_error_naming_the_key(bad):
    with pytest.raises(ValueError, match=RRC_KEY):
        check_resized_crop(bad)
    from theanompi_b200.models.alex_net import AlexNet
    with pytest.raises(ValueError, match=RRC_KEY):
        _build(AlexNet, random_resized_crop=bad, **IMG)


def _refused():
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet, Wide_ResNetTorch
    from theanompi_b200.models.lasagne_model_zoo.lsgan import LSGAN, NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    wrn = dict(batch_size=8, file_batch_size=8, depth=10, widen=1, data_kwargs=dict(n_synthetic=64, synthetic=True))
    return [(AlexNet_sc, IMG), (Cifar10_model, dict(batch_size=4, file_batch_size=8, data_kwargs=dict(n_synthetic=64, synthetic=True))),
            (Wide_ResNet, wrn), (Wide_ResNetTorch, wrn),
            (NativeWGAN, dict(data_kwargs=dict(n_synthetic=128))), (NativeLSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (WGAN, dict(data_kwargs=dict(n_synthetic=128))), (LSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (LSTM, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (LSTMTorch, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200)))]


def test_models_without_the_imagenet_loader_refuse_it_at_construction():
    for cls, kw in _refused():
        assert cls.supports_resized_crop is False, cls
        with pytest.raises(ValueError, match=RRC_KEY + " is not supported"):
            _build(cls, random_resized_crop={}, **kw)
        _build(cls, random_resized_crop=None, **kw)


def test_supporting_models():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50, ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    for cls in (AlexNet, GoogLeNet, VGG16, ResNet50, ResNet152, ResNet50Torch):
        assert cls.supports_resized_crop is True, cls
    m = _build(ResNet50, random_resized_crop={"scale": [0.5, 1.0], "seed": 3}, blocks=(1, 1, 1, 1), **IMG)
    assert m.resized_crop == {"scale": (0.5, 1.0), "ratio": (0.75, 4.0 / 3.0), "seed": 3}
    assert _build(ResNet50, blocks=(1, 1, 1, 1), **IMG).resized_crop is None


@pytest.mark.parametrize("flag", ["batch_crop_mirror", "rand_crop"])
def test_a_batch_wide_or_centre_crop_contradicts_it(flag):
    from theanompi_b200.models.alex_net import AlexNet
    cls = type("AlexNetFixed", (AlexNet,), {flag: flag == "batch_crop_mirror"})
    with pytest.raises(ValueError, match="%s .*contradicts %s" % (RRC_KEY, flag)):
        _build(cls, random_resized_crop={}, **IMG)


# --------------------------------------------------------------------------- the draw
def test_boxes_lie_inside_the_image():
    rs = np.random.RandomState(0)
    for t in range(200):
        H, W = (int(v) for v in rs.randint(1, 300, 2))
        lo = float(rs.uniform(0.01, 1.0)); scale = (lo, float(rs.uniform(lo, 1.0)))
        rlo = float(np.exp(rs.uniform(-3, 3))); ratio = (rlo, rlo * float(np.exp(rs.uniform(0, 2))))
        boxes, flips = draw_resized_crops(64, (H, W), scale, ratio, np.random.default_rng(t))
        assert boxes.dtype == np.int32 and boxes.shape == (64, 4) and flips.dtype == np.uint8 and set(flips) <= {0, 1}
        y0, x0, h, w = boxes.T
        assert (h >= 1).all() and (w >= 1).all() and (y0 >= 0).all() and (x0 >= 0).all()
        assert (y0 + h <= H).all() and (x0 + w <= W).all()


@pytest.mark.parametrize("hw,ratio,want", [
    ((256, 256), (2.0, 3.0), (64, 0, 128, 256)),          # W / H = 1 < 2: full width, h = round(256 / 2), centred
    ((256, 256), (0.25, 0.4), (0, 77, 256, 102)),         # W / H = 1 > 0.4: full height, w = round(256 · 0.4) = round(102.4)
    ((100, 300), (0.5, 2.0), (0, 50, 100, 200))])         # W / H = 3 > 2: w = 200, centred
def test_fallback_is_the_clamped_centred_box(hw, ratio, want):
    """scale = [1, 1] with a ratio range that excludes the image's own never fits, so every image takes torchvision's fallback."""
    boxes, _ = draw_resized_crops(16, hw, (1.0, 1.0), ratio, np.random.default_rng(1))
    assert (boxes == np.int32(want)).all(), boxes[0]


def test_fallback_matches_torchvision():
    tv = pytest.importorskip("torchvision")
    img = torch.zeros(3, 256, 256)
    torch.manual_seed(0)
    for ratio in ((2.0, 3.0), (0.25, 0.4)):
        want = tv.transforms.RandomResizedCrop.get_params(img, [1.0, 1.0], list(ratio))
        boxes, _ = draw_resized_crops(4, (256, 256), (1.0, 1.0), ratio, np.random.default_rng(0))
        assert tuple(int(v) for v in boxes[0]) == tuple(want)


@pytest.mark.parametrize("hw,scale,ratio", [((256, 256), (0.08, 1.0), (0.75, 4.0 / 3.0)), ((256, 256), (0.5, 1.0), (0.5, 2.0)),
                                            ((120, 300), (0.2, 0.9), (1.0, 3.0))])
def test_h_and_w_distributions_match_torchvision(hw, scale, ratio):
    """Two-sample Kolmogorov–Smirnov on h, w, y0 and x0 over 20,000 draws each, at fixed seeds: p > 1e-3 (a correct draw fails one of
    these 12 comparisons with probability about 1 %), and the flip rate within 5σ of ½."""
    tv = pytest.importorskip("torchvision")
    from scipy.stats import ks_2samp
    n = 20000
    boxes, flips = draw_resized_crops(n, hw, scale, ratio, np.random.default_rng(12345))
    torch.manual_seed(54321)
    img = torch.zeros(1, *hw)
    want = np.array([tv.transforms.RandomResizedCrop.get_params(img, list(scale), list(ratio)) for _ in range(n)])
    for k, name in enumerate(("y0", "x0", "h", "w")):
        p = ks_2samp(boxes[:, k], want[:, k]).pvalue
        assert p > 1e-3, (name, p)
    assert abs(flips.mean() - 0.5) < 5 * 0.5 / np.sqrt(n)


def test_ranks_draw_apart_and_a_key_reproduces():
    cfg = check_resized_crop({"seed": 7})
    a = draw_resized_crops(128, (256, 256), cfg["scale"], cfg["ratio"], resized_crop_rng(cfg, 0))
    b = draw_resized_crops(128, (256, 256), cfg["scale"], cfg["ratio"], resized_crop_rng(cfg, 1))
    c = draw_resized_crops(128, (256, 256), cfg["scale"], cfg["ratio"], resized_crop_rng(cfg, 0))
    assert not np.array_equal(a[0], b[0])
    assert np.array_equal(a[0], c[0]) and np.array_equal(a[1], c[1])
    d = draw_resized_crops(128, (256, 256), cfg["scale"], cfg["ratio"], resized_crop_rng(check_resized_crop({"seed": 8}), 0))
    assert not np.array_equal(a[0], d[0])


# --------------------------------------------------------------------------- the reference resample
def _batch(N=6, H=40, W=48, C=3, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (N, H, W, C), dtype=torch.uint8, generator=g)
    mean = torch.rand(H, W, C, generator=g) * 255
    return x, mean, torch.tensor([1 / 255 / 0.229, 1 / 255 / 0.224, 1 / 255 / 0.225])


@pytest.mark.parametrize("out_hw", [(24, 24), (24, 30), (40, 48)])
def test_reference_matches_torchvision_resized_crop(out_hw):
    """Boxes smaller than, equal to and larger than the output, mirrored and not: torchvision.transforms.v2.functional.resized_crop
    (BILINEAR, antialias=False) of the normalised image, then the flip."""
    pytest.importorskip("torchvision")
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms.v2 import functional as TF
    x, mean, cs = _batch()
    oh, ow = out_hw
    boxes = torch.tensor([[0, 0, 40, 48], [3, 5, 7, 9], [40 - oh, 48 - ow, oh, ow],        # the third: the output's size, at the corner
                          [39, 47, 1, 1], [5, 4, 35, 44], [0, 20, 30, 28]], dtype=torch.int32)
    flips = torch.tensor([0, 1, 0, 1, 1, 0], dtype=torch.uint8)
    got = ref.resized_crop_mirror_normalize(x, mean, cs, out_hw, boxes, flips)
    norm = ((x.float() - mean) * cs).permute(0, 3, 1, 2)
    for i in range(x.shape[0]):
        y0, x0, h, w = (int(v) for v in boxes[i])
        want = TF.resized_crop(norm[i], y0, x0, h, w, list(out_hw), interpolation=InterpolationMode.BILINEAR, antialias=False)
        want = want.permute(1, 2, 0)
        if flips[i]:
            want = want.flip(1)
        torch.testing.assert_close(got[i], want, rtol=1e-6, atol=1e-6)


def test_box_of_the_output_size_is_the_fixed_crop():
    x, mean, cs = _batch()
    offs = torch.tensor([[0, 0], [16, 24], [3, 7], [8, 1], [16, 0], [0, 24]], dtype=torch.int32)
    flips = torch.tensor([0, 1, 1, 0, 1, 0], dtype=torch.uint8)
    boxes = torch.cat([offs, torch.tensor([[24, 24]] * 6, dtype=torch.int32)], 1)
    for m in (mean, mean[0, 0], mean[0, 0, :1]):
        for s in (cs, 1 / 255.0):
            got = ref.resized_crop_mirror_normalize(x, m, s, (24, 24), boxes, flips)
            want = ref.crop_mirror_normalize(x, m, s, (24, 24), offs, flips)
            assert torch.equal(got, want)


def test_reference_refuses_a_box_outside_the_image():
    x, mean, cs = _batch(N=1)
    with pytest.raises(ValueError, match="not inside"):
        ref.resized_crop_mirror_normalize(x, mean, cs, (8, 8), torch.tensor([[35, 0, 8, 8]]), torch.zeros(1))


# --------------------------------------------------------------------------- loader
def _data():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=8, size_hw=32)
    d.batch_data(8)
    return d


def _raw(d, item):
    raw = np.empty((8, 32, 32, 3), np.uint8)
    src = d.read(item, raw)
    return torch.from_numpy(src.numpy() if src is not None else raw)


def test_cpu_loader_train_batches_are_the_reference_of_their_boxes():
    d = _data()
    cfg = check_resized_crop({"scale": [0.1, 1.0], "ratio": [0.5, 2.0], "seed": 5})
    ld = d.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, resized_crop=cfg, rank=2)
    rng = resized_crop_rng(cfg, 2)
    mean, cs = torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5])
    ld.request(d.train_img[0], "train")
    for k in range(1, 4):
        ld.request(d.train_img[k % 3], "train")
        b = ld.get()
        boxes, flips = draw_resized_crops(8, (32, 32), cfg["scale"], cfg["ratio"], rng)
        assert np.array_equal(b.boxes, boxes) and np.array_equal(b.flips, flips)
        want = ref.resized_crop_mirror_normalize(_raw(d, b.item), mean, cs, (20, 24), boxes, flips)
        assert tuple(b.x.shape) == (8, 20, 24, 3) and torch.equal(b.x, want)
        assert b.h2d_bytes == 8 * 32 * 32 * 3 + 8 * 17
    ld.drain(); d.para_load_close()


def test_cpu_loader_val_batches_and_runs_without_the_key_are_unchanged():
    outs = []
    for cfg in (None, check_resized_crop({})):
        d = _data()
        ld = d.para_load_init("cpu", 24, 24, rand_crop=True, batch_crop_mirror=False, resized_crop=cfg)
        if cfg is None:
            rs = np.random.RandomState(1234)                  # the loader's fixed-crop generator
        seq = []
        for mode in ("val", "train", "val") if cfg is not None else ("val",):
            ld.request(d.train_img[0], mode); ld.request(d.train_img[1], mode)
            for _ in range(2):
                b = ld.get()
                if mode == "val":
                    seq.append(b.x.clone())
                    assert b.boxes is None and b.h2d_bytes == 8 * 32 * 32 * 3 + 8 * 9
            ld.drain()
        d.para_load_close()
        outs.append(seq)
    for got in outs[1][:2], outs[1][2:]:
        assert all(torch.equal(a, b) for a, b in zip(got, outs[0]))
    # without the key the train draw is the fixed-crop generator's, exactly as before
    d = _data()
    ld = d.para_load_init("cpu", 24, 24, rand_crop=True, batch_crop_mirror=False)
    ld.request(d.train_img[0], "train"); ld.request(d.train_img[1], "train")
    b = ld.get()
    offs, flips = draw_crops(8, (32, 32), (24, 24), "train", True, False, rs)
    want = ref.crop_mirror_normalize(_raw(d, b.item), torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5]),
                                     (24, 24), torch.from_numpy(offs), torch.from_numpy(flips))
    assert b.boxes is None and torch.equal(b.x, want)
    ld.drain(); d.para_load_close()


def test_serial_load_batch_applies_it():
    from theanompi_b200.models.alex_net import AlexNet
    cfg = {"scale": [0.3, 0.6], "seed": 11}
    m = _build(AlexNet, random_resized_crop=cfg, **IMG)
    item = m.data.train_img_shard[0]
    x = m.data.load_batch(item, "train", m)
    vcfg = check_resized_crop(cfg)
    boxes, flips = draw_resized_crops(4, (256, 256), vcfg["scale"], vcfg["ratio"], resized_crop_rng(vcfg, 0))
    raw = np.empty((4, 256, 256, 3), np.uint8)
    src = m.data.read(item, raw)
    raw = torch.from_numpy(src.numpy() if src is not None else raw)
    want = ref.resized_crop_mirror_normalize(raw, torch.from_numpy(m.data.rawdata[4]), torch.from_numpy(1.0 / 255.0 / m.data.rawdata[5]),
                                             (227, 227), boxes, flips)
    assert tuple(x.shape) == (4, 227, 227, 3) and torch.equal(x, want)
    assert (boxes[:, 2] * boxes[:, 3] <= 0.6 * 256 * 256 * 1.05).all()
    # validation keeps the centre crop
    v = m.data.load_batch(item, "val", m)
    want_v = ((raw.numpy().astype(np.float32) - m.data.rawdata[4]) / 255.0 / m.data.rawdata[5])[:, 14:241, 14:241]
    assert torch.equal(v, torch.from_numpy(np.ascontiguousarray(want_v)))


def test_tiny_models_train_with_it_on_the_cpu():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    from theanompi_b200.utils.recorder import Recorder
    for cls, kw in ((AlexNet, {}), (ResNet50, dict(blocks=(1, 1, 1, 1)))):
        m = _build(cls, random_resized_crop={}, **dict(IMG, **kw))
        m.compile_iter_fns("avg")
        rec = Recorder(None, 10 ** 6, cls.__name__, False, device="cpu")
        for i in range(2):
            m.train_iter(i, rec)
        m.reset_iter("val")
        m.val_iter(0, rec)
        assert all(np.isfinite(float(c)) for c in rec.train_info["cost"]) and np.isfinite(float(rec.val_info["cost"][-1]))
