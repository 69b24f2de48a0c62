"""Ten-crop and mirrored validation (config['val_crops']) on the CPU: the key and the models that refuse it, the view table and
``reference.multi_crop_normalize`` against torchvision's ``ten_crop`` / ``center_crop``, ``reference.multi_view_xent`` against a float64
computation, and the CPU loader and the serial path with the key."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.data.utils import VC_KEY, check_val_crops  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

IMG = dict(no_paraload=True, n_class=8, batch_size=4, file_batch_size=4,
           data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
FLT_MIN = float(np.finfo(np.float32).tiny)


def _reseed():
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)


def _build(cls, **kw):
    _reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu")
    cfg.update(kw)
    return cls(cfg)


# --------------------------------------------------------------------------- configuration
def test_key_values_and_json_round_trip():
    assert [check_val_crops(v) for v in (1, 2, 10, np.int64(10))] == [1, 2, 10, 10]
    assert check_val_crops(json.loads(json.dumps({VC_KEY: 10}))[VC_KEY]) == 10


@pytest.mark.parametrize("bad", [0, 3, 5, 11, -1, True, False, 2.0, 10.0, "10", None, [10]])
def test_malformed_value_is_a_value_error_naming_the_key(bad):
    from theanompi_b200.models.alex_net import AlexNet
    with pytest.raises(ValueError, match=VC_KEY):
        check_val_crops(bad)
    with pytest.raises(ValueError, match=VC_KEY):
        _build(AlexNet, val_crops=bad, **IMG)


@pytest.mark.parametrize("name", ["AlexNet", "GoogLeNet", "VGG16", "ResNet50", "ResNet152", "ResNet50Torch"])
def test_imagenet_models_support_it_and_check_the_value(name):
    from theanompi_b200.models import alex_net, googlenet
    from theanompi_b200.models.lasagne_model_zoo import resnet50, resnet152_outdated, vgg16
    cls = {"AlexNet": alex_net.AlexNet, "GoogLeNet": googlenet.GoogLeNet, "VGG16": vgg16.VGG16, "ResNet50": resnet50.ResNet50,
           "ResNet152": resnet152_outdated.ResNet152, "ResNet50Torch": resnet50.ResNet50Torch}[name]
    assert cls.supports_resized_crop
    # the key is checked before the model or its loader is built
    with pytest.raises(ValueError, match=VC_KEY):
        _build(cls, val_crops=4, **IMG)


def _refusing():
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet, Wide_ResNetTorch
    from theanompi_b200.models.lasagne_model_zoo.lsgan import LSGAN, NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.wgan import WGAN, NativeWGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    return [Cifar10_model, Wide_ResNet, Wide_ResNetTorch, AlexNet_sc, LSTM, LSTMTorch, WGAN, NativeWGAN, LSGAN, NativeLSGAN]


@pytest.mark.parametrize("idx", range(10))
@pytest.mark.parametrize("v", [2, 10])
def test_other_models_refuse_it(idx, v):
    cls = _refusing()[idx]
    assert not cls.supports_resized_crop
    with pytest.raises(ValueError, match=VC_KEY):
        _build(cls, val_crops=v, n_class=8, batch_size=4, file_batch_size=4)


# --------------------------------------------------------------------------- views
def test_view_table_follows_ten_crop():
    t = ref.multi_crop_views((256, 256), (227, 227), 10).tolist()
    assert t == [[0, 0, 0], [0, 29, 0], [29, 0, 0], [29, 29, 0], [14, 14, 0],
                 [0, 29, 1], [0, 0, 1], [29, 29, 1], [29, 0, 1], [14, 15, 1]]
    assert ref.multi_crop_views((256, 256), (227, 227), 2).tolist() == [[14, 14, 0], [14, 15, 1]]
    assert ref.multi_crop_views((256, 256), (224, 224), 1).tolist() == [[16, 16, 0]]
    for bad in (0, 3, 5):
        with pytest.raises(ValueError):
            ref.multi_crop_views((256, 256), (227, 227), bad)


@pytest.mark.parametrize("ch", [227, 224])
@pytest.mark.parametrize("mean_mode", ["pixel", "scalar"])
def test_reference_views_equal_torchvision(ch, mean_mode):
    import torchvision.transforms.v2.functional as TF
    g = torch.Generator().manual_seed(ch)
    x = torch.randint(0, 256, (3, 256, 256, 3), generator=g, dtype=torch.uint8)
    mean = torch.rand((256, 256, 3), generator=g) * 255 if mean_mode == "pixel" else torch.tensor([127.5])
    cs = torch.tensor([1 / 255 / 0.229, 1 / 255 / 0.224, 1 / 255 / 0.225])
    norm = ((x.float() - mean) * cs).permute(0, 3, 1, 2)                # the normalised fp32 image, NCHW
    ten = ref.multi_crop_normalize(x, mean, cs, (ch, ch), 10)
    assert ten.shape == (10, 3, ch, ch, 3) and ten.dtype == torch.float32
    for v, want in enumerate(TF.ten_crop(norm, [ch, ch])):
        assert torch.equal(ten[v], want.permute(0, 2, 3, 1)), v
    two = ref.multi_crop_normalize(x, mean, cs, (ch, ch), 2)
    assert torch.equal(two[0], TF.center_crop(norm, [ch, ch]).permute(0, 2, 3, 1))
    assert torch.equal(two[1], TF.center_crop(norm.flip(3), [ch, ch]).permute(0, 2, 3, 1))
    # view 4 is today's validation crop
    offs, flips = torch.tensor([[(256 - ch) // 2] * 2] * 3, dtype=torch.int32), torch.zeros(3, dtype=torch.uint8)
    assert torch.equal(ten[4], ref.crop_mirror_normalize(x, mean, cs, (ch, ch), offs, flips))
    assert torch.equal(ref.multi_crop_normalize(x, mean, cs, (ch, ch), 1)[0], ten[4])


# --------------------------------------------------------------------------- scores
def _xent64(zs, y):
    p = torch.stack([torch.softmax(z.double(), 1) for z in zs]).mean(0)
    B, C = p.shape
    py = p[torch.arange(B), y]
    rank = torch.tensor([int((p[b] > py[b]).sum()) + int((p[b, :y[b]] == py[b]).sum()) for b in range(B)])
    return float((-py.clamp_min(FLT_MIN).log()).mean()), float((rank >= 1).double().mean()), float((rank >= 5).double().mean()), p


def test_multi_view_xent_against_float64():
    g = torch.Generator().manual_seed(3)
    B, C, V = 12, 50, 10
    zs = [torch.randn((B, C), generator=g) * 2 for _ in range(V)]
    y = torch.randint(0, C, (B,), generator=g)
    y[0], y[1] = 0, C - 1
    for z in zs:
        z[2, :] = 1.0                          # a fully tied row: the label's rank is its index
        z[3, :8] = 4.0                         # tied at the top, label 6 (rank 6: a top-5 error) …
        z[4, :8] = 4.0                         # … and label 2 (rank 2: top-1 error only)
        z[5, y[5]] = -1e4                      # p̄_y underflows to the FLT_MIN clamp
    y[2], y[3], y[4] = 7, 6, 2
    c, e1, e5, p = ref.multi_view_xent(zs, y)
    wc, we1, we5, wp = _xent64(zs, y)
    assert p.dtype == torch.float64 and torch.allclose(p, wp, rtol=1e-14, atol=0)
    assert abs(float(c) - wc) <= 1e-12 * abs(wc) and float(e1) == we1 and float(e5) == we5
    py = p[torch.arange(B), y]
    assert float(py[5]) < FLT_MIN and float(-py[5].clamp_min(FLT_MIN).log()) == pytest.approx(87.336544750553927)
    c32, e132, e532, p32 = ref.multi_view_xent(zs, y, torch.float32)
    assert p32.dtype == torch.float32 and abs(float(c32) - wc) <= 1e-5 * wc
    assert round(float(e132) * B) == round(we1 * B) and round(float(e532) * B) == round(we5 * B)


def test_view_metrics_tie_rule():
    p = torch.tensor([[0.25, 0.25, 0.25, 0.25, 0.0, 0.0]] * 4)
    c, e1, e5 = ref.view_metrics(p, torch.tensor([0, 1, 3, 4]))
    # ranks 0, 1, 3 and 4 (label 4 sits below the four tied 0.25s): top-1 errors 3 / 4, no top-5 error
    assert float(e1) == 0.75 and float(e5) == 0.0
    assert float(c) == pytest.approx((3 * np.log(4) - np.log(FLT_MIN)) / 4)


# --------------------------------------------------------------------------- loaders
@pytest.mark.parametrize("V", [2, 10])
def test_cpu_loader_views_and_unchanged_training_batches(V):
    from theanompi_b200.models.data.imagenet import ImageNet_data
    seqs = {}
    for vc in (1, V):
        d = ImageNet_data(file_batch_size=4, n_train_files=2, n_val_files=1, synthetic=True)
        d.batch_data(4)
        ld = d.para_load_init("cpu", 227, 227, True, False, val_crops=vc)
        seq = []
        for item, m in ((d.train_img[0], "train"), (d.val_img[0], "val"), (d.train_img[1], "train")):
            ld.request(item, m)
            b = ld.get()
            seq.append((m, b.x.clone(), b.h2d_bytes))
        d.para_load_close()
        seqs[vc] = (seq, d)
    (a, d), (b, _) = seqs[V], seqs[1]
    assert [s[2] for s in a] == [s[2] for s in b]
    assert torch.equal(a[0][1], b[0][1]) and torch.equal(a[2][1], b[2][1])
    raw = np.empty((4, 256, 256, 3), dtype=np.uint8)
    src = d.read(d.val_img[0], raw)
    raw = torch.from_numpy(src.numpy() if src is not None else raw)
    want = ref.multi_crop_normalize(raw, torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5]), (227, 227), V)
    assert a[1][1].shape == (V, 4, 227, 227, 3) and torch.equal(a[1][1], want)
    assert torch.equal(a[1][1][0 if V == 2 else 4], b[1][1])


@pytest.mark.parametrize("V", [2, 10])
def test_serial_path_has_the_views_and_unchanged_training_batches(V):
    from theanompi_b200.models.alex_net import AlexNet
    runs = {}
    for vc in (1, V):
        m = _build(AlexNet, val_crops=vc, **IMG)
        assert m.data.loader is None and m.val_x is None
        d = m.data
        xs = []
        for mode, img, lab in (("train", d.train_img_shard, d.train_labels_shard), ("val", d.val_img_shard, d.val_labels_shard),
                               ("train", d.train_img_shard, d.train_labels_shard)):
            m._load_file_batch(mode, 0, img, lab, len(img))
            xs.append((m.shared_x.clone(), None if m.val_x is None else m.val_x.clone()))
        runs[vc] = (m, xs)
    (m, a), (m1, b) = runs[V], runs[1]
    assert torch.equal(a[0][0], b[0][0]) and torch.equal(a[2][0], b[2][0])
    assert a[1][1].shape == (V, 4, 227, 227, 3)
    # the single-crop serial batch divides by 255 and by std where the views (like the loader) multiply by 1 / (255·std)
    assert torch.allclose(a[1][1][0 if V == 2 else 4], b[1][0], rtol=1e-6, atol=1e-6), "the centre view is the validation crop"
    # validation on the CPU runs the reference on the views' logits
    m.compile_val()
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    try:
        c, e1, e5 = m.val_fn(0)
        zs = []
        with torch.no_grad():
            for v in range(V):
                m.forward(m.val_x[v, :4])
                zs.append(m.output_layer.logits.clone())
    finally:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn()
    wc, we1, we5, _ = _xent64(zs, m.shared_y[:4])
    assert abs(float(c) - wc) <= 1e-5 * (1 + wc) and round(float(e1) * 4) == round(we1 * 4) and round(float(e5) * 4) == round(we5 * 4)
