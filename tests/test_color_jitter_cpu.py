"""Colour jitter and PCA lighting (config['color_jitter']) on the CPU: the validation of the key and the models that refuse it, the
composed per-image records against the float64 sequential oracle (tests/color_oracle.py), the draw's statistics and its independence of
the crop draws, the torch reference against the oracle, and the CPU ParaLoader and the serial load_batch path with the key."""
import itertools
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import color_oracle as co  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.data.utils import (CJ_KEY, check_color_jitter, check_resized_crop, color_jitter_maps,  # noqa: E402
                                              color_jitter_records, color_jitter_rng, draw_crops, draw_resized_crops, resized_crop_rng)
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

IMG = dict(no_paraload=True, n_class=8, batch_size=4, file_batch_size=4,
           data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
ALL4 = {"brightness": 0.4, "contrast": 0.4, "saturation": 0.4, "lighting": 0.1}


def _reseed():
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)


def _build(cls, **kw):
    _reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu")
    cfg.update(kw)
    return cls(cfg)


# --------------------------------------------------------------------------- configuration
def test_defaults_and_json_round_trip():
    assert check_color_jitter(None) is None
    assert check_color_jitter({"lighting": 0.1}) == {"brightness": 0.0, "contrast": 0.0, "saturation": 0.0, "lighting": 0.1, "seed": 0}
    cfg = dict(ALL4, seed=np.int64(-1))
    assert check_color_jitter(cfg) == dict(ALL4, seed=2 ** 64 - 1)
    assert check_color_jitter(json.loads(json.dumps({"color_jitter": dict(ALL4, seed=3)}))["color_jitter"]) == dict(ALL4, seed=3)
    assert check_color_jitter({"brightness": 1, "contrast": np.float32(1.0)})["contrast"] == 1.0


@pytest.mark.parametrize("bad", [
    [0.4, 0.4], "lighting", 0.1, {"hue": 0.1}, {}, {"lighting": 0.0}, {"brightness": 0, "contrast": 0, "saturation": 0, "lighting": 0},
    {"brightness": True}, {"lighting": False}, {"brightness": float("nan")}, {"contrast": float("inf")}, {"saturation": "0.4"},
    {"lighting": [0.1]}, {"lighting": None}, {"brightness": -0.1}, {"contrast": 1.5}, {"lighting": 1.0000001},
    {"lighting": 0.1, "seed": 1.0}, {"lighting": 0.1, "seed": True}, {"lighting": 0.1, "seed": "0"}, {"lighting": 0.1, "seed": None}])
def test_malformed_config_is_a_value_error_naming_the_key(bad):
    from theanompi_b200.models.alex_net import AlexNet
    with pytest.raises(ValueError, match=CJ_KEY):
        check_color_jitter(bad)
    with pytest.raises(ValueError, match=CJ_KEY):
        _build(AlexNet, color_jitter=bad, **IMG)


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


def test_models_without_the_imagenet_loader_refuse_it():
    for cls, kw in _refused():
        with pytest.raises(ValueError, match=CJ_KEY + " is not supported"):
            _build(cls, color_jitter={"lighting": 0.1}, **kw)


def test_supporting_models_and_any_crop_mode():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50, ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    for cls in (AlexNet, GoogLeNet, VGG16, ResNet50, ResNet152, ResNet50Torch):
        assert cls.supports_resized_crop is True, cls
    m = _build(ResNet50, color_jitter=dict(ALL4, seed=3), random_resized_crop={}, blocks=(1, 1, 1, 1), **IMG)
    assert m.color_jitter == dict(ALL4, seed=3)
    assert _build(ResNet50, blocks=(1, 1, 1, 1), **IMG).color_jitter is None
    for flag in ("batch_crop_mirror", "rand_crop"):
        cls = type("AlexNetFixed", (AlexNet,), {flag: flag == "batch_crop_mirror"})
        assert _build(cls, color_jitter={"lighting": 0.1}, **IMG).color_jitter["lighting"] == 0.1
    # the constructors of the other supporting models (heavier to build) take the same path through ModelBase
    for cls in (GoogLeNet, VGG16, ResNet152, ResNet50Torch):
        assert cls.check_color_jitter is AlexNet.check_color_jitter


# --------------------------------------------------------------------------- the composed record
def _apply_record(rec, v):
    """M·v + K·μ + ℓ in float64 from a record."""
    rec = np.asarray(rec, np.float64)
    M, K, ell = rec[0:9].reshape(3, 3), rec[9:18].reshape(3, 3), rec[18:21]
    return v @ M.T + K @ v.reshape(-1, 3).mean(0) + ell


def _compose64(factors, order, alpha):
    """A float64 record (no fp32 rounding) from color_jitter_maps."""
    M, K, ell = color_jitter_maps(factors, order, alpha)
    rec = np.zeros((len(factors), 24))
    rec[:, :9], rec[:, 9:18], rec[:, 18:21] = M.reshape(-1, 9), K.reshape(-1, 9), ell
    return rec


def test_record_matches_the_sequential_oracle_in_every_order():
    """All six orders and the edge factors 0, 1 and 2 (strengths 0 and 1): the float64 composed map agrees with the sequential
    application within 1e-12 relative; the fp32 record of color_jitter_records within its rounding."""
    rng = np.random.default_rng(0)
    v = rng.uniform(0, 255, (7, 5, 3))
    for perm in itertools.permutations(range(3)):
        for fac in ([1.3, 0.7, 1.2], [0.0, 1.0, 2.0], [1.0, 1.0, 1.0], [2.0, 0.0, 0.0], [0.6, 2.0, 1.0]):
            alpha = rng.normal(0, 0.1, 3)
            want = co.apply_sequential(v, fac, perm, alpha)
            got64 = _apply_record(_compose64(np.array([fac]), np.array([perm]), np.array([alpha]))[0], v)
            assert np.abs(got64 - want).max() <= 1e-12 * np.abs(want).max() + 1e-12

    # the fp32 records the loader draws, replayed through the oracle
    cfg = check_color_jitter({"brightness": 1.0, "contrast": 1.0, "saturation": 1.0, "lighting": 1.0, "seed": 2})
    rec, fac, order, alpha = color_jitter_records(64, cfg, color_jitter_rng(cfg, 0))
    assert sorted(set(map(tuple, order))) == sorted(itertools.permutations(range(3)))
    for i in range(64):
        want = co.apply_sequential(v, fac[i], order[i], alpha[i])
        S = np.abs(v) @ np.abs(rec[i, :9].reshape(3, 3)).T + np.abs(rec[i, 9:18].reshape(3, 3)) @ v.reshape(-1, 3).mean(0) + np.abs(rec[i, 18:21])
        assert (np.abs(_apply_record(rec[i], v) - want) <= 2 ** -23 * S + 1e-9).all(), i
        assert (rec[i, 21:] == 0).all()


def test_the_order_is_immaterial_and_wrong_records_fail():
    """Brightness, saturation and contrast commute: g sums to 1, so saturation keeps the grey level and its mean, and brightness
    scales both.  Every order composes the same map within 1e-12 relative.  A record whose later operations leave K untouched, or whose
    ℓ has its channels reversed, fails."""
    rng = np.random.default_rng(1)
    v = rng.uniform(0, 255, (6, 6, 3))
    fac, perm, alpha = np.array([1.3, 0.6, 1.35]), (2, 0, 1), np.array([0.1, -0.08, 0.05])
    want = co.apply_sequential(v, fac, perm, alpha)
    for other in itertools.permutations(range(3)):
        w2 = co.apply_sequential(v, fac, other, alpha)
        assert np.abs(w2 - want).max() <= 1e-12 * np.abs(want).max()
    good = _compose64(fac[None], np.array([perm]), alpha[None])[0]
    tol = 2 ** -21 * (np.abs(want).max() + 255 * 4)
    assert np.abs(_apply_record(good, v) - want).max() <= tol
    # contrast first, then brightness and saturation applied to M only
    a, s, c = fac
    G = np.outer(np.ones(3), co.CJ_GRAY)
    P = s * np.eye(3) + (1 - s) * G
    stale = good.copy()
    stale[9:18] = ((1 - c) * G).reshape(-1)
    assert np.abs(_apply_record(stale, v) - want).max() > 100 * tol
    assert np.allclose((P @ (a * (1 - c) * G)).reshape(-1), good[9:18], rtol=1e-6, atol=1e-7)
    rev = good.copy()
    rev[18:21] = good[18:21][::-1]
    assert np.abs(_apply_record(rev, v) - want).max() > 100 * tol


# --------------------------------------------------------------------------- the draw
def test_draw_statistics():
    n = 100_000
    cfg = check_color_jitter({"brightness": 0.4, "contrast": 0.3, "saturation": 0.2, "lighting": 0.1, "seed": 5})
    rec, fac, order, alpha = color_jitter_records(n, cfg, color_jitter_rng(cfg, 0))
    assert rec.dtype == np.float32 and rec.shape == (n, 24) and rec.nbytes == n * 96
    for j, k in enumerate(("brightness", "saturation", "contrast")):
        v = cfg[k]
        assert fac[:, j].min() >= 1 - v and fac[:, j].max() <= 1 + v
        assert abs(fac[:, j].mean() - 1) < 4 * v / np.sqrt(3 * n)
    counts = {}
    for p in map(tuple, order):
        counts[p] = counts.get(p, 0) + 1
    assert sorted(counts) == sorted(itertools.permutations(range(3)))
    sd = np.sqrt(n * (1 / 6) * (5 / 6))
    assert all(abs(c - n / 6) < 5 * sd for c in counts.values()), counts
    assert np.abs(alpha.mean(0)).max() < 5 * 0.1 / np.sqrt(n)
    assert np.abs(alpha.std(0) - 0.1).max() < 5 * 0.1 / np.sqrt(2 * n)
    np.testing.assert_allclose(rec[:, 18:21], co.lighting(alpha).astype(np.float32), rtol=2 ** -22, atol=1e-6)


def test_zero_strengths_give_factors_of_exactly_one_without_shifting_the_stream():
    full = check_color_jitter(dict(ALL4, seed=9))
    light = check_color_jitter({"lighting": 0.1, "seed": 9})
    _, f_full, o_full, a_full = color_jitter_records(512, full, color_jitter_rng(full, 3))
    rec, f, o, a = color_jitter_records(512, light, color_jitter_rng(light, 3))
    assert (f == 1.0).all()
    assert np.array_equal(o, o_full) and np.array_equal(a, a_full)
    # M = I and K = 0 exactly: only the lighting remains
    assert np.array_equal(rec[:, :9], np.tile(np.eye(3, dtype=np.float32).reshape(1, 9), (512, 1)))
    assert (rec[:, 9:18] == 0).all()
    nolight = check_color_jitter({"brightness": 0.4, "seed": 9})
    rec2, f2, _, _ = color_jitter_records(512, nolight, color_jitter_rng(nolight, 3))
    assert np.array_equal(f2[:, 0], f_full[:, 0]) and (f2[:, 1:] == 1.0).all() and (rec2[:, 18:] == 0).all()


def test_same_key_same_records_other_rank_other_records():
    cfg = check_color_jitter(dict(ALL4, seed=7))
    a = color_jitter_records(128, cfg, color_jitter_rng(cfg, 0))[0]
    b = color_jitter_records(128, cfg, color_jitter_rng(cfg, 1))[0]
    c = color_jitter_records(128, cfg, color_jitter_rng(cfg, 0))[0]
    assert np.array_equal(a, c) and not np.array_equal(a, b)


# --------------------------------------------------------------------------- the reference
def _batch(N=6, H=40, W=48, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)
    means = {0: torch.tensor([127.5]), 1: torch.tensor([123.7, 116.3, 103.5]), 2: torch.rand(H, W, 3, generator=g) * 255}
    return x, means


def _records(n, seed=0, cfg=ALL4):
    cfg = check_color_jitter(dict(cfg, seed=seed))
    return color_jitter_records(n, cfg, color_jitter_rng(cfg, 0))


@pytest.mark.parametrize("resized", [False, True])
@pytest.mark.parametrize("mean_mode", [0, 1, 2])
@pytest.mark.parametrize("cscale", [False, True])
def test_reference_matches_the_oracle(resized, mean_mode, cscale):
    """fp32 torch against the float64 sequential oracle.  The bound is the fp32 arithmetic (2^-18·(|want| + S)) plus the resample's
    coordinate: ``F.interpolate`` on the CPU may round the source coordinate s once more than the oracle, which moves λ by up to
    2^-22·L and v̂ by that × 255."""
    x, means = _batch(seed=mean_mode)
    N, H, W = x.shape[:3]
    out_hw = (20, 24)
    if resized:
        boxes = np.concatenate([np.int32([[0, 0, H, W], [3, 5, 1, 1], [H - 7, W - 9, 7, 9]]),
                                draw_resized_crops(N - 3, (H, W), (0.08, 1.0), (0.75, 4 / 3), np.random.default_rng(mean_mode))[0]])
    else:
        boxes = np.int32([[(H - 20) // 2, (W - 24) // 2, 20, 24]] * N) + np.int32([[i % 3, i % 5, 0, 0] for i in range(N)])
    flips = np.uint8([i % 2 for i in range(N)])
    rec, fac, order, alpha = _records(N, seed=mean_mode)
    mean = means[mean_mode]
    sc = torch.from_numpy(1.0 / 255.0 / np.float32([0.229, 0.224, 0.225])) if cscale else 1.0 / 255.0
    got = ref.color_crop_mirror_normalize(x, mean, sc, out_hw, boxes, flips, rec).numpy()
    sc64 = sc.double().numpy() if cscale else sc
    want, S = co.oracle(x.numpy(), mean.double().numpy(), sc64, out_hw, boxes, flips, fac, order, alpha, rec)
    row = np.abs(rec[:, :9]).reshape(N, 3, 3).sum(2) + np.abs(rec[:, 9:18]).reshape(N, 3, 3).sum(2)     # |M|𝟙 + |K|𝟙 per channel
    dv = 2.0 ** -22 * max(H, W) * 255.0
    extra = (row[:, None, None, :] * dv + (dv if mean_mode == 2 else 0.0)) * np.broadcast_to(np.asarray(sc64), (3,))
    err = np.abs(got - want)
    assert (err <= 2.0 ** -18 * (np.abs(want) + S) + extra).all(), err.max()


def test_reference_with_the_identity_record_is_the_crop_reference():
    x, means = _batch(seed=3)
    N, H, W = x.shape[:3]
    offs = np.int32([[i, 2 * i] for i in range(N)])
    boxes = np.concatenate([offs, np.int32([[20, 24]] * N)], 1)
    flips = np.uint8([1, 0, 1, 1, 0, 0])
    ident = np.zeros((N, 24), np.float32)
    ident[:, [0, 4, 8]] = 1.0
    cs = torch.from_numpy(1.0 / 255.0 / np.float32([0.229, 0.224, 0.225]))
    for m in means.values():
        a = ref.color_crop_mirror_normalize(x, m, cs, (20, 24), boxes, flips, ident)
        b = ref.crop_mirror_normalize(x, m, cs, (20, 24), torch.from_numpy(offs), torch.from_numpy(flips))
        torch.testing.assert_close(a, b, rtol=2e-7, atol=1e-6)


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


@pytest.mark.parametrize("rrc", [None, {"scale": [0.1, 1.0], "seed": 5}])
def test_cpu_loader_train_batches_are_the_reference_of_their_draw(rrc):
    """Boxes and flips (or fixed-crop offsets) are exactly those drawn without the key; the batch is the reference of the records."""
    cj = check_color_jitter(dict(ALL4, seed=2))
    rrc = check_resized_crop(rrc) if rrc is not None else None
    d = _data()
    ld = d.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, resized_crop=rrc, rank=2, color_jitter=cj)
    d0 = _data()
    ld0 = d0.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, resized_crop=rrc, rank=2)
    rng = color_jitter_rng(cj, 2)
    mean, cs = torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5])
    rs = np.random.RandomState(1234)
    rrc_rng = resized_crop_rng(rrc, 2) if rrc is not None else None
    for L in (ld, ld0):
        L.request(d.train_img[0], "train")
    for k in range(1, 4):
        for L in (ld, ld0):
            L.request(d.train_img[k % 3], "train")
        b, b0 = ld.get(), ld0.get()
        rec = color_jitter_records(8, cj, rng)[0]
        assert np.array_equal(b.records, rec)
        if rrc is not None:
            boxes, flips = draw_resized_crops(8, (32, 32), rrc["scale"], rrc["ratio"], rrc_rng)
            assert np.array_equal(b0.boxes, boxes) and np.array_equal(b0.flips, flips)
        else:
            offs, flips = draw_crops(8, (32, 32), (20, 24), "train", True, False, rs)
            boxes = np.concatenate([offs, np.int32([[20, 24]] * 8)], 1)
            assert b0.boxes is None
        assert np.array_equal(b.boxes, boxes) and np.array_equal(b.flips, flips)
        want = ref.color_crop_mirror_normalize(_raw(d, b.item), mean, cs, (20, 24), boxes, flips, rec)
        assert tuple(b.x.shape) == (8, 20, 24, 3) and torch.equal(b.x, want)
        assert b.h2d_bytes == 8 * 32 * 32 * 3 + 8 * 17 + 8 * 96
    for L, dd in ((ld, d), (ld0, d0)):
        L.drain(); dd.para_load_close()


def test_cpu_loader_val_batches_are_unchanged():
    outs = []
    for cj in (None, check_color_jitter(ALL4)):
        d = _data()
        ld = d.para_load_init("cpu", 24, 24, rand_crop=True, batch_crop_mirror=False, color_jitter=cj)
        seq = []
        for mode in ("val", "train", "val"):
            ld.request(d.train_img[0], mode); ld.request(d.train_img[1], mode)
            for _ in range(2):
                b = ld.get()
                if mode == "val":
                    seq.append(b.x.clone())
                    assert b.records is None and b.h2d_bytes == 8 * 32 * 32 * 3 + 8 * 9
            ld.drain()
        d.para_load_close()
        outs.append(seq)
    assert all(torch.equal(a, b) for a, b in zip(*outs))


@pytest.mark.parametrize("rrc", [None, {"scale": [0.3, 0.6], "seed": 11}])
def test_serial_load_batch_applies_it(rrc):
    from theanompi_b200.models.alex_net import AlexNet
    cj = dict(ALL4, seed=4)
    m = _build(AlexNet, color_jitter=cj, random_resized_crop=rrc, **IMG)
    item = m.data.train_img_shard[0]
    np.random.seed(77)
    x = m.data.load_batch(item, "train", m)
    raw = np.empty((4, 256, 256, 3), np.uint8)
    src = m.data.read(item, raw)
    raw = torch.from_numpy(src.numpy() if src is not None else raw)
    if rrc is not None:
        vr = check_resized_crop(rrc)
        boxes, flips = draw_resized_crops(4, (256, 256), vr["scale"], vr["ratio"], resized_crop_rng(vr, 0))
    else:
        np.random.seed(77)                                   # the serial path's crops come from the global RandomState
        offs, flips = draw_crops(4, (256, 256), (227, 227), "train", True, False)
        boxes = np.concatenate([offs, np.int32([[227, 227]] * 4)], 1)
    vc = check_color_jitter(cj)
    rec = color_jitter_records(4, vc, color_jitter_rng(vc, 0))[0]
    want = ref.color_crop_mirror_normalize(raw, torch.from_numpy(m.data.rawdata[4]), torch.from_numpy(1.0 / 255.0 / m.data.rawdata[5]),
                                           (227, 227), boxes, flips, rec)
    assert tuple(x.shape) == (4, 227, 227, 3) and torch.equal(x, want)
    # validation keeps the centre crop, unjittered
    v = m.data.load_batch(item, "val", m)
    want_v = ((raw.numpy().astype(np.float32) - m.data.rawdata[4]) / 255.0 / m.data.rawdata[5])[:, 14:241, 14:241]
    assert torch.equal(v, torch.from_numpy(np.ascontiguousarray(want_v)))


def test_serial_path_without_the_key_keeps_its_stream():
    """Without the key the serial path draws its crops from the global RandomState and normalises before cropping, as before."""
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.data.utils import crop_and_mirror
    m = _build(AlexNet, **IMG)
    item = m.data.train_img_shard[0]
    np.random.seed(5)
    x = m.data.load_batch(item, "train", m)
    raw = np.empty((4, 256, 256, 3), np.uint8)
    src = m.data.read(item, raw)
    raw = src.numpy() if src is not None else raw
    np.random.seed(5)
    want = crop_and_mirror((raw.astype(np.float32) - m.data.rawdata[4]) / 255.0 / m.data.rawdata[5], "train", True, False, 227)
    assert torch.equal(x, torch.from_numpy(want))


def test_tiny_models_train_with_it_on_the_cpu():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    from theanompi_b200.utils.recorder import Recorder
    for cls, kw in ((AlexNet, dict(color_jitter={"lighting": 0.1})),
                    (ResNet50, dict(blocks=(1, 1, 1, 1), color_jitter=ALL4, random_resized_crop={}))):
        m = _build(cls, **dict(IMG, **kw))
        m.compile_iter_fns("avg")
        rec = Recorder(None, 10 ** 6, cls.__name__, False, device="cpu")
        for i in range(2):
            m.train_iter(i, rec)
        m.reset_iter("val")
        m.val_iter(0, rec)
        assert all(np.isfinite(float(c)) for c in rec.train_info["cost"]) and np.isfinite(float(rec.val_info["cost"][-1]))
