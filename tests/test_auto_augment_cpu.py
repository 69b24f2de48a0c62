"""TrivialAugmentWide / RandAugment (config['auto_augment']) on the CPU: the key's validation and the models that refuse it, the
magnitude tables against torchvision's ``_AUGMENTATION_SPACE``, the draw's statistics and independence, the torch reference per op
against torchvision's own op code (tests/auto_augment_oracle.py) on random images and edge cases, and the CPU loader and serial path."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import auto_augment_oracle as oracle  # noqa: E402
from test_color_jitter_cpu import ALL4, IMG, _build, _data, _raw, _refused  # noqa: E402
from theanompi_b200.models.data.utils import (AA_KEY, AA_OPS, auto_augment_records, auto_augment_rng, auto_augment_space,  # noqa: E402
                                              check_auto_augment, check_resized_crop, draw_crops, draw_resized_crops,
                                              resized_crop_rng)
from theanompi_b200.ops import reference as ref  # noqa: E402


# --------------------------------------------------------------------------- configuration
def test_defaults_and_json_round_trip():
    assert check_auto_augment(None) is None
    assert check_auto_augment({}) == {"policy": "trivial_wide", "num_magnitude_bins": 31, "seed": 0}
    assert check_auto_augment({"policy": "rand"}) == {"policy": "rand", "num_magnitude_bins": 31, "num_ops": 2, "magnitude": 9, "seed": 0}
    cfg = {"policy": "rand", "num_ops": 4, "magnitude": 0, "num_magnitude_bins": 2, "seed": np.int64(-1)}
    got = check_auto_augment(json.loads(json.dumps({AA_KEY: dict(cfg, seed=5)}))[AA_KEY])
    assert got == dict(cfg, seed=5) and check_auto_augment(cfg)["seed"] == 2 ** 64 - 1


@pytest.mark.parametrize("bad", [
    "rand", ["policy"], {"policy": "auto"}, {"policy": None}, {"level": 1}, {"num_ops": 2}, {"magnitude": 9},
    {"policy": "rand", "num_ops": 0}, {"policy": "rand", "num_ops": 5}, {"policy": "rand", "num_ops": True},
    {"policy": "rand", "num_ops": 2.0}, {"policy": "rand", "magnitude": -1}, {"policy": "rand", "magnitude": 31},
    {"policy": "rand", "magnitude": 3, "num_magnitude_bins": 3}, {"policy": "rand", "magnitude": "9"}, {"num_magnitude_bins": 1},
    {"num_magnitude_bins": 31.0}, {"num_magnitude_bins": False}, {"seed": 1.5}, {"seed": True}, {"seed": None}])
def test_malformed_config_is_a_value_error_naming_the_key(bad):
    from theanompi_b200.models.alex_net import AlexNet
    with pytest.raises(ValueError, match=AA_KEY):
        check_auto_augment(bad)
    with pytest.raises(ValueError, match=AA_KEY):
        _build(AlexNet, auto_augment=bad, **IMG)


def test_models_refuse_it_or_accept_it_and_color_jitter_is_refused_with_it():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50, ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    for cls, kw in _refused():
        with pytest.raises(ValueError, match=AA_KEY + " is not supported"):
            _build(cls, auto_augment={}, **kw)
    m = _build(ResNet50, auto_augment={"policy": "rand"}, random_resized_crop={}, random_erasing={}, blocks=(1, 1, 1, 1), **IMG)
    assert m.auto_augment["policy"] == "rand"
    with pytest.raises(ValueError, match=AA_KEY + " and color_jitter"):
        _build(AlexNet, auto_augment={}, color_jitter=ALL4, **IMG)
    for cls in (GoogLeNet, VGG16, ResNet152, ResNet50Torch):
        assert cls.supports_resized_crop is True and cls.check_auto_augment is AlexNet.check_auto_augment


# --------------------------------------------------------------------------- tables and draw
@pytest.mark.parametrize("policy", ["trivial_wide", "rand"])
@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227)])
def test_magnitude_tables_are_torchvisions(policy, out_hw):
    want = oracle.torchvision_space(policy, 31, out_hw)
    got = auto_augment_space(policy, 31, out_hw)
    assert tuple(want) == AA_OPS == tuple(got)
    for k in AA_OPS:
        assert got[k][1] == want[k][1], k
        assert (got[k][0] is None) == (want[k][0] is None), k
        if got[k][0] is not None:
            assert np.array_equal(got[k][0], want[k][0]), k


def test_draw_statistics():
    from scipy import stats
    n = 60000
    cfg = check_auto_augment({"seed": 3})
    rec, op, mag = auto_augment_records(n, cfg, auto_augment_rng(cfg, 0), (224, 224))
    assert rec.shape == (n, 1, 12) and rec.dtype == np.float32
    assert stats.chisquare(np.bincount(op.ravel(), minlength=14)).pvalue > 1e-4
    table = auto_augment_space("trivial_wide", 31, (224, 224))["Rotate"][0]
    rot = np.abs(mag[op == 5])
    bins = np.searchsorted(table, rot - 1e-9)
    assert stats.chisquare(np.bincount(bins, minlength=31)).pvalue > 1e-4
    signed = (op >= 1) & (op <= 9) & (mag != 0)
    assert stats.binomtest(int((mag[signed] < 0).sum()), int(signed.sum()), 0.5).pvalue > 1e-4
    r = check_auto_augment({"policy": "rand", "num_ops": 3, "magnitude": 30, "seed": 3})
    rec, op, mag = auto_augment_records(n // 10, r, auto_augment_rng(r, 0), (224, 224))
    assert rec.shape == (n // 10, 3, 12)
    assert np.allclose(np.abs(mag[op == 5]), 30.0) and np.allclose(np.abs(mag[op == 3]), 150.0 / 331.0 * 224, rtol=1e-6)


def test_ranks_draw_apart_and_a_key_reproduces():
    cfg = check_auto_augment({"seed": 4})
    a = auto_augment_records(64, cfg, auto_augment_rng(cfg, 0), (224, 224))[0]
    assert np.array_equal(a, auto_augment_records(64, cfg, auto_augment_rng(cfg, 0), (224, 224))[0])
    assert not np.array_equal(a, auto_augment_records(64, cfg, auto_augment_rng(cfg, 1), (224, 224))[0])


# --------------------------------------------------------------------------- the reference against torchvision
def _record(name, m, hw=(40, 48)):
    """The record the host draw composes for op ``name`` at signed magnitude m: the draw with that op's table set to |m|."""
    from theanompi_b200.models.data import utils
    cfg = check_auto_augment({"seed": 0})
    space = utils.auto_augment_space
    try:
        utils.auto_augment_space = lambda p, nb, hw_: {kk: (np.full(nb, abs(m)) if kk == name else v[0], v[1])
                                                        for kk, v in space(p, nb, hw_).items()}
        rec, op, mag = auto_augment_records(2000, cfg, np.random.default_rng(0), hw)
    finally:
        utils.auto_augment_space = space
    k = np.flatnonzero((op[:, 0] == AA_OPS.index(name)) & ((np.sign(mag[:, 0]) == np.sign(m)) | (m == 0)))[0]
    return rec[k, 0], float(mag[k, 0])


@pytest.mark.parametrize("hw", [(40, 48), (224, 224), (2, 2), (3, 3)])
def test_reference_matches_torchvision_per_op_on_random_images(hw):
    cfg = check_auto_augment({"seed": hw[0]})
    rec, op, mag = auto_augment_records(300, cfg, auto_augment_rng(cfg, 0), hw)
    g = torch.Generator().manual_seed(hw[1])
    seen = set()
    for k in range(300):
        img = torch.randint(0, 256, (3,) + hw, dtype=torch.uint8, generator=g)
        want = oracle.torchvision_op(img, AA_OPS[op[k, 0]], mag[k, 0])
        assert torch.equal(ref.aa_apply_op(img, rec[k, 0]), want), (AA_OPS[op[k, 0]], mag[k, 0])
        seen.add(int(op[k, 0]))
    assert seen == set(range(14))


@pytest.mark.parametrize("name,m,img", [
    ("AutoContrast", 0.0, "constant"), ("Equalize", 0.0, "constant"), ("Equalize", 0.0, "two"), ("Solarize", 100.0 / 255.0, "ramp"),
    ("Posterize", 8.0, "random"), ("Posterize", 2.0, "random"), ("ShearX", -0.99, "random"), ("ShearY", -0.3, "random"),
    ("TranslateX", -32.0, "random"), ("TranslateY", -17.9, "random"), ("Rotate", 135.0, "random"), ("Rotate", -135.0, "random"),
    ("Sharpness", 0.99, "random"), ("Sharpness", -0.99, "random"), ("Brightness", -0.99, "random"), ("Color", 0.99, "random"),
    ("Contrast", -0.99, "random")])
def test_reference_matches_torchvision_at_the_edges(name, m, img):
    from theanompi_b200.models.data.utils import AA_RECORD_FLOATS, inverse_affine_matrix  # noqa: F401
    hw = (40, 48)
    g = torch.Generator().manual_seed(7)
    x = {"constant": torch.full((3,) + hw, 77, dtype=torch.uint8), "ramp": torch.arange(3 * 40 * 48).remainder(256).to(torch.uint8).view(3, *hw),
         "two": torch.where(torch.rand((3,) + hw, generator=g) < 0.998, 10, 200).to(torch.uint8),
         "random": torch.randint(0, 256, (3,) + hw, dtype=torch.uint8, generator=g)}[img]
    rec, mag = _record(name, m, hw)
    assert np.isclose(mag, m, rtol=1e-6)
    assert torch.equal(ref.aa_apply_op(x, rec), oracle.torchvision_op(x, name, mag)), name
    if name == "Solarize":
        assert (x == 100).any()                                   # a value exactly at the threshold
    if img == "constant":
        assert torch.equal(ref.aa_apply_op(x, rec), x)


@pytest.mark.parametrize("hw", [(2, 2), (3, 3)])
def test_sharpness_on_tiny_images(hw):
    g = torch.Generator().manual_seed(1)
    x = torch.randint(0, 256, (3,) + hw, dtype=torch.uint8, generator=g)
    rec, mag = _record("Sharpness", 0.7, hw)
    assert torch.equal(ref.aa_apply_op(x, rec), oracle.torchvision_op(x, "Sharpness", mag))


def test_crop_reference_is_the_rounded_resample():
    g = torch.Generator().manual_seed(2)
    x = torch.randint(0, 256, (3, 32, 32, 3), dtype=torch.uint8, generator=g)
    boxes = np.int32([[0, 0, 20, 24], [3, 5, 29, 17], [4, 4, 24, 24]])
    u = ref.aa_crop_u8(x, (20, 24), boxes, np.uint8([0, 1, 0]))
    assert torch.equal(u[0], x[0, :20, :24]) and torch.equal(u[1], u[1])
    want = ref.resized_crop_mirror_normalize(x, torch.zeros(1), 1.0, (20, 24), boxes, np.uint8([0, 1, 0]))
    assert torch.equal(u, want.round().to(torch.uint8))


# --------------------------------------------------------------------------- loader and serial path
@pytest.mark.parametrize("policy,rrc", [("trivial_wide", None), ("rand", {"scale": [0.1, 1.0], "seed": 5})])
def test_cpu_loader_train_batches_are_the_reference_of_their_draw(policy, rrc):
    aa = check_auto_augment({"policy": policy, "seed": 2})
    rrc = check_resized_crop(rrc) if rrc is not None else None
    d, d0 = _data(), _data()
    ld = d.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, resized_crop=rrc, rank=2, auto_augment=aa)
    ld0 = d0.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, resized_crop=rrc, rank=2)
    rng, rs = auto_augment_rng(aa, 2), np.random.RandomState(1234)
    rrc_rng = resized_crop_rng(rrc, 2) if rrc is not None else None
    mean, cs = torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5])
    for L in (ld, ld0):
        L.request(d.train_img[0], "train")
    for k in range(1, 3):
        for L in (ld, ld0):
            L.request(d.train_img[k % 3], "train")
        b, b0 = ld.get(), ld0.get()
        rec = auto_augment_records(8, aa, rng, (20, 24))[0]
        assert np.array_equal(b.aa_records, rec)
        if rrc is not None:
            boxes, flips = draw_resized_crops(8, (32, 32), rrc["scale"], rrc["ratio"], rrc_rng)
            assert np.array_equal(b0.boxes, boxes)
        else:
            offs, flips = draw_crops(8, (32, 32), (20, 24), "train", True, False, rs)
            boxes = np.concatenate([offs, np.int32([[20, 24]] * 8)], 1)
        assert np.array_equal(b.boxes, boxes) and np.array_equal(b.flips, flips)
        want = ref.auto_augment_crop_normalize(_raw(d, b.item), mean, cs, (20, 24), boxes, flips, rec)
        assert torch.equal(b.x, want)
    for L, dd in ((ld, d), (ld0, d0)):
        L.drain(); dd.para_load_close()


def test_val_batches_and_runs_without_the_key_are_unchanged():
    outs = []
    for aa in (None, check_auto_augment({})):
        d = _data()
        ld = d.para_load_init("cpu", 24, 24, rand_crop=True, batch_crop_mirror=False, auto_augment=aa)
        ld.request(d.train_img[0], "train"); ld.request(d.train_img[1], "val")
        ld.get()
        b = ld.get()
        assert b.aa_records is None
        outs.append(b.x.clone())
        ld.drain(); d.para_load_close()
    assert torch.equal(*outs)


def test_serial_load_batch_applies_it_and_tiny_models_train():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    from theanompi_b200.utils.recorder import Recorder
    m = _build(AlexNet, auto_augment={"seed": 4}, random_erasing={"p": 0.5}, **IMG)
    item = m.data.train_img_shard[0]
    np.random.seed(77)
    x = m.data.load_batch(item, "train", m)
    raw = np.empty((4, 256, 256, 3), np.uint8)
    src = m.data.read(item, raw)
    raw = torch.from_numpy(src.numpy() if src is not None else raw)
    np.random.seed(77)
    offs, flips = draw_crops(4, (256, 256), (227, 227), "train", True, False)
    boxes = np.concatenate([offs, np.int32([[227, 227]] * 4)], 1)
    va = check_auto_augment({"seed": 4})
    rec = auto_augment_records(4, va, auto_augment_rng(va, 0), (227, 227))[0]
    from theanompi_b200.models.data.utils import check_random_erasing, draw_erase_boxes, random_erasing_rng
    vr = check_random_erasing({"p": 0.5})
    want = ref.auto_augment_crop_normalize(raw, torch.from_numpy(m.data.rawdata[4]), torch.from_numpy(1.0 / 255.0 / m.data.rawdata[5]),
                                           (227, 227), boxes, flips, rec)
    want = ref.random_erase(want, draw_erase_boxes(4, (227, 227), vr, random_erasing_rng(vr, 0)))
    assert torch.equal(x, want)
    for cls, kw in ((AlexNet, dict(auto_augment={})),
                    (ResNet50, dict(blocks=(1, 1, 1, 1), auto_augment={"policy": "rand"}, random_resized_crop={}, random_erasing={}))):
        mm = _build(cls, **dict(IMG, **kw))
        mm.compile_iter_fns("avg")
        r = Recorder(None, 10 ** 6, cls.__name__, False, device="cpu")
        for i in range(2):
            mm.train_iter(i, r)
        assert all(np.isfinite(float(c)) for c in r.train_info["cost"])
