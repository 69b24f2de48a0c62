"""Random erasing (config['random_erasing']) on the CPU: the validation of the key and the models that refuse it, the erase-box draw
against torchvision's ``RandomErasing`` (distributions, probability, reproducibility, independence of the crop and colour draws), the
torch reference against ``torchvision.transforms.v2.functional.erase``, and the CPU ParaLoader and the serial load_batch path with
the key over every crop path."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_color_jitter_cpu import ALL4, IMG, _build, _data, _raw, _refused  # noqa: E402
from theanompi_b200.models.data.utils import (RE_KEY, check_color_jitter, check_random_erasing, check_resized_crop,  # noqa: E402
                                              color_jitter_records, color_jitter_rng, draw_crops, draw_erase_boxes, draw_resized_crops,
                                              random_erasing_rng, resized_crop_rng)
from theanompi_b200.ops import reference as ref  # noqa: E402

DEFAULTS = {"p": 0.5, "scale": (0.02, 0.33), "ratio": (0.3, 3.3), "seed": 0}


# --------------------------------------------------------------------------- configuration
def test_defaults_and_json_round_trip():
    assert check_random_erasing(None) is None
    assert check_random_erasing({}) == DEFAULTS
    cfg = {"p": 0.1, "scale": [0.05, 0.2], "ratio": [0.5, 2], "seed": np.int64(-1)}
    want = {"p": 0.1, "scale": (0.05, 0.2), "ratio": (0.5, 2.0), "seed": 2 ** 64 - 1}
    assert check_random_erasing(cfg) == want
    assert check_random_erasing(json.loads(json.dumps({RE_KEY: dict(cfg, seed=7)}))[RE_KEY]) == dict(want, seed=7)
    assert check_random_erasing({"p": 1, "scale": (1, 1)}) == dict(DEFAULTS, p=1.0, scale=(1.0, 1.0))
    assert check_random_erasing({"p": np.float32(0.0)})["p"] == 0.0


@pytest.mark.parametrize("bad", [
    0.5, [0.5], "p", {"value": 0}, {"value": "random"}, {"P": 0.5}, {"p": True}, {"p": None}, {"p": "0.5"}, {"p": float("nan")},
    {"p": -0.01}, {"p": 1.5}, {"scale": 0.3}, {"scale": [0.1]}, {"scale": [0.1, 0.2, 0.3]}, {"scale": [0.0, 0.3]}, {"scale": [0.4, 0.3]},
    {"scale": [0.1, 1.2]}, {"scale": [0.1, float("inf")]}, {"scale": [True, 0.3]}, {"ratio": [0.0, 3.3]}, {"ratio": [3.3, 0.3]},
    {"ratio": [-1, 3.3]}, {"ratio": "wide"}, {"seed": 1.0}, {"seed": True}, {"seed": "0"}, {"seed": None}])
def test_malformed_config_is_a_value_error_naming_the_key(bad):
    from theanompi_b200.models.alex_net import AlexNet
    with pytest.raises(ValueError, match=RE_KEY):
        check_random_erasing(bad)
    with pytest.raises(ValueError, match=RE_KEY):
        _build(AlexNet, random_erasing=bad, **IMG)


def test_models_without_the_imagenet_loader_refuse_it():
    for cls, kw in _refused():
        with pytest.raises(ValueError, match=RE_KEY + " is not supported"):
            _build(cls, random_erasing={"p": 0.1}, **kw)


def test_supporting_models_and_every_crop_path():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50, ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    m = _build(ResNet50, random_erasing={"p": 0.25, "seed": 3}, color_jitter=ALL4, random_resized_crop={}, blocks=(1, 1, 1, 1), **IMG)
    assert m.random_erasing == dict(DEFAULTS, p=0.25, seed=3)
    assert _build(ResNet50, blocks=(1, 1, 1, 1), **IMG).random_erasing is None
    for flag in ("batch_crop_mirror", "rand_crop"):
        cls = type("AlexNetFixed", (AlexNet,), {flag: flag == "batch_crop_mirror"})
        assert _build(cls, random_erasing={}, **IMG).random_erasing == DEFAULTS
    # the constructors of the other supporting models (heavier to build) take the same path through ModelBase
    for cls in (GoogLeNet, VGG16, ResNet152, ResNet50Torch):
        assert cls.supports_resized_crop is True and cls.check_random_erasing is AlexNet.check_random_erasing


# --------------------------------------------------------------------------- the draw
def _torchvision_boxes(n, out_hw, cfg, seed):
    """(i, j, h, w) as torchvision's RandomErasing draws them, (0, 0, 0, 0) when it erases nothing."""
    T = pytest.importorskip("torchvision.transforms")
    torch.manual_seed(seed)
    img = torch.empty(3, *out_hw)
    out = np.zeros((n, 4), np.int64)
    for k in range(n):
        if torch.rand(1) < cfg["p"]:
            i, j, h, w, v = T.RandomErasing.get_params(img, scale=cfg["scale"], ratio=cfg["ratio"], value=[0])
            if v is not img:
                out[k] = (i, j, h, w)
    return out


@pytest.mark.parametrize("out_hw,cfg", [((224, 224), {}), ((227, 227), {"p": 0.25}),
                                        ((160, 288), {"p": 0.8, "scale": [0.3, 0.9], "ratio": [0.2, 5.0]})])
def test_draw_matches_torchvision_in_distribution(out_hw, cfg):
    from scipy import stats
    cfg = check_random_erasing(dict(cfg, seed=5))
    n = 20000
    got = draw_erase_boxes(n, out_hw, cfg, random_erasing_rng(cfg, 0))
    want = _torchvision_boxes(n, out_hw, cfg, 5)
    H, W = out_hw
    assert got.dtype == np.int32 and got.shape == (n, 4)
    on_g, on_w = got[:, 2] > 0, want[:, 2] > 0
    assert np.all((got[:, 0] >= 0) & (got[:, 1] >= 0) & (got[:, 0] + got[:, 2] <= H) & (got[:, 1] + got[:, 3] <= W))
    assert np.all(got[~on_g] == 0) and np.all((got[on_g, 2] < H) & (got[on_g, 3] < W))
    # the erased share: the two are binomial draws with the same probability
    assert stats.binomtest(int(on_g.sum()), n, on_w.mean() if 0 < on_w.mean() < 1 else cfg["p"]).pvalue > 1e-4
    for col in (2, 3):                                       # h and w
        assert stats.ks_2samp(got[on_g, col], want[on_w, col]).pvalue > 1e-4, col
    # the position is uniform over what fits
    jitter = np.random.default_rng(0)
    for col, L in ((0, H), (1, W)):
        u = (got[on_g, col] + jitter.random(int(on_g.sum()))) / (L - got[on_g, col + 2] + 1)
        assert stats.kstest(u, "uniform").pvalue > 1e-4, col


def test_draw_is_torchvisions_rounding_of_each_attempt():
    """Replaying the generator: h = round(√(a·r)), w = round(√(a/r)), the first attempt with h < H and w < W, erased when U < p."""
    cfg = check_random_erasing({"p": 0.7, "scale": [0.2, 0.9], "ratio": [0.3, 3.3], "seed": 9})
    n, H, W = 4000, 30, 20
    got = draw_erase_boxes(n, (H, W), cfg, random_erasing_rng(cfg, 1))
    rng = random_erasing_rng(cfg, 1)
    u = rng.random(n)
    area = H * W * rng.uniform(0.2, 0.9, (n, 10))
    r = np.exp(rng.uniform(np.log(0.3), np.log(3.3), (n, 10)))
    fell_through = 0
    for k in range(n):
        hw = [(int(round(np.sqrt(a * q))), int(round(np.sqrt(a / q)))) for a, q in zip(area[k], r[k])]
        fit = [t for t in hw if t[0] < H and t[1] < W]
        if u[k] < 0.7 and fit:
            assert tuple(got[k, 2:]) == fit[0], k
        else:
            fell_through += bool(u[k] < 0.7)
            assert tuple(got[k]) == (0, 0, 0, 0), k
    assert fell_through > 0                                   # this configuration exercises the no-fit case


def test_same_key_same_boxes_other_rank_or_seed_other_boxes():
    cfg = check_random_erasing({"seed": 4})
    a = draw_erase_boxes(64, (224, 224), cfg, random_erasing_rng(cfg, 0))
    assert np.array_equal(a, draw_erase_boxes(64, (224, 224), cfg, random_erasing_rng(cfg, 0)))
    assert not np.array_equal(a, draw_erase_boxes(64, (224, 224), cfg, random_erasing_rng(cfg, 1)))
    cfg5 = check_random_erasing({"seed": 5})
    assert not np.array_equal(a, draw_erase_boxes(64, (224, 224), cfg5, random_erasing_rng(cfg5, 0)))
    # p changes which images are erased, not the stream
    c0, c1 = check_random_erasing({"p": 0.0, "seed": 4}), check_random_erasing({"p": 1.0, "seed": 4})
    assert not draw_erase_boxes(64, (224, 224), c0, random_erasing_rng(c0, 0)).any()
    full = draw_erase_boxes(64, (224, 224), c1, random_erasing_rng(c1, 0))
    on = a[:, 2] > 0
    assert np.array_equal(a[on], full[on])


# --------------------------------------------------------------------------- the reference
def test_reference_matches_torchvision_erase():
    F = pytest.importorskip("torchvision.transforms.v2.functional")
    g = torch.Generator().manual_seed(0)
    x = torch.randn(6, 20, 24, 3, generator=g)
    boxes = np.int32([[0, 0, 0, 0], [0, 0, 19, 23], [3, 5, 7, 2], [19, 23, 1, 1], [10, 0, 10, 24], [4, 6, 0, 9]])
    got = ref.random_erase(x, boxes)
    assert not torch.equal(got, x)
    for n, (i, j, h, w) in enumerate(boxes):
        want = F.erase(x[n].permute(2, 0, 1), int(i), int(j), int(h), int(w), torch.tensor([0.0])[:, None, None]).permute(1, 2, 0)
        assert torch.equal(got[n], want), n
    assert torch.equal(ref.random_erase(x.to(torch.bfloat16), boxes), got.to(torch.bfloat16))
    with pytest.raises(ValueError, match="random_erase"):
        ref.random_erase(x, np.int32([[15, 0, 6, 4]] * 6))


# --------------------------------------------------------------------------- loader
@pytest.mark.parametrize("crop", ["fixed", "resized", "color", "resized+color"])
def test_cpu_loader_train_batches_are_the_reference_of_their_draw(crop):
    """The batch is the batch of a loader without the key (same crops, same colour records), erased in the recorded boxes."""
    re = check_random_erasing({"p": 0.6, "seed": 8})
    rrc = check_resized_crop({"scale": [0.1, 1.0], "seed": 5}) if "resized" in crop else None
    cj = check_color_jitter(dict(ALL4, seed=2)) if "color" in crop else None
    kw = dict(rand_crop=True, batch_crop_mirror=False, resized_crop=rrc, rank=2, color_jitter=cj)
    d, d0 = _data(), _data()
    ld = d.para_load_init("cpu", 24, 20, random_erasing=re, **kw)
    ld0 = d0.para_load_init("cpu", 24, 20, **kw)
    rng = random_erasing_rng(re, 2)
    for L in (ld, ld0):
        L.request(d.train_img[0], "train")
    erased = 0
    for k in range(1, 5):
        for L in (ld, ld0):
            L.request(d.train_img[k % 3], "train")
        b, b0 = ld.get(), ld0.get()
        boxes = draw_erase_boxes(8, (20, 24), re, rng)
        assert np.array_equal(b.erase, boxes) and b0.erase is None
        for a in ("boxes", "flips", "records"):
            assert (getattr(b, a) is None and getattr(b0, a) is None) or np.array_equal(getattr(b, a), getattr(b0, a)), a
        assert tuple(b.x.shape) == (8, 20, 24, 3) and torch.equal(b.x, ref.random_erase(b0.x, boxes))
        assert b.h2d_bytes == b0.h2d_bytes + 8 * 16
        erased += int((boxes[:, 2] > 0).sum())
    assert erased > 0
    for L, dd in ((ld, d), (ld0, d0)):
        L.drain(); dd.para_load_close()


def test_cpu_loader_val_batches_are_unchanged():
    outs = []
    for re in (None, check_random_erasing({"p": 1.0})):
        d = _data()
        ld = d.para_load_init("cpu", 24, 24, rand_crop=True, batch_crop_mirror=False, random_erasing=re)
        seq = []
        for mode in ("val", "train", "val"):
            ld.request(d.train_img[0], mode); ld.request(d.train_img[1], mode)
            for _ in range(2):
                b = ld.get()
                if mode == "val":
                    seq.append(b.x.clone())
                    assert b.erase is None and b.h2d_bytes == 8 * 32 * 32 * 3 + 8 * 9
            ld.drain()
        d.para_load_close()
        outs.append(seq)
    assert all(torch.equal(a, b) for a, b in zip(*outs))


@pytest.mark.parametrize("rrc,cj", [(None, None), ({"scale": [0.3, 0.6], "seed": 11}, None), (None, ALL4)])
def test_serial_load_batch_applies_it(rrc, cj):
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.data.utils import crop_and_mirror
    re = {"p": 0.9, "seed": 6}
    m = _build(AlexNet, random_erasing=re, random_resized_crop=rrc, color_jitter=cj, **IMG)
    item = m.data.train_img_shard[0]
    np.random.seed(77)
    x = m.data.load_batch(item, "train", m)
    raw = np.empty((4, 256, 256, 3), np.uint8)
    src = m.data.read(item, raw)
    raw = torch.from_numpy(src.numpy() if src is not None else raw)
    mean, cs = torch.from_numpy(m.data.rawdata[4]), torch.from_numpy(1.0 / 255.0 / m.data.rawdata[5])
    np.random.seed(77)                                       # the serial path's fixed crops come from the global RandomState
    if rrc is not None:
        vr = check_resized_crop(rrc)
        boxes, flips = draw_resized_crops(4, (256, 256), vr["scale"], vr["ratio"], resized_crop_rng(vr, 0))
        base = ref.resized_crop_mirror_normalize(raw, mean, cs, (227, 227), boxes, flips)
    elif cj is not None:
        offs, flips = draw_crops(4, (256, 256), (227, 227), "train", True, False)
        boxes = np.concatenate([offs, np.int32([[227, 227]] * 4)], 1)
        vc = check_color_jitter(cj)
        base = ref.color_crop_mirror_normalize(raw, mean, cs, (227, 227), boxes, flips, color_jitter_records(4, vc, color_jitter_rng(vc, 0))[0])
    else:
        base = torch.from_numpy(crop_and_mirror((raw.numpy().astype(np.float32) - m.data.rawdata[4]) / 255.0 / m.data.rawdata[5],
                                                "train", True, False, 227))
    vre = check_random_erasing(re)
    eb = draw_erase_boxes(4, (227, 227), vre, random_erasing_rng(vre, 0))
    assert (eb[:, 2] > 0).any()
    assert tuple(x.shape) == (4, 227, 227, 3) and torch.equal(x, ref.random_erase(base, eb))
    # validation keeps the centre crop, unerased
    v = m.data.load_batch(item, "val", m)
    want_v = ((raw.numpy().astype(np.float32) - m.data.rawdata[4]) / 255.0 / m.data.rawdata[5])[:, 14:241, 14:241]
    assert torch.equal(v, torch.from_numpy(np.ascontiguousarray(want_v)))


def test_tiny_models_train_with_it_on_the_cpu():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    from theanompi_b200.utils.recorder import Recorder
    for cls, kw in ((AlexNet, dict(random_erasing={"p": 0.5})),
                    (ResNet50, dict(blocks=(1, 1, 1, 1), random_erasing={}, color_jitter=ALL4, random_resized_crop={}))):
        m = _build(cls, **dict(IMG, **kw))
        m.compile_iter_fns("avg")
        rec = Recorder(None, 10 ** 6, cls.__name__, False, device="cpu")
        for i in range(2):
            m.train_iter(i, rec)
        m.reset_iter("val")
        m.val_iter(0, rec)
        assert all(np.isfinite(float(c)) for c in rec.train_info["cost"]) and np.isfinite(float(rec.val_info["cost"][-1]))
