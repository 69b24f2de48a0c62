"""AutoAugment and AugMix (config['auto_augment'] policies "autoaugment" and "augmix") and the ``interpolation`` key on the CPU: the
keys' validation, the sub-policy table and op spaces against torchvision v2, the draws' statistics and independence, the torch
reference against torchvision's own ``AutoAugment.forward`` / ``AugMix.forward`` replayed with the record's draws
(tests/augmix_oracle.py), bilinear ops, and the CPU loader and serial path."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import augmix_oracle as oracle  # noqa: E402
from test_color_jitter_cpu import ALL4, IMG, _build, _data, _raw, _refused  # noqa: E402
from theanompi_b200.models.data.utils import (AA_AUGMIX_OPS, AA_IMAGENET_POLICY, AA_INVERT, AA_KEY, AA_NONE, AA_OP_IDS,  # noqa: E402
                                              aa_bilinear, aa_slots, augmix_records, auto_augment_records, auto_augment_rng,
                                              auto_augment_space, check_auto_augment, check_random_erasing, check_resized_crop,
                                              draw_erase_boxes, draw_resized_crops, random_erasing_rng, resized_crop_rng)
from theanompi_b200.ops import reference as ref  # noqa: E402

NAMES = {v: k for k, v in AA_OP_IDS.items()}


# --------------------------------------------------------------------------- configuration
def test_defaults_interpolation_and_json_round_trip():
    assert check_auto_augment({"policy": "autoaugment"}) == {"policy": "autoaugment", "interpolation": "nearest", "seed": 0}
    want = {"policy": "augmix", "severity": 3, "mixture_width": 3, "chain_depth": -1, "alpha": 1.0, "all_ops": True,
            "interpolation": "bilinear", "seed": 0}
    assert check_auto_augment({"policy": "augmix"}) == want
    cfg = {"policy": "augmix", "severity": 10, "mixture_width": 4, "chain_depth": 2, "alpha": 16, "all_ops": False,
           "interpolation": "nearest", "seed": 7}
    assert check_auto_augment(json.loads(json.dumps({AA_KEY: cfg}))[AA_KEY]) == dict(cfg, alpha=16.0)
    # the existing policies keep their dicts unless the key is given, and their default stays nearest
    assert "interpolation" not in check_auto_augment({}) and not aa_bilinear(check_auto_augment({"policy": "rand"}))
    assert check_auto_augment({"interpolation": "bilinear"})["interpolation"] == "bilinear"
    assert aa_bilinear(check_auto_augment({"policy": "rand", "interpolation": "bilinear"}))
    assert aa_bilinear(check_auto_augment({"policy": "augmix"})) and not aa_bilinear(check_auto_augment({"policy": "autoaugment"}))
    assert [aa_slots(check_auto_augment(c)) for c in ({}, {"policy": "rand", "num_ops": 3}, {"policy": "autoaugment"},
                                                      {"policy": "augmix", "mixture_width": 2})] == [1, 3, 2, 6]


@pytest.mark.parametrize("bad,key", [
    ({"policy": "AutoAugment"}, "policy"), ({"interpolation": "bicubic"}, "interpolation"), ({"interpolation": 1}, "interpolation"),
    ({"policy": "autoaugment", "num_magnitude_bins": 10}, "num_magnitude_bins"), ({"policy": "autoaugment", "severity": 3}, "severity"),
    ({"policy": "augmix", "num_ops": 2}, "num_ops"), ({"policy": "augmix", "magnitude": 2}, "magnitude"),
    ({"policy": "rand", "alpha": 1.0}, "alpha"), ({"all_ops": True}, "all_ops"), ({"policy": "rand", "mixture_width": 2}, "mixture_width"),
    ({"policy": "augmix", "severity": 0}, "severity"), ({"policy": "augmix", "severity": 11}, "severity"),
    ({"policy": "augmix", "severity": True}, "severity"), ({"policy": "augmix", "severity": 3.0}, "severity"),
    ({"policy": "augmix", "mixture_width": 0}, "mixture_width"), ({"policy": "augmix", "mixture_width": 5}, "mixture_width"),
    ({"policy": "augmix", "mixture_width": False}, "mixture_width"), ({"policy": "augmix", "chain_depth": 0}, "chain_depth"),
    ({"policy": "augmix", "chain_depth": 4}, "chain_depth"), ({"policy": "augmix", "chain_depth": -2}, "chain_depth"),
    ({"policy": "augmix", "chain_depth": "1"}, "chain_depth"), ({"policy": "augmix", "alpha": 0.0}, "alpha"),
    ({"policy": "augmix", "alpha": -1.0}, "alpha"), ({"policy": "augmix", "alpha": 16.5}, "alpha"),
    ({"policy": "augmix", "alpha": float("nan")}, "alpha"), ({"policy": "augmix", "alpha": float("inf")}, "alpha"),
    ({"policy": "augmix", "alpha": True}, "alpha"), ({"policy": "augmix", "alpha": "1"}, "alpha"),
    ({"policy": "augmix", "all_ops": 1}, "all_ops"), ({"policy": "augmix", "all_ops": "true"}, "all_ops"),
    ({"policy": "augmix", "seed": 1.0}, "seed"), ({"policy": "autoaugment", "seed": None}, "seed")])
def test_malformed_values_are_value_errors_naming_the_key(bad, key):
    from theanompi_b200.models.alex_net import AlexNet
    with pytest.raises(ValueError, match=r"%s\[%r\]" % (AA_KEY, key)):
        check_auto_augment(bad)
    with pytest.raises(ValueError, match=AA_KEY):
        _build(AlexNet, auto_augment=bad, **IMG)


@pytest.mark.parametrize("policy", ["autoaugment", "augmix"])
def test_models_refuse_or_accept_the_policies_and_color_jitter_is_refused(policy):
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    for cls, kw in _refused():
        with pytest.raises(ValueError, match=AA_KEY + " is not supported"):
            _build(cls, auto_augment={"policy": policy}, **kw)
    with pytest.raises(ValueError, match=AA_KEY + " and color_jitter"):
        _build(AlexNet, auto_augment={"policy": policy}, color_jitter=ALL4, **IMG)
    m = _build(ResNet50, auto_augment={"policy": policy}, random_resized_crop={}, blocks=(1, 1, 1, 1), **IMG)
    assert m.auto_augment["policy"] == policy


# --------------------------------------------------------------------------- tables
def test_imagenet_sub_policies_are_torchvisions():
    A = pytest.importorskip("torchvision.transforms.v2._auto_augment")
    assert tuple(tuple(tuple(op) for op in sub) for sub in A.AutoAugment()._policies) == AA_IMAGENET_POLICY
    assert len(AA_IMAGENET_POLICY) == 25


@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227)])
@pytest.mark.parametrize("policy,all_ops", [("autoaugment", True), ("augmix", True), ("augmix", False)])
def test_op_spaces_are_torchvisions(policy, all_ops, out_hw):
    A = pytest.importorskip("torchvision.transforms.v2._auto_augment")
    space = {"autoaugment": A.AutoAugment._AUGMENTATION_SPACE, "augmix": A.AugMix._AUGMENTATION_SPACE if all_ops else
             A.AugMix._PARTIAL_AUGMENTATION_SPACE}[policy]
    got = auto_augment_space(policy, 10, out_hw, all_ops)
    assert tuple(got) == tuple(space)
    if policy == "augmix":
        assert tuple(got) == (AA_AUGMIX_OPS if all_ops else AA_AUGMIX_OPS[:9])
    for k, (fn, signed) in space.items():
        want = fn(10, out_hw[0], out_hw[1])
        assert got[k][1] == signed, k
        assert (got[k][0] is None) == (want is None), k
        if want is not None:
            assert np.array_equal(got[k][0], want.double().numpy()), k


# --------------------------------------------------------------------------- draws
def _aa_raw(n, cfg, rank=0):
    """The raw "autoaugment" draw in its documented order: sub-policy, application uniforms, sign uniforms."""
    rng = auto_augment_rng(cfg, rank)
    return rng.integers(0, 25, n), rng.random((n, 2)), rng.random((n, 2))


def _augmix_raw(n, cfg, rank=0):
    """The raw "augmix" draw in its documented order: m, d, depths (chain_depth −1 only), op indices, bins, sign uniforms."""
    rng, w = auto_augment_rng(cfg, rank), cfg["mixture_width"]
    m = rng.dirichlet([cfg["alpha"]] * 2, n).astype(np.float32)
    d = rng.dirichlet([cfg["alpha"]] * w, n).astype(np.float32)
    depth = rng.integers(1, 4, (n, w)) if cfg["chain_depth"] < 0 else np.full((n, w), cfg["chain_depth"])
    return m, d, depth, rng.integers(0, 13 if cfg["all_ops"] else 9, (n, w, 3)), rng.integers(0, cfg["severity"], (n, w, 3)), \
        rng.random((n, w, 3))


def test_autoaugment_draw_statistics():
    from scipy import stats
    n = 50000
    cfg = check_auto_augment({"policy": "autoaugment", "seed": 3})
    rec, op, mag = auto_augment_records(n, cfg, auto_augment_rng(cfg, 0), (224, 224))
    assert rec.shape == (n, 2, 12) and rec.dtype == np.float32 and not rec[..., 3].any()
    sub, au, su = _aa_raw(n, cfg)
    assert stats.chisquare(np.bincount(sub, minlength=25)).pvalue > 1e-4
    for j in range(2):
        ids = np.array([AA_OP_IDS[s[j][0]] for s in AA_IMAGENET_POLICY])
        p = np.array([s[j][1] for s in AA_IMAGENET_POLICY])
        assert np.array_equal(op[:, j], np.where(au[:, j] <= p[sub], ids[sub], 0))
        for k in range(25):                                   # the application rate of each op of each sub-policy is its p
            applied = int((op[sub == k, j] != 0).sum())
            assert stats.binomtest(applied, int((sub == k).sum()), p[k]).pvalue > 1e-4 if 0 < p[k] < 1 else applied == p[k] * (sub == k).sum()
    signed = np.isin(op, [1, 2, 3, 4, 5, 7, 8, 9]) & (mag != 0)
    assert stats.binomtest(int((mag[signed] < 0).sum()), int(signed.sum()), 0.5).pvalue > 1e-4
    assert (op == AA_INVERT).any() and np.all(mag[op == AA_INVERT] == 0)


@pytest.mark.parametrize("alpha", [1.0, 0.4])
@pytest.mark.parametrize("all_ops", [True, False])
def test_augmix_draw_statistics(alpha, all_ops):
    from scipy import stats
    n, width, sev = 40000, 3, 7
    cfg = check_auto_augment({"policy": "augmix", "alpha": alpha, "all_ops": all_ops, "severity": sev, "seed": 5})
    rec, wts, op, mag = augmix_records(n, cfg, auto_augment_rng(cfg, 0), (224, 224))
    assert rec.shape == (n, 9, 12) and wts.shape == (n, 4) and wts.dtype == np.float32 and np.all(rec[..., 3] == ((op >= 1) & (op <= 5)))
    m, d, depth, k, bins, su = _augmix_raw(n, cfg)
    assert np.array_equal(wts[:, 0], m[:, 0]) and np.array_equal(wts[:, 1:], d * m[:, 1:])        # fp32 products, as torchvision's
    # Dirichlet moments: Beta(α, α) for m₀ and Dirichlet(α·1₃) for d, each mean within 5 standard errors and each variance within 5 %
    for x, mean, var in ((m[:, 0].astype(np.float64), 0.5, 1.0 / (4 * (2 * alpha + 1))),
                         (d[:, 0].astype(np.float64), 1.0 / width, (1.0 / width) * (1 - 1.0 / width) / (width * alpha + 1))):
        assert abs(x.mean() - mean) < 5 * np.sqrt(var / n), (x.mean(), mean)
        assert abs(x.var() / var - 1) < 0.05, (x.var(), var)
    live = (op != AA_NONE).reshape(n, width, 3)
    assert np.array_equal(live.sum(2), depth) and np.all(live[..., 0]) and np.all(live[..., 1] >= live[..., 2])
    assert stats.chisquare(np.bincount(depth.ravel(), minlength=4)[1:]).pvalue > 1e-4
    names = AA_AUGMIX_OPS if all_ops else AA_AUGMIX_OPS[:9]
    ids = op[op != AA_NONE]
    assert stats.chisquare(np.array([(ids == AA_OP_IDS[s]).sum() for s in names])).pvalue > 1e-4
    assert set(np.unique(ids)) == {AA_OP_IDS[s] for s in names}
    table = auto_augment_space("augmix", 10, (224, 224))["Rotate"][0]
    got_bins = np.searchsorted(table, np.abs(mag[op == AA_OP_IDS["Rotate"]]) - 1e-9)
    assert got_bins.max() == sev - 1 and stats.chisquare(np.bincount(got_bins, minlength=sev)).pvalue > 1e-4
    signed = np.isin(op, [1, 2, 3, 4, 5, 7, 8, 9]) & (mag != 0)
    assert stats.binomtest(int((mag[signed] < 0).sum()), int(signed.sum()), 0.5).pvalue > 1e-4
    fixed = check_auto_augment({"policy": "augmix", "chain_depth": 2, "mixture_width": 1})
    op1 = augmix_records(100, fixed, auto_augment_rng(fixed, 0), (224, 224))[2]
    assert op1.shape == (100, 3) and np.all(op1[:, 2] == AA_NONE) and not np.any(op1[:, :2] == AA_NONE)


@pytest.mark.parametrize("policy", ["autoaugment", "augmix"])
def test_draws_are_independent_of_the_other_streams(policy):
    """The policy draws come from (seed, rank, 2): the random-resized-crop boxes and the erase boxes of the CPU loader are the same
    with the policy on or off, and two ranks draw apart."""
    aa = check_auto_augment({"policy": policy, "seed": 2})
    rrc, re = check_resized_crop({"seed": 5}), check_random_erasing({"p": 1.0, "seed": 6})
    got = []
    for a in (aa, None):
        d = _data()
        ld = d.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, resized_crop=rrc, rank=1, random_erasing=re,
                              auto_augment=a)
        ld.request(d.train_img[0], "train")
        b = ld.get()
        got.append((b.boxes, b.flips, b.erase, b.aa_records))
        ld.drain(); d.para_load_close()
    (bx, fl, er, rec), (bx0, fl0, er0, rec0) = got
    assert np.array_equal(bx, bx0) and np.array_equal(fl, fl0) and np.array_equal(er, er0) and rec0 is None
    assert np.array_equal(bx, draw_resized_crops(8, (32, 32), rrc["scale"], rrc["ratio"], resized_crop_rng(rrc, 1))[0])
    assert np.array_equal(er, draw_erase_boxes(8, (20, 24), re, random_erasing_rng(re, 1)))
    a = auto_augment_records(64, aa, auto_augment_rng(aa, 0), (224, 224))[0]
    assert np.array_equal(a, auto_augment_records(64, aa, auto_augment_rng(aa, 0), (224, 224))[0])
    assert not np.array_equal(a, auto_augment_records(64, aa, auto_augment_rng(aa, 1), (224, 224))[0])


# --------------------------------------------------------------------------- the reference against torchvision
def _augmented(img, rec, weights=None):
    """The reference's augmented uint8 image u' for one CHW image: auto_augment_crop_normalize on the box of the whole image, mean 0,
    scale 1."""
    C, h, w = img.shape
    out = ref.auto_augment_crop_normalize(img.permute(1, 2, 0).unsqueeze(0).contiguous(), torch.zeros(1), 1.0, (h, w),
                                          np.int32([[0, 0, h, w]]), np.uint8([0]), rec[None],
                                          weights=None if weights is None else weights[None])
    return out[0].permute(2, 0, 1).round().to(torch.uint8)


def _assert_same(got, want, what, geometric):
    """Exact; a record with a geometric op may also pass under the tie rule (a miss at fewer than 1e-3 of the elements)."""
    if torch.equal(got, want):
        return
    assert geometric, "%s: %d elements differ" % (what, int((got != want).sum()))
    diff = (got != want).float().mean().item()
    assert diff < 1e-3, "%s: %g of the elements differ" % (what, diff)


@pytest.mark.parametrize("interp", ["nearest", "bilinear"])
@pytest.mark.parametrize("hw", [(40, 48), (224, 224)])
def test_autoaugment_reference_is_torchvisions_forward(interp, hw):
    cfg = check_auto_augment({"policy": "autoaugment", "interpolation": interp, "seed": hw[0]})
    n = 150 if hw[0] < 100 else 40
    rec = auto_augment_records(n, cfg, auto_augment_rng(cfg, 0), hw)[0]
    sub, au, su = _aa_raw(n, cfg)
    g = torch.Generator().manual_seed(hw[1])
    for k in range(n):
        img = torch.randint(0, 256, (3,) + hw, dtype=torch.uint8, generator=g)
        want = oracle.autoaugment(img, int(sub[k]), au[k], su[k], interp)
        geo = bool(((rec[k, :, 0] >= 1) & (rec[k, :, 0] <= 5)).any())
        _assert_same(_augmented(img, rec[k]), want, "sub-policy %d" % sub[k], geo)
    if hw[0] < 100:
        assert set(sub) == set(range(25)) and (rec[..., 0] == AA_INVERT).any()


@pytest.mark.parametrize("case", [
    dict(), dict(interpolation="nearest"), dict(all_ops=False), dict(chain_depth=1, mixture_width=1), dict(chain_depth=3, mixture_width=4),
    dict(severity=10, alpha=0.3, mixture_width=2), dict(all_ops=False, chain_depth=2, severity=1, interpolation="nearest")])
def test_augmix_reference_is_torchvisions_forward(case):
    hw = (40, 48)
    cfg = check_auto_augment(dict(case, policy="augmix", seed=len(case)))
    n = 60
    rec, wts, op, _ = augmix_records(n, cfg, auto_augment_rng(cfg, 0), hw)
    m, d, depth, kk, bins, su = _augmix_raw(n, cfg)
    names = list(auto_augment_space("augmix", 10, hw, cfg["all_ops"]))
    g = torch.Generator().manual_seed(11)
    for k in range(n):
        img = torch.randint(0, 256, (3,) + hw, dtype=torch.uint8, generator=g)
        want = oracle.augmix(img, m[k], d[k], depth[k], [[names[j] for j in row] for row in kk[k]], bins[k], su[k], cfg["severity"],
                             cfg["chain_depth"], cfg["all_ops"], cfg["interpolation"])
        geo = bool(((op[k] >= 1) & (op[k] <= 5)).any())
        _assert_same(_augmented(img, rec[k], wts[k]), want, "image %d" % k, geo)


@pytest.mark.parametrize("interp", ["nearest", "bilinear"])
@pytest.mark.parametrize("name", AA_AUGMIX_OPS + ("Invert",))
def test_each_op_is_torchvisions_in_both_interpolations(name, interp):
    """Every op of the two new spaces, through its record, at every bin's magnitude and both signs."""
    A = pytest.importorskip("torchvision.transforms.v2._auto_augment")
    from theanompi_b200.models.data.utils import aa_compose_records
    hw = (40, 48)
    space = dict(auto_augment_space("augmix", 10, hw), Invert=(None, False))
    mags = space[name][0] if space[name][0] is not None else np.zeros(1)
    g = torch.Generator().manual_seed(3)
    for mag in np.concatenate([mags, -mags if space[name][1] else []]):
        img = torch.randint(0, 256, (3,) + hw, dtype=torch.uint8, generator=g)
        rec = aa_compose_records(np.array([AA_OP_IDS[name]]), np.array([mag]), hw, interp == "bilinear")[0]
        want = A.AugMix()._apply_image_or_video_transform(img, name, float(mag), interpolation=oracle.interpolation(interp),
                                                           fill={torch.Tensor: None})
        _assert_same(ref.aa_apply_op(img, rec), want, "%s %g" % (name, mag), 1 <= AA_OP_IDS[name] <= 5)
    assert torch.equal(ref.aa_apply_op(img, np.float32([AA_NONE] + [0] * 11)), img)


def test_augmix_mix_is_fp32_multiply_then_add_then_truncation():
    g = torch.Generator().manual_seed(4)
    u = torch.randint(0, 256, (3, 9, 11), dtype=torch.uint8, generator=g)
    chains = [torch.randint(0, 256, (3, 9, 11), dtype=torch.uint8, generator=g) for _ in range(3)]
    w = np.float32([0.3, 0.1, 0.25, 0.35])
    got = ref.augmix_mix(u, chains, w)
    acc = np.float32(w[0]) * u.numpy().astype(np.float32)
    for i in range(3):
        acc = (acc + np.float32(w[1 + i]) * chains[i].numpy().astype(np.float32)).astype(np.float32)
    assert np.array_equal(got.numpy(), np.trunc(acc).astype(np.uint8))
    assert torch.equal(ref.augmix_mix(u, chains[:1], np.float32([0.0, 1.0])), chains[0])


# --------------------------------------------------------------------------- loader and serial path
@pytest.mark.parametrize("policy", ["autoaugment", "augmix"])
def test_cpu_loader_train_batches_are_the_reference_of_their_draw(policy):
    aa = check_auto_augment({"policy": policy, "seed": 2})
    d = _data()
    ld = d.para_load_init("cpu", 24, 20, rand_crop=True, batch_crop_mirror=False, rank=2, auto_augment=aa)
    rng = auto_augment_rng(aa, 2)
    mean, cs = torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5])
    ld.request(d.train_img[0], "train")
    for k in range(1, 3):
        ld.request(d.train_img[k % 3], "train")
        b = ld.get()
        if policy == "augmix":
            rec, wts = augmix_records(8, aa, rng, (20, 24))[:2]
            assert np.array_equal(b.aa_weights, wts) and b.h2d_bytes == 8 * 32 * 32 * 3 + 8 * 17 + rec.nbytes + wts.nbytes
        else:
            rec, wts = auto_augment_records(8, aa, rng, (20, 24))[0], None
            assert b.aa_weights is None
        assert np.array_equal(b.aa_records, rec)
        want = ref.auto_augment_crop_normalize(_raw(d, b.item), mean, cs, (20, 24), b.boxes, b.flips, rec, weights=wts)
        assert torch.equal(b.x, want)
    ld.drain(); d.para_load_close()


@pytest.mark.parametrize("policy", ["autoaugment", "augmix"])
def test_serial_load_batch_applies_it_and_tiny_models_train(policy):
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.data.utils import draw_crops
    from theanompi_b200.utils.recorder import Recorder
    m = _build(AlexNet, auto_augment={"policy": policy, "seed": 4}, **IMG)
    item = m.data.train_img_shard[0]
    np.random.seed(77)
    x = m.data.load_batch(item, "train", m)
    raw = np.empty((4, 256, 256, 3), np.uint8)
    src = m.data.read(item, raw)
    raw = torch.from_numpy(src.numpy() if src is not None else raw)
    np.random.seed(77)
    offs, flips = draw_crops(4, (256, 256), (227, 227), "train", True, False)
    boxes = np.concatenate([offs, np.int32([[227, 227]] * 4)], 1)
    va = check_auto_augment({"policy": policy, "seed": 4})
    wts = None
    if policy == "augmix":
        rec, wts = augmix_records(4, va, auto_augment_rng(va, 0), (227, 227))[:2]
    else:
        rec = auto_augment_records(4, va, auto_augment_rng(va, 0), (227, 227))[0]
    want = ref.auto_augment_crop_normalize(raw, torch.from_numpy(m.data.rawdata[4]), torch.from_numpy(1.0 / 255.0 / m.data.rawdata[5]),
                                           (227, 227), boxes, flips, rec, weights=wts)
    assert torch.equal(x, want)
    mm = _build(AlexNet, auto_augment={"policy": policy}, **IMG)
    mm.compile_iter_fns("avg")
    r = Recorder(None, 10 ** 6, "AlexNet", False, device="cpu")
    for i in range(2):
        mm.train_iter(i, r)
    assert all(np.isfinite(float(c)) for c in r.train_info["cost"])
