"""Stochastic depth (config['drop_path_rate']) on the CPU path: the validation of the key and the models that refuse it, the p_l rule,
the statistics of the reference draw, the reference batch-norm / add with a drop row against fp64 torch autograd of the formula,
tiny ResNet50 / Wide_ResNet training and validation, and a two-rank gloo BSP run through the Rule API."""
import math
import os
import pickle
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import drop_path  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402

IMG = dict(no_paraload=True, n_class=8, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))


def _reseed():
    """Weights, the synthetic data and the host-side crops of a model built next are the same every time."""
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)


def _resnet(**kw):
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    _reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, blocks=(1, 1, 1, 1), learning_rate=0.01, **IMG)
    cfg.update(kw)
    return ResNet50(cfg)


def _wrn(**kw):
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    _reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=8, file_batch_size=16, depth=10, widen=1,
               data_kwargs=dict(n_synthetic=256, synthetic=True))
    cfg.update(kw)
    return Wide_ResNet(cfg)


def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=8, data_kwargs=dict(n_synthetic=64, synthetic=True))
    cfg.update(kw)
    return Cifar10_model(cfg)


# --------------------------------------------------------------------------- configuration
@pytest.mark.parametrize("bad", [True, False, float("nan"), float("inf"), "0.1", -0.1, 1.0, 1.5, None])
def test_rate_must_be_a_real_in_0_1(bad):
    m = _wrn(drop_path_rate=bad)
    with pytest.raises(ValueError, match="drop_path_rate"):
        m.compile_iter_fns("avg")


def test_zero_and_absent_build_nothing_and_positive_builds_the_table():
    for kw in ({}, dict(drop_path_rate=0), dict(drop_path_rate=0.0)):
        m = _wrn(**kw)
        m.compile_iter_fns("avg")
        assert m.drop_path is None and m.drop_row(1) is None
    m = _wrn(drop_path_rate=0.2)
    m.compile_iter_fns("avg")
    dp = m.drop_path
    assert (dp.L, dp.B) == (3, 8) and tuple(dp.table.shape) == (3, 8)
    assert m.drop_row(2) is None                                  # only the training forward reads the table


def _refused():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNetTorch
    from theanompi_b200.models.lasagne_model_zoo.lsgan import LSGAN, NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    from theanompi_b200.models.cifar10 import Cifar10_model
    img = dict(batch_size=4, file_batch_size=4, **IMG)
    return [(AlexNet, img), (AlexNet_sc, img), (GoogLeNet, img),
            (Cifar10_model, dict(batch_size=4, file_batch_size=8, data_kwargs=dict(n_synthetic=64, synthetic=True))),
            (NativeWGAN, dict(data_kwargs=dict(n_synthetic=128))), (NativeLSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (WGAN, dict(data_kwargs=dict(n_synthetic=128))), (LSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (LSTM, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (LSTMTorch, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (ResNet50Torch, dict(img, blocks=(1, 1, 1, 1))),
            (Wide_ResNetTorch, dict(batch_size=8, file_batch_size=8, depth=10, widen=1, data_kwargs=dict(n_synthetic=64, synthetic=True)))]


def test_models_without_residual_blocks_and_the_twins_refuse_it():
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    assert VGG16.supports_drop_path is False                      # its 224² fp32 FC weights are too large to build here
    for cls, kw in _refused():
        assert cls.supports_drop_path is False, cls
        layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", drop_path_rate=0.1, **kw))
        with pytest.raises(ValueError, match="drop_path_rate = 0.1 is not supported.*ResNet50, ResNet152 and Wide_ResNet"):
            m.compile_iter_fns("avg")
        layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", drop_path_rate=0.0, **kw))
        m.compile_iter_fns("avg")
        assert m.drop_path is None


def test_resnet152_inherits_it():
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    assert ResNet152.supports_drop_path is True and ResNet152.blocks == (3, 8, 36, 3) and sum(ResNet152.blocks) == 50


# --------------------------------------------------------------------------- the p_l rule and the draw
@pytest.mark.parametrize("p,L", [(0.1, 16), (0.2, 50), (0.3, 12), (0.5, 3), (0.4, 2)])
def test_block_rates_are_linspace(p, L):
    r = drop_path.block_rates(p, L)
    assert r[0] == 0.0 and r[-1] == p
    assert np.allclose(r, torch.linspace(0, p, L, dtype=torch.float64).numpy(), rtol=0, atol=1e-15)
    assert np.array_equal(drop_path.keep_scales(r), np.float32(1.0 / (1.0 - r)))
    t = drop_path.thresholds(r)
    assert t[0] == 0 and np.all(t / 2.0 ** 24 >= r) and np.all((t - 1) / 2.0 ** 24 < r)


def test_one_block_never_drops():
    assert drop_path.block_rates(0.7, 1).tolist() == [0.0]
    tab = ref.drop_path_draw(drop_path.block_rates(0.7, 1), 1, 0, 5, 32)
    assert torch.equal(tab, torch.ones(1, 32))
    with pytest.raises(ValueError):
        drop_path.block_rates(0.1, 0)


def test_reference_draw_statistics():
    p, L, B = 0.4, 5, 64
    rates = drop_path.block_rates(p, L)
    tabs = torch.stack([ref.drop_path_draw(rates, 0x5EED, rank, step, B) for rank in range(3) for step in range(400)])
    N = tabs.shape[0] * B
    keep = drop_path.keep_scales(rates)
    for l in range(L):
        vals = tabs[:, l].reshape(-1)
        assert set(torch.unique(vals).tolist()) <= {0.0, float(keep[l])}
        frac = float((vals == 0).double().mean())
        sd = math.sqrt(max(rates[l] * (1 - rates[l]), 1e-12) / N)
        assert abs(frac - rates[l]) < 5 * sd + 1e-12, (l, frac, rates[l])
        if rates[l] > 0:
            mean_sd = math.sqrt(rates[l] / (1 - rates[l]) / N)
            assert abs(float(vals.double().mean()) - 1.0) < 5 * mean_sd, l
        else:
            assert torch.all(vals == 1.0)


def test_ranks_and_steps_draw_different_tables():
    rates = drop_path.block_rates(0.5, 4)
    a = ref.drop_path_draw(rates, 7, 0, 3, 32)
    assert torch.equal(a, ref.drop_path_draw(rates, 7, 0, 3, 32))
    for other in (ref.drop_path_draw(rates, 7, 1, 3, 32), ref.drop_path_draw(rates, 7, 0, 4, 32), ref.drop_path_draw(rates, 8, 0, 3, 32)):
        assert not torch.equal(a, other)


# --------------------------------------------------------------------------- reference ops against fp64 autograd
def _rows(kind, B, p=0.3):
    s = 1.0 / (1.0 - p)
    if kind == "all":
        return torch.zeros(B)
    if kind == "none":
        return torch.full((B,), np.float32(s))
    g = torch.Generator().manual_seed(B)
    return torch.where(torch.rand(B, generator=g) < 0.5, torch.zeros(B), torch.full((B,), np.float32(s)))


@pytest.mark.parametrize("kind", ["all", "none", "mixed"])
@pytest.mark.parametrize("relu", [True, False])
def test_reference_batch_norm_with_drop(kind, relu):
    torch.manual_seed(0)
    B, H, W, C = 6, 3, 5, 8
    x, res, dy = torch.randn(B, H, W, C), torch.randn(B, H, W, C), torch.randn(B, H, W, C)
    gamma, beta = torch.rand(C) + 0.5, torch.randn(C)
    s = _rows(kind, B)
    rm, rv = torch.zeros(C), torch.ones(C)
    y, mean, rstd = ref.batch_norm_fwd(x, gamma, beta, rm, rv, True, 0.1, 1e-5, relu, res, drop=s)
    dx, dres, dg, db = ref.batch_norm_bwd(x, dy, y, gamma, mean, rstd, relu, True, drop=s)
    xd, gd, bd, rd = (t.double().requires_grad_() for t in (x, gamma, beta, res))
    m = xd.mean((0, 1, 2))
    v = ((xd - m) ** 2).mean((0, 1, 2))
    yd = s.double().view(B, 1, 1, 1) * ((xd - m) / torch.sqrt(v + 1e-5) * gd + bd) + rd
    if relu:
        yd = torch.relu(yd)
    yd.backward(dy.double())
    assert torch.allclose(y.double(), yd.detach(), atol=1e-4)
    for got, want in ((dx, xd.grad), (dres, rd.grad), (dg, gd.grad), (db, bd.grad)):
        assert torch.allclose(got.double(), want, atol=1e-3, rtol=1e-4)
    # the running statistics are those of the whole batch, dropped samples included
    assert torch.allclose(rm, 0.1 * x.reshape(-1, C).mean(0), atol=1e-6)
    with pytest.raises(ValueError, match="residual"):
        ref.batch_norm_fwd(x, gamma, beta, None, None, True, 0.1, 1e-5, relu, None, drop=s)


@pytest.mark.parametrize("kind", ["all", "none", "mixed"])
def test_reference_add_with_drop(kind):
    torch.manual_seed(1)
    B = 5
    a, b, dy = torch.randn(B, 4, 4, 8), torch.randn(B, 4, 4, 8), torch.randn(B, 4, 4, 8)
    s = _rows(kind, B)
    ad, bd = a.double().requires_grad_(), b.double().requires_grad_()
    yd = s.double().view(B, 1, 1, 1) * ad + bd
    yd.backward(dy.double())
    ar, br = a.clone().requires_grad_(), b.clone().requires_grad_()
    y = ops.add(ar, br, drop=s)
    y.backward(dy)
    assert torch.allclose(y.double(), yd.detach(), atol=1e-6)
    assert torch.allclose(ar.grad.double(), ad.grad, atol=1e-6) and torch.equal(br.grad, dy)
    assert torch.allclose(ref.add_scaled(dy, s).double(), ad.grad, atol=1e-6)


def test_functional_batch_norm_carries_the_row_into_backward():
    torch.manual_seed(2)
    B, C = 4, 8
    x, res = torch.randn(B, 2, 2, C, requires_grad=True), torch.randn(B, 2, 2, C, requires_grad=True)
    gamma, beta = torch.nn.Parameter(torch.rand(C) + 0.5), torch.nn.Parameter(torch.randn(C))
    s = _rows("mixed", B)
    y = ops.batch_norm(x, gamma, beta, None, None, True, 0.1, 1e-5, True, res, drop=s)
    dy = torch.randn_like(y)
    y.backward(dy)
    yr, mean, rstd = ref.batch_norm_fwd(x.detach(), gamma.detach(), beta.detach(), None, None, True, 0.1, 1e-5, True, res.detach(), drop=s)
    dx, dres, dg, db = ref.batch_norm_bwd(x.detach(), dy, yr, gamma.detach(), mean, rstd, True, True, drop=s)
    assert torch.equal(y, yr) and torch.equal(x.grad, dx) and torch.equal(res.grad, dres)
    assert torch.equal(gamma.grad, dg) and torch.equal(beta.grad, db)


# --------------------------------------------------------------------------- tiny models on the CPU path
def _train(m, n):
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(n):
        m.train_iter(i, rec)
    return [float(c) for c in rec.train_info["cost"]]


def _val(m):
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.reset_iter("val")
    m.val_iter(0, rec)
    return float(rec.val_info["cost"][-1])


def _force_ones(m):
    dp = m.drop_path
    dp.draw = lambda: dp.table.fill_(1.0)                         # every block of every step keeps every sample, with scale 1


@pytest.mark.parametrize("make", [_resnet, _wrn], ids=["resnet50", "wide_resnet"])
def test_forced_ones_matches_no_key_and_p_changes_the_weights(make):
    runs = {}
    for name, kw in (("absent", {}), ("zero", dict(drop_path_rate=0.0)), ("ones", dict(drop_path_rate=0.3)),
                     ("drop", dict(drop_path_rate=0.5))):
        ops.seed_dropout(0x5EED)
        m = make(**kw)
        m.compile_iter_fns("avg")
        if name == "ones":
            _force_ones(m)
        costs = _train(m, 3)
        assert all(math.isfinite(c) for c in costs), (name, costs)
        runs[name] = m.arena.W.clone(), m.arena.U.clone()
    for name in ("zero", "ones"):
        assert torch.equal(runs[name][0], runs["absent"][0]) and torch.equal(runs[name][1], runs["absent"][1]), name
    assert not torch.equal(runs["drop"][0], runs["absent"][0])


@pytest.mark.parametrize("make", [_resnet, _wrn], ids=["resnet50", "wide_resnet"])
def test_training_reads_the_table_and_validation_never_drops(make, monkeypatch):
    ops.seed_dropout(0x5EED)
    m = make(drop_path_rate=0.5)
    m.compile_iter_fns("avg")
    seen = []
    bn, add = ops.batch_norm, ops.add

    def spy_bn(*a, drop=None, **k):
        seen.append(drop)
        return bn(*a, drop=drop, **k)

    def spy_add(a, b, drop=None):
        seen.append(drop)
        return add(a, b, drop=drop)
    monkeypatch.setattr(ops, "batch_norm", spy_bn)
    monkeypatch.setattr(ops, "add", spy_add)
    step = ops.rng_state()["step"]
    _train(m, 1)
    rows = [d for d in seen if d is not None]
    assert len(rows) == len(m.body) - 1                            # block 0 has p_0 = 0: no row
    want = ref.drop_path_draw(m.drop_path.rates, ops.rng_state()["seed"], 0, step, m.batch_size)
    assert torch.equal(m.drop_path.table, want)
    for l, r in enumerate(rows, start=1):
        assert torch.equal(r, want[l])
    seen.clear()
    c1 = _val(m)
    assert seen and all(d is None for d in seen)
    monkeypatch.undo()
    m.drop_path_rate = 0.0
    m.check_drop_path()
    assert m.drop_path is None and _val(m) == c1                   # the same weights validate the same without the key


def test_grad_accum_micro_steps_draw_fresh_tables():
    ops.seed_dropout(3)
    m = _resnet(drop_path_rate=0.6, grad_accum=2)
    m.compile_iter_fns("avg")
    tabs = []
    for i in range(4):
        _train(m, 1)
        tabs.append(m.drop_path.table.clone())
    assert all(not torch.equal(tabs[i], tabs[j]) for i in range(4) for j in range(i))
    assert m.n_updates == 2


# --------------------------------------------------------------------------- distributed
def test_rule_bsp_avg_two_gloo_ranks(tmp_path, monkeypatch):
    """BSP sync_type='avg' with drop_path_rate in rule.model_config: the key reaches both ResNet50 workers (an invalid value stops
    them at compile_iter_fns) and the run completes with finite training costs recorded."""
    import subprocess
    import theanompi_b200 as tm
    monkeypatch.chdir(tmp_path)
    tm.BSP.sync_type, tm.BSP.exch_strategy = "avg", "ar"
    rcs = {}
    for name, p in (("good", 0.3), ("bad", 1.0)):
        rule = tm.BSP()
        rule.model_config = dict(batch_size=4, file_batch_size=4, n_epochs=1, learning_rate=0.01, max_batches=3, printFreq=2,
                                 blocks=(1, 1, 1, 1), drop_path_rate=p, **IMG)
        rule.env["OMP_NUM_THREADS"] = "2"
        rule.init(devices=["cpu0", "cpu1"], modelfile="theanompi_b200.models.lasagne_model_zoo.resnet50", modelclass="ResNet50")
        try:
            rcs[name] = rule.proc.wait(timeout=600)
        except subprocess.TimeoutExpired:
            rule.proc.kill()
            raise
        if name == "good":
            with open(tmp_path / "inforec" / "inforec.pkl", "rb") as f:
                costs = [c for _, c, _ in pickle.load(f)["train_info"]]
            assert costs and all(math.isfinite(c) and c > 0 for c in costs), costs
    assert rcs["good"] == 0 and rcs["bad"] != 0, rcs
