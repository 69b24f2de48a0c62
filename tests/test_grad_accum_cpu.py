"""Gradient accumulation (``config['grad_accum']``) on the CPU reference path: the micro-step kind sequence across file batches and
sub-batches, the discarded window at ``reset_iter``, the update counter, the refusals, and n micro-batches of B/n against one batch of
B after one update (sgd, lars, lamb, clipping)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import accum  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402


def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.05,
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    m = Cifar10_model(cfg)
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()        # the switches reach the layers built so far: deterministic comparisons
    return m


@pytest.fixture(autouse=True)
def no_dropout():
    yield
    Dropout.SetDropoutOn(); Crop.SetRandCropOn()


def _expected_kinds(n, steps):
    out = []
    for i in range(steps):
        j = i % n
        out.append("first" if j == 0 else ("last" if j == n - 1 else "mid"))
    return out if n > 1 else ["first"] * steps


@pytest.mark.parametrize("n", [1, 2, 3, 5])
@pytest.mark.parametrize("batch", [16, 8])
def test_kind_sequence_and_update_count(n, batch, no_dropout):
    """Windows run across file batches (batch 16: one micro-step per file) and sub-batches (batch 8: two per file)."""
    m = _cifar(batch_size=batch, grad_accum=n)
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    kinds, w_before = [], []
    steps = 2 * n + 1 if n > 1 else 5
    for i in range(steps):
        kinds.append(m.micro_step_kind() if n > 1 else "first")
        w_before.append(m.arena.W.clone())
        m.train_iter(i, rec)
    assert kinds == _expected_kinds(n, steps)
    assert m.n_updates == (steps // n if n > 1 else steps)
    assert len(rec.train_info["cost"]) == steps                          # every micro-step's cost is recorded
    w_before.append(m.arena.W.clone())
    for i, k in enumerate(kinds):
        moved = not torch.equal(w_before[i], w_before[i + 1])
        assert moved == (k == "last" or n == 1), (i, k)                   # weights move at the end of a window only


def test_reset_iter_discards_open_window(no_dropout):
    m = _cifar(batch_size=8, grad_accum=3)
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(5):                                                    # one window + 2 micro-steps of the next
        m.train_iter(i, rec)
    assert m.n_updates == 1 and m.micro_step_kind() == "last"
    w = m.arena.W.clone()
    m.reset_iter("train")
    assert m.n_discarded == 2 and m.micro_step_kind() == "first"
    # the next window starts from a stored G: its update equals a fresh model's first update from the same weights and data
    for i in range(3):
        m.train_iter(i, rec)
    assert m.n_updates == 2 and not torch.equal(w, m.arena.W)
    m.reset_iter("train")
    assert m.n_discarded == 2                                             # nothing open: nothing discarded


def test_first_micro_step_overwrites_stale_gradient(no_dropout):
    """G left over from a discarded window must not leak into the next one."""
    a = _cifar(batch_size=8, grad_accum=2)
    b = _cifar(batch_size=8, grad_accum=2)
    for m in (a, b):
        m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for m in (a, b):
        m.train_iter(0, rec)
        m.reset_iter("train")
    for v in a.arena.views("G"):
        v.fill_(123.0)
    for i in range(2):
        a.train_iter(i, rec); b.train_iter(i, rec)
    assert a.n_discarded == b.n_discarded == 1
    for va, vb in zip(a.arena.views("W"), b.arena.views("W")):
        assert torch.equal(va, vb)


@pytest.mark.parametrize("kw", [dict(), dict(optimizer="lars", learning_rate=1.0), dict(optimizer="lamb", learning_rate=0.01),
                                dict(grad_clip=0.5)], ids=["sgd", "lars", "lamb", "clip"])
def test_four_micro_batches_match_one_batch(kw, no_dropout):
    """grad_accum = 4 at batch 4 against grad_accum = 1 at batch 16 over the same 16 samples: one update, fp32 tolerance."""
    one = _cifar(batch_size=16, grad_accum=1, **kw)
    four = _cifar(batch_size=4, grad_accum=4, **kw)
    w0 = one.arena.W.clone()
    assert torch.equal(w0, four.arena.W)
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    one.compile_iter_fns("avg"); four.compile_iter_fns("avg")
    one.train_iter(0, rec)
    for i in range(4):
        four.train_iter(i, rec)
    assert one.n_updates == four.n_updates == 1
    step = (one.arena.W - w0).abs().max()
    assert float(step) > 1e-4                                             # a real update happened
    torch.testing.assert_close(four.arena.W, one.arena.W, rtol=1e-5, atol=1e-6)
    if "grad_clip" in kw:
        torch.testing.assert_close(four.clip_opt.grad_norm, one.clip_opt.grad_norm, rtol=1e-5, atol=0)
    if kw.get("optimizer") == "lamb":
        assert int(one.lamb.t) == int(four.lamb.t) == 1                  # the step counter advances once per window


def test_loss_gradient_scale():
    g = torch.Generator().manual_seed(3)
    lg = torch.randn(6, 10, generator=g)
    lab = torch.randint(0, 10, (6,), generator=g)
    l1, _, _, d1 = ref.softmax_xent(lg, lab)
    l3, _, _, d3 = ref.softmax_xent(lg, lab, grad_scale=float(np.float32(1 / 3)))
    assert float(l1) == float(l3)                                         # the reported loss is not scaled
    torch.testing.assert_close(d3, d1 * float(np.float32(1 / 3)), rtol=0, atol=0)
    from theanompi_b200 import ops
    x = lg.clone().requires_grad_(True)
    with accum.mode(False, 0.25):
        loss, _, _ = ops.softmax_xent(x, lab)
        loss.backward()
    torch.testing.assert_close(x.grad, d1 * 0.25)
    assert accum.grad_scale() == 1.0 and not accum.accumulating()         # restored on exit


def test_sink_adds_on_the_reference_path():
    from theanompi_b200.ops.functional import _sink
    p = torch.nn.Parameter(torch.zeros(4))
    p.gbuf = torch.ones(4)
    _sink(p, torch.full((4,), 2.0))
    assert torch.equal(p.gbuf, torch.full((4,), 2.0))
    with accum.mode(True):
        _sink(p, torch.full((4,), 3.0))
    assert torch.equal(p.gbuf, torch.full((4,), 5.0))


def test_refusals():
    for bad in (0, -1, 2.5, True, "2"):
        m = _cifar(grad_accum=bad)
        with pytest.raises(ValueError, match="grad_accum must be an int >= 1"):
            m.compile_iter_fns("avg")
    m = _cifar(grad_accum=2, size=2)
    with pytest.raises(ValueError, match="with 2 workers is not implemented.*runs on one worker"):
        m.check_grad_accum()
    m = _cifar(grad_accum=2)
    with pytest.raises(ValueError, match="fused exchange strategy.*runs on one worker"):
        m.compile_iter_fns("avg", fused_tail=lambda: None)
    _cifar(grad_accum=1, size=2).check_grad_accum(fused_tail=lambda: None)    # n = 1: nothing to refuse


def test_refusals_of_other_models():
    from theanompi_b200.models.lstm import LSTM
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    from theanompi_b200.models.torch_base import TorchModelBase
    for cls in (LSTM, NativeWGAN, WGAN, TorchModelBase):
        assert cls.supports_grad_accum is False
        m = cls.__new__(cls)
        m.grad_accum, m.size, m.name = 3, 1, cls.__name__
        with pytest.raises(ValueError, match="does not accumulate gradients.*runs on one worker"):
            m.check_grad_accum()


def test_wide_resnet_adam_window_counts_once():
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    layers2.reseed()
    m = Wide_ResNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=8, depth=10, widen=1,
                         grad_accum=2, data_kwargs=dict(n_synthetic=64, synthetic=True)))
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(4):
        m.train_iter(i, rec)
    assert int(m.adam.t) == 2 and m.n_updates == 2
