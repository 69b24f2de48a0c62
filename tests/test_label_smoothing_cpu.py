"""Label smoothing (``config['label_smoothing']``) on the CPU reference path: ``reference.softmax_xent`` against
``F.cross_entropy(label_smoothing=ε)`` and its autograd gradient in fp64, the validation of the key and the refusals, training steps
of Cifar10_model, GoogLeNet, the LSTM and a torch twin whose recorded cost is the smoothed loss while validation stays plain NLL, and a
two-rank gloo BSP run through the Rule API."""
import math
import os
import pickle
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402


def _oracle(lg, lab, eps, weight=1.0, grad_scale=1.0):
    """fp64 torch: weight · F.cross_entropy(label_smoothing=ε) and d(that)/dlogits · grad_scale."""
    x = lg.double().clone().requires_grad_(True)
    loss = weight * F.cross_entropy(x, lab, label_smoothing=eps)
    loss.backward()
    return float(loss.detach()), x.grad * grad_scale


# --------------------------------------------------------------------------- reference.softmax_xent
@pytest.mark.parametrize("C", [2, 10, 1000])
@pytest.mark.parametrize("eps", [0.05, 0.1, 0.5, 1.0])
def test_reference_matches_torch_cross_entropy(eps, C):
    g = torch.Generator().manual_seed(C)
    B = 24
    lg = torch.randn(B, C, generator=g, dtype=torch.float64) * 3
    lab = torch.randint(0, C, (B,), generator=g)
    weight, grad_scale = 0.3, 0.25
    loss, e1, e5, dl = ref.softmax_xent(lg, lab, grad_scale=grad_scale, weight=weight, label_smoothing=eps)
    want, dwant = _oracle(lg, lab, eps, weight, grad_scale)
    assert abs(float(loss) - want) < 1e-5 * max(1.0, abs(want)), (float(loss), want)
    assert float((dl.double() - dwant).abs().max()) < 1e-6 * float(dwant.abs().max()) + 1e-9
    _, e1_0, e5_0, _ = ref.softmax_xent(lg, lab)
    assert float(e1) == float(e1_0) and float(e5) == float(e5_0)        # the errors depend only on the ranking


def test_reference_at_zero_is_the_present_call():
    g = torch.Generator().manual_seed(7)
    lg = torch.randn(16, 10, generator=g)
    lab = torch.randint(0, 10, (16,), generator=g)
    for gs in (1.0, 1 / 3):
        a = ref.softmax_xent(lg, lab, grad_scale=gs)
        b = ref.softmax_xent(lg, lab, grad_scale=gs, label_smoothing=0.0)
        for x, y in zip(a, b):
            assert torch.equal(x, y)
    loss, _, _, dl = a
    want, dwant = _oracle(lg, lab, 0.0, grad_scale=1 / 3)
    assert abs(float(loss) - want) < 1e-5 and float((dl.double() - dwant).abs().max()) < 1e-7


def test_functional_node_passes_epsilon_through_autograd():
    g = torch.Generator().manual_seed(3)
    lg = torch.randn(8, 10, generator=g).requires_grad_(True)
    lab = torch.randint(0, 10, (8,), generator=g)
    loss, _, _ = ops.softmax_xent(lg, lab, 0.1)
    loss.backward()
    want, dwant = _oracle(lg.detach(), lab, 0.1)
    assert abs(float(loss) - want) < 1e-5
    assert float((lg.grad.double() - dwant).abs().max()) < 1e-6


def test_softmax_cache_is_keyed_on_epsilon():
    layers2.reseed()
    sm = layers2.Softmax(None, 10, input_shape=(8, 16), printinfo=False)
    x = torch.randn(8, 16)
    y = torch.randint(0, 10, (8,))
    sm.forward(x)
    plain = sm.negative_log_likelihood(y)
    smooth = sm.negative_log_likelihood(y, 0.2)
    again = sm.negative_log_likelihood(y)
    lg = sm.logits.detach().double()
    assert abs(float(plain) - float(F.cross_entropy(lg, y))) < 1e-5
    assert abs(float(smooth) - float(F.cross_entropy(lg, y, label_smoothing=0.2))) < 1e-5
    assert float(again) == float(plain) and float(smooth) != float(plain)
    sm.negative_log_likelihood(y, 0.2)
    assert float(sm.errors(y)) == float(ref.softmax_xent(lg, y)[1])     # the errors reuse the smoothed launch


# --------------------------------------------------------------------------- configuration
def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.05,
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    m = Cifar10_model(cfg)
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    return m


@pytest.fixture(autouse=True)
def dropout_back_on():
    yield
    Dropout.SetDropoutOn(); Crop.SetRandCropOn()


@pytest.mark.parametrize("bad", [-0.1, 1.5, float("nan"), float("inf"), True, False, "0.1", None, [0.1], 1 + 0j])
def test_invalid_values_are_refused(bad):
    m = _cifar(label_smoothing=bad)
    with pytest.raises(ValueError, match="label_smoothing"):
        m.compile_iter_fns("avg")


@pytest.mark.parametrize("good", [0, 0.0, 0.1, 1, 1.0, np.float32(0.2), np.float64(0.3)])
def test_valid_values_are_accepted(good):
    m = _cifar(label_smoothing=good)
    m.compile_iter_fns("avg")
    assert isinstance(m.label_smoothing, float) and m.label_smoothing == float(good)


def test_gans_refuse_a_nonzero_epsilon():
    from theanompi_b200.models.lasagne_model_zoo.lsgan import LSGAN, NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    for cls in (NativeWGAN, NativeLSGAN, WGAN, LSGAN):
        assert cls.supports_label_smoothing is False
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", label_smoothing=0.1, data_kwargs=dict(n_synthetic=128)))
        with pytest.raises(ValueError, match="label_smoothing.*AlexNet, GoogLeNet"):
            m.compile_iter_fns("avg")
        cls(dict(verbose=False, rank=0, size=1, device="cpu", label_smoothing=0.0, data_kwargs=dict(n_synthetic=128))).compile_iter_fns("avg")


def _train(m, n, rec):
    for i in range(n):
        m.train_iter(i, rec)


def test_zero_is_an_absent_key():
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    a, b = _cifar(), _cifar(label_smoothing=0.0)
    a.compile_iter_fns("avg"); b.compile_iter_fns("avg")
    _train(a, 4, rec); _train(b, 4, rec)
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)


# --------------------------------------------------------------------------- training steps
def _step_logits(m, step):
    """Run one training step of ``m`` and return (recorded cost, the logits and labels of that step)."""
    seen = {}
    fwd = m.forward

    def spy(x):
        out = fwd(x)
        seen["logits"] = out.detach().double().clone()
        return out
    m.forward = spy
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.train_iter(step, rec)
    m.forward = fwd
    return float(rec.train_info["cost"][-1]), seen["logits"], m.y_in.clone()


def test_cifar_step_records_the_smoothed_loss_and_validates_without_it():
    m = _cifar(label_smoothing=0.1)
    m.compile_iter_fns("avg")
    for i in range(3):
        cost, lg, y = _step_logits(m, i)
        assert abs(cost - float(F.cross_entropy(lg, y, label_smoothing=0.1))) < 1e-5, i
        assert abs(cost - float(F.cross_entropy(lg, y))) > 1e-4, i
    # validation: plain NLL of the eval-mode logits
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.reset_iter("val")
    seen = {}
    fwd = m.forward
    m.forward = lambda x: seen.setdefault("lg", fwd(x))
    m.val_iter(0, rec)
    m.forward = fwd
    lg = seen["lg"].detach().double()
    y = m.shared_y[:m.batch_size]
    assert abs(float(rec.val_info["cost"][-1]) - float(F.cross_entropy(lg, y))) < 1e-5


def test_smoothing_changes_the_update():
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    a, b = _cifar(), _cifar(label_smoothing=0.1)
    a.compile_iter_fns("avg"); b.compile_iter_fns("avg")
    _train(a, 2, rec); _train(b, 2, rec)
    assert not torch.equal(a.arena.W, b.arena.W)


def test_grad_accum_micro_steps_smooth():
    """grad_accum = 2: every micro-step kind records the smoothed loss of its own logits."""
    m = _cifar(batch_size=8, grad_accum=2, label_smoothing=0.2)
    m.compile_iter_fns("avg")
    for i in range(4):
        cost, lg, y = _step_logits(m, i)
        assert abs(cost - float(F.cross_entropy(lg, y, label_smoothing=0.2))) < 1e-5, i


def test_googlenet_step_smooths_the_aux_heads():
    from theanompi_b200.models.googlenet import GoogLeNet
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    m = GoogLeNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, n_class=8, no_paraload=True,
                       label_smoothing=0.1, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))
    m.compile_iter_fns("avg")
    Dropout.SetDropoutOn()
    heads = [m.output_layer, m.aux1.softmax_layer, m.aux2.softmax_layer]
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.train_iter(0, rec)
    y = m.y_in
    parts = [float(F.cross_entropy(h.logits.detach().double(), y, label_smoothing=0.1)) for h in heads]
    want = parts[0] + 0.3 * parts[1] + 0.3 * parts[2]
    assert abs(float(rec.train_info["cost"][-1]) - want) < 1e-4 * max(1.0, want)
    for h in heads:                                                       # every head's cached launch is the smoothed one
        assert h._cache[1] == 0.1


def test_lstm_trains_smoothed_and_validates_plain():
    from theanompi_b200.models.lstm import LSTM
    layers2.reseed()
    m = LSTM(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, label_smoothing=0.3,
                  data_kwargs=dict(n_synthetic=96, n_words=200)))
    m.compile_iter_fns("avg")
    seen = []
    fl = m.forward_logits

    def spy(x, mk):
        out = fl(x, mk)
        seen.append(out.detach().double().clone())
        return out
    m.forward_logits = spy
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    ys = []
    orig_to = m._to

    def to(x, mk, y):
        t = orig_to(x, mk, y)
        ys.append(t[2])
        return t
    m._to = to
    m.train_iter(0, rec)
    assert abs(float(rec.train_info["cost"][-1]) - float(F.cross_entropy(seen[0], ys[0], label_smoothing=0.3))) < 1e-5
    seen.clear(); ys.clear()
    m.val_iter(1, rec)
    want = np.mean([float(F.cross_entropy(lg, y)) for lg, y in zip(seen, ys)])
    assert abs(float(rec.val_info["cost"][-1]) - want) < 1e-5


def test_torch_twin_step_matches_cross_entropy():
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50Torch
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    m = ResNet50Torch(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, blocks=(1, 1, 1, 1),
                           no_paraload=True, n_class=8, label_smoothing=0.1,
                           data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))
    m.compile_iter_fns("avg")
    seen = {}
    fwd = m.forward

    def spy(x):
        out = fwd(x)
        seen["lg"] = out.detach().double().clone()
        return out
    m.forward = spy
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.train_iter(0, rec)
    assert abs(float(rec.train_info["cost"][-1]) - float(F.cross_entropy(seen["lg"], m.y_in, label_smoothing=0.1))) < 1e-5
    c, _, _ = m.val_fn(0)                                                 # eval mode: plain NLL of the eval-mode logits
    assert abs(float(c) - float(F.cross_entropy(seen["lg"], m.shared_y[:4]))) < 1e-5


# --------------------------------------------------------------------------- distributed
def test_rule_bsp_cdd_two_gloo_ranks(tmp_path, monkeypatch):
    """BSP sync_type='cdd' over the split 'ar' strategy with label_smoothing in rule.model_config: the key reaches both workers
    (an invalid value stops them at compile_iter_fns) and the run completes with the smoothed training cost recorded."""
    import subprocess
    import theanompi_b200 as tm
    monkeypatch.chdir(tmp_path)
    tm.BSP.sync_type, tm.BSP.exch_strategy = "cdd", "ar"
    rcs = {}
    for eps in (0.1, 1.5):
        rule = tm.BSP()
        rule.model_config = dict(batch_size=16, file_batch_size=16, n_epochs=1, learning_rate=0.01, max_batches=6, printFreq=4,
                                 label_smoothing=eps, data_kwargs=dict(n_synthetic=320, synthetic=True))
        rule.env["OMP_NUM_THREADS"] = "2"
        rule.init(devices=["cpu0", "cpu1"], modelfile="theanompi_b200.models.cifar10", modelclass="Cifar10_model")
        try:
            rcs[eps] = rule.proc.wait(timeout=300)
        except subprocess.TimeoutExpired:
            rule.proc.kill()
            raise
        if eps == 0.1:
            with open(tmp_path / "inforec" / "inforec.pkl", "rb") as f:
                costs = [c for _, c, _ in pickle.load(f)["train_info"]]
            assert costs and all(math.isfinite(c) and c > 0 for c in costs), costs
    assert rcs[0.1] == 0 and rcs[1.5] != 0, rcs
