"""Per-update learning-rate schedules (``config['lr_schedule']``) on the CPU reference path: ``reference.lr_at`` against hand-computed
values, the validation errors, a scheduled run against a run that sets each update's lr by hand (sgd, lars, grad_accum), the dropped
window, adjust_hyperp, checkpoint / resume, the refusals and a two-rank BSP 'cdd' run over the split 'ar' strategy."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops.reference import lr_at  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402

f32 = np.float32


# --------------------------------------------------------------------------- lr_at
def test_constant_and_warmup():
    for u in (0, 1, 5, 100):
        assert lr_at(u, 0.1) == f32(0.1)
    W = 4
    want = {0: 0.0, 1: 0.025, 3: 0.075, 4: 0.1, 7: 0.1, 50: 0.1}
    for u, v in want.items():
        assert lr_at(u, 0.1, warmup_steps=W) == f32(v), u
    # warmup_start s: peak·(s + (1 − s)·u / W)
    assert lr_at(0, 2.0, warmup_steps=4, warmup_start=0.25) == f32(0.5)
    assert lr_at(2, 2.0, warmup_steps=4, warmup_start=0.25) == f32(2.0 * (0.25 + 0.75 * 2 / 4))
    assert lr_at(3, 2.0, warmup_steps=4, warmup_start=0.25) == f32(2.0 * (0.25 + 0.75 * 3 / 4))
    assert lr_at(4, 2.0, warmup_steps=4, warmup_start=0.25) == f32(2.0)
    assert lr_at(0, 2.0, warmup_steps=4, warmup_start=1.0) == f32(2.0)


@pytest.mark.parametrize("W", [0, 10])
def test_cosine(W):
    T, peak, fin = 110, 0.4, 0.01
    kw = dict(decay="cosine", warmup_steps=W, total_steps=T, final_lr=fin)
    assert lr_at(W, peak, **kw) == f32(peak)                                          # p = 0
    assert lr_at(W + (T - W) // 2, peak, **kw) == f32(fin + (peak - fin) * 0.5)        # p = ½: cos = 0 up to rounding
    p = (T - 1 - W) / (T - W)
    assert lr_at(T - 1, peak, **kw) == f32(fin + (peak - fin) * 0.5 * (1 + math.cos(math.pi * p)))
    assert lr_at(T, peak, **kw) == f32(fin) and lr_at(T + 10, peak, **kw) == f32(fin)  # clamped at p = 1
    if W:
        assert lr_at(0, peak, **kw) == f32(0.0) and lr_at(1, peak, **kw) == f32(peak / W)
        assert lr_at(W - 1, peak, **kw) == f32(peak * (W - 1) / W)


@pytest.mark.parametrize("W", [0, 10])
def test_poly(W):
    T, peak = 100 + W, 0.4
    kw = dict(decay="poly", warmup_steps=W, total_steps=T, power=2.0)
    assert lr_at(W, peak, **kw) == f32(peak)
    assert lr_at(W + (T - W) // 2, peak, **kw) == f32(peak * 0.25)
    assert lr_at(T - 1, peak, **kw) == f32(peak * (1 / (T - W)) ** 2)
    assert lr_at(T, peak, **kw) == f32(0.0) and lr_at(T + 10, peak, **kw) == f32(0.0)
    assert lr_at(W + 25, peak, decay="poly", warmup_steps=W, total_steps=T, final_lr=0.1) == f32(0.1 + 0.3 * 0.75)   # power 1
    if W:
        assert lr_at(W - 1, peak, **kw) == f32(peak * (W - 1) / W)


@pytest.mark.parametrize("W", [0, 3])
def test_multistep_edges(W):
    kw = dict(decay="multistep", warmup_steps=W, milestones=[5, 9], gamma=0.5)
    want = {4: 1.0, 5: 0.5, 8: 0.5, 9: 0.25, 100: 0.25}
    for u, v in want.items():
        assert lr_at(u, 1.0, **kw) == f32(v), u
    assert lr_at(10, 0.1, decay="multistep", milestones=[10]) == f32(0.1 * 0.1)      # default gamma 0.1, u equal to the milestone
    if W:
        assert lr_at(W - 1, 1.0, **kw) == f32((W - 1) / W) and lr_at(W, 1.0, **kw) == f32(1.0)


# --------------------------------------------------------------------------- models
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


SCHED = dict(warmup_steps=4, warmup_start=0.1, decay="cosine", total_steps=14, final_lr=0.001)


@pytest.mark.parametrize("bad, key", [
    (dict(foo=1), "foo"), (dict(decay="linear"), "decay"), (dict(warmup_steps=10, total_steps=10), "total_steps"),
    (dict(warmup_steps=-1), "warmup_steps"), (dict(warmup_start=1.5), "warmup_start"), (dict(warmup_start=-0.1), "warmup_start"),
    (dict(decay="multistep", milestones=[5, 3]), "milestones"), (dict(decay="multistep", milestones=[4, 4]), "milestones"),
    (dict(decay="multistep", milestones=list(range(1, 10))), "milestones"),
    (dict(decay="multistep", warmup_steps=5, milestones=[3]), "milestones"), (dict(decay="poly", power=-1.0), "power"),
    (dict(warmup_steps=2.5), "warmup_steps"), ([("decay", "cosine")], "lr_schedule must be a dict"),
])
def test_validation_errors(bad, key):
    m = _cifar(lr_schedule=bad)
    with pytest.raises(ValueError, match=key):
        m.compile_iter_fns("avg")


def test_updates_per_epoch_and_default_total():
    m = _cifar(batch_size=8, grad_accum=2, n_epochs=3, lr_schedule=dict(decay="cosine"))
    m.compile_iter_fns("avg")
    assert m.updates_per_epoch == m.data.n_batch_train * 2 // 2
    assert m.lr_sched.total_steps == 3 * m.updates_per_epoch
    off = _cifar()
    off.compile_iter_fns("avg")
    assert off.lr_sched is None


def _run(m, n_updates, rec, oracle=None, start=0):
    """Train ``n_updates`` updates; with ``oracle`` (a schedule-off model's lr function) set each update's lr by hand first.
    Returns the lr of every update, read from arena.hyper[0] after its first micro-step."""
    lrs, u, i = [], start, 0
    while u < start + n_updates:
        first = m.grad_accum == 1 or m.micro_step_kind() == "first"
        if first and oracle is not None:
            m.shared_lr.set_value(oracle(u))
        m.train_iter(i, rec)
        i += 1
        if first:
            lrs.append(float(m.arena.hyper[0]))
        if m.grad_accum == 1 or m.micro_step_kind() == "first":
            u += 1
    return lrs


@pytest.mark.parametrize("kw", [dict(), dict(optimizer="lars", learning_rate=1.0), dict(batch_size=8, grad_accum=3, learning_rate=0.01)],
                         ids=["sgd", "lars", "grad_accum3"])
def test_schedule_matches_set_value_oracle(kw):
    """A scheduled run and a schedule-off run that writes lr_at(u) with set_value before each update: bit-identical arenas after 12
    updates.  Under grad_accum every micro-step of a window uses its update's lr and u counts windows."""
    a = _cifar(lr_schedule=SCHED, **kw)
    b = _cifar(**kw)
    a.compile_iter_fns("avg"); b.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    la = _run(a, 12, rec)
    lb = _run(b, 12, rec, oracle=a.lr_sched.lr_at)
    assert int(a.lr_sched.u) == 12 and a.n_updates == b.n_updates == 12
    assert la == lb == [float(a.lr_sched.lr_at(u)) for u in range(12)]
    assert len(set(la)) > 8                                             # the lr really changes every update
    assert bool(torch.isfinite(a.arena.W).all())
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)


def test_dropped_window_gives_back_its_update_index():
    m = _cifar(batch_size=8, grad_accum=3, lr_schedule=dict(warmup_steps=10, total_steps=20))
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(5):                                                  # one window, then 2 micro-steps of the next
        m.train_iter(i, rec)
    assert int(m.lr_sched.u) == 2 and float(m.arena.hyper[0]) == float(m.lr_sched.lr_at(1))
    m.reset_iter("train")
    assert int(m.lr_sched.u) == 1 and m.n_discarded == 2
    assert m.shared_lr.get_value() == float(m.lr_sched.lr_at(0))        # the host sees the lr of the last update
    m.train_iter(0, rec)
    assert int(m.lr_sched.u) == 2 and float(m.arena.hyper[0]) == float(m.lr_sched.lr_at(1))   # the next window reuses its lr
    for i in range(2):
        m.train_iter(i, rec)
    m.reset_iter("train")                                               # nothing open: nothing given back
    assert int(m.lr_sched.u) == 2 and m.shared_lr.get_value() == float(m.lr_sched.lr_at(1))


def test_adjust_hyperp_leaves_a_scheduled_lr_alone():
    m = _cifar(lr_schedule=dict(decay="multistep", milestones=[100]))
    m.lr_policy, m.lr_step = "step", [0, 1]
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.train_iter(0, rec)
    before = float(m.arena.hyper[0])
    m.reset_iter("train")
    m.adjust_hyperp(0); m.adjust_hyperp(1)
    assert float(m.arena.hyper[0]) == before == m.shared_lr.get_value()
    m.train_iter(0, rec)
    assert float(m.arena.hyper[0]) == float(f32(0.05))
    off = _cifar()
    off.lr_policy, off.lr_step = "step", [0]
    off.compile_iter_fns("avg")
    off.adjust_hyperp(0)
    assert off.shared_lr.get_value() == pytest.approx(0.005)            # without a schedule the per-epoch policy still acts


def test_checkpoint_resume_is_bit_identical(tmp_path):
    """Checkpoint at update 5 (the end of an epoch), resume in a fresh model: the same arena after 12 updates as a run that was
    never interrupted."""
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    straight = _cifar(lr_schedule=SCHED)
    straight.compile_iter_fns("avg")
    _run(straight, 5, rec)
    straight.reset_iter("train")
    _run(straight, 7, rec, start=5)

    first = _cifar(lr_schedule=SCHED)
    first.compile_iter_fns("avg")
    _run(first, 5, rec)
    first.reset_iter("train")
    save_checkpoint(first, str(tmp_path / "ckpt.pt"))
    resumed = _cifar(lr_schedule=SCHED)
    resumed.compile_iter_fns("avg")
    load_checkpoint(resumed, str(tmp_path / "ckpt.pt"))
    assert int(resumed.lr_sched.u) == 5 and resumed.shared_lr.get_value() == float(resumed.lr_sched.lr_at(4))
    lrs = _run(resumed, 7, rec, start=5)
    assert lrs == [float(resumed.lr_sched.lr_at(u)) for u in range(5, 12)]
    assert torch.equal(resumed.arena.W, straight.arena.W) and torch.equal(resumed.arena.U, straight.arena.U)


def test_lstm_schedule_and_checkpoint_state():
    from theanompi_b200.models.lstm import LSTM
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, optimizer="sgd", learning_rate=0.1,
               lr_schedule=dict(warmup_steps=3, decay="poly", power=2.0, total_steps=9), data_kwargs=dict(n_synthetic=96, n_words=200))
    m = LSTM(cfg)
    m.compile_iter_fns("avg")
    assert m.updates_per_epoch == m.data.n_batch_train
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    lrs = []
    for i in range(6):
        m.train_iter(i, rec)
        lrs.append(float(m.arena.hyper[0]))
    assert lrs == [float(lr_at(u, 0.1, "poly", 3, 0.0, 9, 0.0, 2.0)) for u in range(6)]
    assert m.extra_state()["lr_schedule"] == {"u": 6}
    m.reset_iter("train")
    assert m.shared_lr.get_value() == lrs[-1]


def test_gan_and_torch_twin_refusals():
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    from theanompi_b200.models.lstm import LSTMTorch
    from theanompi_b200.models.torch_base import TorchModelBase
    for cls in (NativeWGAN, WGAN, LSTMTorch, TorchModelBase):
        assert cls.supports_lr_schedule is False
    models = [NativeWGAN(dict(verbose=False, rank=0, size=1, device="cpu", lr_schedule=dict(decay="cosine"),
                              data_kwargs=dict(n_synthetic=128))),
              WGAN(dict(verbose=False, rank=0, size=1, device="cpu", lr_schedule=dict(decay="cosine"), data_kwargs=dict(n_synthetic=128))),
              LSTMTorch(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, lr_schedule=dict(decay="cosine"),
                             data_kwargs=dict(n_synthetic=64, n_words=200)))]
    for m in models:
        with pytest.raises(ValueError, match="lr_schedule is not supported"):
            m.compile_iter_fns("avg")


def test_bsp_cdd_two_gloo_ranks_follow_the_schedule():
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT="29851", OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_lr_schedule_checks.py"), "bsp_cdd"],
                              env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(2)]
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=240)[0])
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, o[-3000:])
