"""Per-update lr schedules on the H100: lr_schedule_kernel against ``reference.lr_at``, and scheduled CUDA-graph training against a
schedule-off model that writes the same lr values with set_value before each step (bit-identical arenas under TMPI_DETERMINISTIC=1,
in a subprocess), the launch count, checkpoint / resume, and a two-GPU fused BSP run."""
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

CASES = [
    ("constant", dict(decay="constant")),
    ("warmup", dict(warmup_steps=7, warmup_start=0.1)),
    ("warmup0", dict(warmup_steps=13)),
    ("multistep", dict(warmup_steps=3, decay="multistep", milestones=[3, 10, 11, 20], gamma=0.3)),
    ("multistep_default", dict(decay="multistep", milestones=[1, 5])),
    ("cosine", dict(warmup_steps=5, decay="cosine", final_lr=1e-4)),
    ("cosine_nowarm", dict(decay="cosine")),
    ("poly2", dict(warmup_steps=4, decay="poly", power=2.0)),
    ("poly_frac", dict(decay="poly", power=0.5, final_lr=0.003)),
]


@pytest.mark.parametrize("name, cfg", CASES, ids=[c[0] for c in CASES])
def test_kernel_matches_lr_at(name, cfg):
    """u = 0 … T+5: warm-up, constant and multistep bit-equal (correctly rounded fp64 operations only), cosine and poly within one
    fp32 ulp (cos / pow); the counter is u + 1 after every launch."""
    from theanompi_b200.utils.opt import LrSchedule
    T = 24
    arena = types.SimpleNamespace(hyper=torch.zeros(8, dtype=torch.float32, device="cuda"))
    s = LrSchedule(arena, dict(cfg, total_steps=cfg.get("total_steps", T)), 0.37, T)
    got, cnt = [], []
    for u in range(T + 6):
        s.step()
        got.append(arena.hyper[0].clone()); cnt.append(s.u.clone())
    torch.cuda.synchronize()
    got = np.array([float(g) for g in got], dtype=np.float32)
    want = np.array([s.lr_at(u) for u in range(T + 6)], dtype=np.float32)
    assert [int(c) for c in cnt] == list(range(1, T + 7))
    exact = s.decay in ("constant", "multistep")
    for u in range(T + 6):
        if exact or u < s.warmup_steps:
            assert got[u].view(np.int32) == want[u].view(np.int32), (name, u, got[u], want[u])
        else:
            assert abs(int(got[u].view(np.int32)) - int(want[u].view(np.int32))) <= 1, (name, u, got[u], want[u])
    assert len(set(got.tolist())) > 1 or s.decay == "constant"


# --------------------------------------------------------------------------- graph oracles (subprocess, deterministic mode)
IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))
SCHED = dict(warmup_steps=6, warmup_start=0.05, decay="cosine", total_steps=24, final_lr=1e-4)
MODELS = {
    "alexnet_sgd": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, no_paraload=True, **IMNET),
                    22),
    "wrn_adam": ("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
                 dict(batch_size=16, file_batch_size=32, depth=10, widen=2, learning_rate=1e-3,
                      data_kwargs=dict(n_synthetic=256, synthetic=True)), 14),
    "wrn_lamb": ("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
                 dict(batch_size=16, file_batch_size=32, depth=10, widen=2, optimizer="lamb", learning_rate=1e-3,
                      data_kwargs=dict(n_synthetic=256, synthetic=True)), 14),
    "resnet50_lars_accum4": ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50",
                             dict(batch_size=8, file_batch_size=8, blocks=(1, 1, 1, 1), no_paraload=True, optimizer="lars",
                                  learning_rate=0.5, grad_accum=4, **IMNET), 24),
}


def _model(mod, cls, dev, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device=dev, **cfg))
    m.rand_crop = False
    layers2.Dropout.SetDropoutOff(); layers2.Crop.SetRandCropOff()
    m.compile_iter_fns("avg")
    return m


def _steps(m, n, rec, lrs=None):
    """``n`` training steps; without ``lrs`` record arena.hyper[0] after every update's first step, with ``lrs`` write lrs[u] by
    set_value before it instead."""
    out, u = [], 0
    for i in range(n):
        first = m.grad_accum == 1 or m.micro_step_kind() == "first"
        if first and lrs is not None:
            m.shared_lr.set_value(lrs[u])
        m.train_iter(i, rec)
        if first:
            if lrs is None:
                out.append(m.arena.hyper[0].clone())
            u += 1
    torch.cuda.synchronize()
    return [float(v) for v in out]


def follows_schedule(lrs, peak):
    """``lrs`` are lr_at(u) of SCHED: bit-equal during the warm-up, within one fp32 ulp after it (cosine)."""
    from theanompi_b200.ops.reference import lr_at
    got = np.array(lrs, dtype=np.float32).view(np.int32).astype(np.int64)
    want = np.array([lr_at(u, peak, **SCHED) for u in range(len(lrs))], dtype=np.float32).view(np.int32).astype(np.int64)
    W = SCHED["warmup_steps"]
    return bool((got[:W] == want[:W]).all() and (np.abs(got[W:] - want[W:]) <= 1).all())


def model_oracle(which):
    """Scheduled graph run and set_value run of ``which``: returns (lrs, arenas equal, graphs captured)."""
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.recorder import Recorder
    mod, cls, cfg, n = MODELS[which]
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    cuda_impl._STEP.clear()
    a = _model(mod, cls, "cuda:0", lr_schedule=SCHED, **cfg)
    if which == "alexnet_sgd":
        assert any(getattr(p, "sgd_epilogue", None) is not None for p in a.arena.params), "the FC SGD epilogue is not armed"
    lrs = _steps(a, n, rec)
    assert follows_schedule(lrs, float(a.learning_rate)), lrs
    graphs = bool(a.captured_steps())
    wa = [a.arena.W.clone(), a.arena.U.clone()]
    a.cleanup()
    del a
    cuda_impl._STEP.clear()
    b = _model(mod, cls, "cuda:0", **cfg)
    _steps(b, n, rec, lrs)
    same = torch.equal(wa[0], b.arena.W) and torch.equal(wa[1], b.arena.U)
    b.cleanup()
    return lrs, same, graphs


def lstm_oracle():
    """The LSTM with batches alternating between the 16- and 48-step buckets: one counter drives both bucket graphs."""
    from theanompi_b200.models import layers2
    from theanompi_b200.models.lstm import LSTM
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.recorder import Recorder
    rs = np.random.RandomState(0)
    B = 16
    batches = []
    for i in range(16):
        L = 10 if i % 2 == 0 else 40
        batches.append((rs.randint(2, 500, (B, L)).astype(np.int64), np.ones((B, L), np.float32), rs.randint(0, 2, B).astype(np.int64)))
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    runs = []
    for sched in (SCHED, None):
        layers2.reseed()
        m = LSTM(dict(verbose=False, rank=0, size=1, device="cuda:0", optimizer="rmsprop", learning_rate=1e-3, lr_schedule=sched,
                      data_kwargs=dict(n_synthetic=64, n_words=500)))
        m.compile_iter_fns("avg")
        cuda_impl._STEP.clear()                       # the same dropout masks in both runs
        m._train_it = iter(batches)
        lrs = runs[0][0] if runs else None
        got = []
        for i in range(len(batches)):
            if lrs is not None:
                m.shared_lr.set_value(lrs[i])
            m.train_iter(i, rec)
            got.append(m.arena.hyper[0].clone())
        torch.cuda.synchronize()
        runs.append(([float(v) for v in got], m.arena.W.clone(), sorted(m.captured_steps())))
    return runs


def _subprocess(code, timeout=900):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("which", list(MODELS))
def test_graph_schedule_matches_set_value_oracle(which):
    """AlexNet-128b bf16 (SGD, FC weight-gradient epilogue armed: it reads the new lr inside backward), Wide_ResNet with Adam and
    LAMB, ResNet50 with LARS at grad_accum = 4 (lr changes at 'first' micro-steps only): the scheduled CUDA-graph run and a
    schedule-off run that writes the recorded lr values with set_value are bit-identical."""
    _subprocess("""
import test_gpu_lr_schedule as t
lrs, same, graphs = t.model_oracle(%r)
print('lrs', lrs[:3], '...', lrs[-2:], 'graphs', graphs, 'identical', same)
assert graphs and same and len(set(lrs)) > len(lrs) // 2
print('OK')
""" % which)


def test_lstm_two_buckets_share_one_counter():
    _subprocess("""
import test_gpu_lr_schedule as t
(la, wa, ga), (lb, wb, gb) = t.lstm_oracle()
print('lrs', la[:4], 'graphs', ga, 'max |dW|', float((wa - wb).abs().max()))
assert ga == [16, 48], ga
assert la == lb and len(set(la)) > 8 and t.follows_schedule(la, 1e-3)
assert t.torch.equal(wa, wb)
print('OK')
""")


def test_launch_count_one_more_per_update():
    from theanompi_b200.ops import native
    from theanompi_b200.models import layers2
    counts = {}
    try:
        mod, cls, cfg, _ = MODELS["alexnet_sgd"]
        for name, sched in (("off", None), ("on", SCHED)):
            m = _model(mod, cls, "cuda:0", cuda_graph=False, lr_schedule=sched, **dict(cfg, batch_size=16, file_batch_size=16))
            for _ in range(2):
                torch.cuda.synchronize()
                native.reset_launch_count()
                m.forward_backward(0)
                torch.cuda.synchronize()
                counts[name] = native.launch_count()
        mod, cls, cfg, _ = MODELS["resnet50_lars_accum4"]
        for name, sched in (("accum_off", None), ("accum_on", SCHED)):
            m = _model(mod, cls, "cuda:0", cuda_graph=False, lr_schedule=sched, **cfg)
            for k in range(4):
                kind = m.micro_step_kind()
                torch.cuda.synchronize()
                native.reset_launch_count()
                m.forward_backward(0)
                torch.cuda.synchronize()
                counts[(name, kind)] = native.launch_count()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(counts)
    assert counts["on"] == counts["off"] + 1
    assert counts[("accum_on", "first")] == counts[("accum_off", "first")] + 1
    for kind in ("mid", "last"):
        assert counts[("accum_on", kind)] == counts[("accum_off", kind)]


def resume_check(tmp):
    """Cifar10_model with graphs, warm-up of 8 updates: a checkpoint after 4 updates resumed in a fresh model ends bit-identical to an
    uninterrupted run after 8."""
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    from theanompi_b200.utils.recorder import Recorder
    cfg = dict(batch_size=16, file_batch_size=16, learning_rate=0.05, lr_schedule=dict(warmup_steps=8, total_steps=20),
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    mod, cls = "theanompi_b200.models.cifar10", "Cifar10_model"
    cuda_impl._STEP.clear()
    a = _model(mod, cls, "cuda:0", **cfg)
    _steps(a, 4, rec); a.reset_iter("train"); lr_a = _steps(a, 4, rec)
    cuda_impl._STEP.clear()
    b = _model(mod, cls, "cuda:0", **cfg)
    _steps(b, 4, rec); b.reset_iter("train")
    save_checkpoint(b, os.path.join(tmp, "ckpt.pt"))
    c = _model(mod, cls, "cuda:0", **cfg)
    load_checkpoint(c, os.path.join(tmp, "ckpt.pt"))
    assert int(c.lr_sched.u) == 4 and c.shared_lr.get_value() == float(c.lr_sched.lr_at(3))
    lr_c = _steps(c, 4, rec)
    return lr_a, lr_c, torch.equal(a.arena.W, c.arena.W) and torch.equal(a.arena.U, c.arena.U)


def test_checkpoint_resume_mid_warmup(tmp_path):
    _subprocess("""
import test_gpu_lr_schedule as t
from theanompi_b200.ops.reference import lr_at
t.lr_at = lr_at
lr_a, lr_c, same = t.resume_check(%r)
print('lrs', lr_a, lr_c, 'identical', same)
assert lr_a == lr_c == [float(t.lr_at(u, 0.05, warmup_steps=8)) for u in range(4, 8)]
assert same
print('OK')
""" % str(tmp_path))


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_fused_bsp_two_gpus_follows_the_schedule(tmp_path):
    """BSP sync_type='cdd' over the fused exchange on two GPUs: both ranks' hyper[0] follow lr_at, and the arena equals a
    schedule-off run that writes the same values with set_value."""
    out = {}
    for k, mode in enumerate(("sched", "oracle")):
        cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
               "--master-port", str(29660 + k), os.path.join(HERE, "mp_lr_schedule_gpu.py"), mode, str(tmp_path)]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600, cwd=ROOT,
                           env=dict(os.environ, TMPI_DETERMINISTIC="1"))
        assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-4000:]
        out[mode] = [torch.load(tmp_path / ("%s_%d.pt" % (mode, rank))) for rank in range(2)]
    for rank in range(2):
        assert out["sched"][rank]["lrs"] == out["oracle"][rank]["lrs"]
        assert torch.equal(out["sched"][rank]["W"], out["oracle"][rank]["W"])
    assert torch.equal(out["sched"][0]["W"], out["sched"][1]["W"])
