"""Sharpness-aware minimization on the H100.  Kernels: ``sam_norm`` against an fp64 norm, ``sam_perturb`` and ``sam_restore`` bit for bit
against ``ops/reference.py`` given the record, on the AlexNet and ResNet50 arena layouts, bf16 (W and H) and tf32 (W only), SAM and ASAM,
and a NaN record that leaves W and H as they are.  Models (in subprocesses, ``TMPI_DETERMINISTIC=1``): AlexNet bf16 / tf32 and
Wide_ResNet-28-4 with Adam replay the captured SAM step bit for bit like the eager step, equal a manual composition on a second model,
never arm the FC epilogue, and run exactly one more training forward and backward plus four launches per step; ResNet50's running
statistics are those of the first pass."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from theanompi_b200.ops import reference as ref  # noqa: E402

IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))
_SHAPES = {}


def _layout(which):
    """The parameter shapes of the real model, in arena order (built once on the CPU)."""
    if which not in _SHAPES:
        from theanompi_b200.models import layers2
        layers2.reseed()
        if which == "alexnet":
            from theanompi_b200.models.alex_net import AlexNet as cls
            cfg = dict(batch_size=16, file_batch_size=16, no_paraload=True, n_class=1000,
                       data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
        else:
            from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50 as cls
            cfg = dict(batch_size=8, file_batch_size=8, no_paraload=True, n_class=1000,
                       data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", **cfg))
        _SHAPES[which] = [tuple(p.shape) for p in m.params]
    return _SHAPES[which]


def _arena(which, shadow, seed=0):
    from theanompi_b200.parallel.arena import FlatArena
    g = torch.Generator().manual_seed(seed)
    params = [torch.randn(s, generator=g) * 0.05 for s in _layout(which)]
    a = FlatArena(params, device="cuda", shadow=shadow)
    a.G.copy_((torch.randn(a.numel, generator=g) * 1e-3).cuda())
    return a


def _fp64_norm(a, adaptive):
    sq = 0.0
    for o, s in zip(a.offsets, a.sizes):
        w, g = a.W[o:o + s].double(), a.G[o:o + s].double()
        v = (w.float() * g.float()).double() if adaptive else g
        sq += float((v * v).sum())
    return float(np.sqrt(sq))


@pytest.mark.parametrize("which", ["alexnet", "resnet50"])
@pytest.mark.parametrize("shadow", [True, False], ids=["bf16", "tf32"])
@pytest.mark.parametrize("adaptive", [False, True], ids=["sam", "asam"])
def test_kernels_match_reference(which, shadow, adaptive):
    from theanompi_b200.ops import cuda_impl
    a = _arena(which, shadow)
    rho = 1.0 if adaptive else 0.05
    partial = torch.zeros(a.n_blocks, dtype=torch.float32, device="cuda")
    rec = torch.zeros(4, dtype=torch.float32, device="cuda")
    cuda_impl.sam_norm(a, rho, adaptive, partial, rec)
    torch.cuda.synchronize()
    n, s, finite = float(rec[0]), float(rec[1]), int(rec[2:3].view(torch.int32))
    # fp32 squares and per-block fp32 sums (a tree of 15 additions) before the fp64 total: well within 1e-5 of the fp64 norm
    want = _fp64_norm(a, adaptive)
    assert finite == 1 and abs(n - want) <= 1e-5 * want, (n, want)
    assert (s, True) == ref.sam_scale(np.float32(n), rho)
    w0, g0 = a.W.clone(), a.G.clone()
    h0 = a.H.clone() if shadow else None
    P = torch.full_like(a.W, float("nan"))
    cuda_impl.sam_perturb(a, P, rec, adaptive)
    wr, pr = w0.cpu(), torch.empty(a.numel)
    hr = torch.empty(a.numel, dtype=torch.bfloat16) if shadow else None
    ref.sam_perturb(wr, g0.cpu(), pr, s, True, a.offsets, a.sizes, adaptive, w_half=hr)
    torch.cuda.synchronize()
    assert torch.equal(a.W.cpu(), wr) and torch.equal(P, w0) and torch.equal(a.G, g0)
    if shadow:
        assert torch.equal(a.H.cpu(), hr)
    assert not torch.equal(a.W, w0)
    cuda_impl.sam_restore(a, P)
    torch.cuda.synchronize()
    assert torch.equal(a.W, w0) and (not shadow or torch.equal(a.H, h0))


@pytest.mark.parametrize("shadow", [True, False], ids=["bf16", "tf32"])
def test_nan_record_leaves_w_and_h(shadow):
    from theanompi_b200.ops import cuda_impl
    a = _arena("alexnet", shadow, seed=1)
    a.G[12345] = float("nan")
    partial = torch.zeros(a.n_blocks, dtype=torch.float32, device="cuda")
    rec = torch.zeros(4, dtype=torch.float32, device="cuda")
    cuda_impl.sam_norm(a, 0.05, False, partial, rec)
    w0, h0 = a.W.clone(), (a.H.clone() if shadow else None)
    P = torch.zeros_like(a.W)
    cuda_impl.sam_perturb(a, P, rec, False)
    torch.cuda.synchronize()
    assert not np.isfinite(float(rec[0])) and int(rec[2:3].view(torch.int32)) == 0
    assert torch.equal(a.W, w0) and torch.equal(P, w0) and (not shadow or torch.equal(a.H, h0))


# --------------------------------------------------------------------------- models (subprocesses, deterministic mode)
MODELS = {
    "alexnet_bf16": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, no_paraload=True, **IMNET)),
    "alexnet_tf32": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, no_paraload=True, dtype="tf32",
                                                                       **IMNET)),
    "wrn_adam": ("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
                 dict(batch_size=32, file_batch_size=32, depth=28, widen=4, learning_rate=1e-3,
                      data_kwargs=dict(n_synthetic=256, synthetic=True))),
    "resnet50": ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50",
                 dict(batch_size=64, file_batch_size=64, no_paraload=True, **IMNET)),
}
SAM = dict(rho=0.05)


def _model(which, monitor_grad=False, **kw):
    import importlib
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import cuda_impl
    mod, cls, cfg = MODELS[which]
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    cuda_impl._STEP.clear()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", **dict(cfg, **kw)))
    m.rand_crop = False
    m.monitor_grad = monitor_grad            # True: the FC epilogue is not armed (utils/opt.py: FlatSGD.arm)
    m.compile_iter_fns("avg")
    return m


def _state(m):
    out = [m.arena.W.clone(), m.arena.U.clone(), m.arena.G.clone()] + ([m.arena.H.clone()] if m.arena.H is not None else [])
    return out + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _rec():
    from theanompi_b200.utils.recorder import Recorder
    return Recorder(None, 10 ** 6, "t", False, device="cuda:0")


def _manual(m, cfg):
    """A train_iter_fn for a model built without the key: pass 1, the SAM launches on its arena, pass 2 with frozen statistics, the
    restore and the step tail, as separate pieces."""
    from theanompi_b200.utils.opt import Sam
    sam = Sam(m.arena, cfg)

    def step(subb=0):
        B = m.batch_size
        m.x_in.copy_(m.shared_x[subb * B:(subb + 1) * B])
        m.y_in.copy_(m.shared_y[subb * B:(subb + 1) * B])
        m.n_updates += 1
        out = m._fwd_bwd_eager()
        with torch.no_grad():
            sam.perturb()
        with m.bn_stats_frozen():
            m._train_pass(None)
        with torch.no_grad():
            sam.restore()
            m._tail()
        m._after_step()
        return out
    return step


def _run(which, n, manual=False, **kw):
    """``n`` training steps of a fresh model (its own device step counter): the state after every step, the SAM norms, the model."""
    rec = _rec()
    m = _model(which, monitor_grad=manual, **kw)
    if manual:
        m.train_iter_fn = _manual(m, SAM)
    states, norms = [], []
    for i in range(n):
        m.train_iter(i, rec)
        torch.cuda.synchronize()
        states.append(_state(m))
        norms.append(None if m.sam_opt is None else float(m.sam_norm))
    return states, norms, m


def model_check(which, n=4):
    """The captured SAM step replays bit for bit like the eager one and like the manual composition; no FC epilogue is armed; the
    launches per step are the plain step's (epilogue disarmed) plus one training forward and backward plus four."""
    from theanompi_b200.ops import native
    graph, norms, m = _run(which, n, sam=SAM)
    assert m.captured_steps() == {"step"} and all(np.isfinite(norms)) and min(norms) > 0, norms
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params), "the FC epilogue is armed"
    del m
    eager, enorms, _ = _run(which, n, sam=SAM, cuda_graph=False)
    assert norms == enorms
    man, _, _ = _run(which, n, manual=True, cuda_graph=False)
    for i in range(n):
        assert _same(graph[i], eager[i]), ("graph replay != eager", i)
        assert _same(graph[i], man[i]), ("step != manual composition", i)
    counts = {}
    rec = _rec()
    for key, kw in (("plain", dict(monitor_grad=True)), ("sam", dict(sam=SAM))):
        m = _model(which, cuda_graph=False, **kw)
        m.train_iter(0, rec)
        torch.cuda.synchronize()
        native.reset_launch_count()
        m.train_iter(1, rec)
        torch.cuda.synchronize()
        counts[key] = native.launch_count()
        if key == "plain":
            native.reset_launch_count()
            m._train_pass(None)
            torch.cuda.synchronize()
            counts["pass"] = native.launch_count()
    assert counts["sam"] == counts["plain"] + counts["pass"] + 4, counts
    return counts, norms


def stats_check():
    """ResNet50-64b: the running statistics after a SAM step are those after the first pass alone."""
    rec = _rec()
    on = _model("resnet50", sam=SAM, cuda_graph=False)
    plain = _model("resnet50", cuda_graph=False)

    def pass_one(subb=0):
        plain.x_in.copy_(plain.shared_x[:plain.batch_size]); plain.y_in.copy_(plain.shared_y[:plain.batch_size])
        return plain._fwd_bwd_eager()
    plain.train_iter_fn = pass_one
    on.train_iter(0, rec)
    plain.train_iter(0, rec)
    torch.cuda.synchronize()
    stats = lambda m: [t for l in m._bn_layers() for t in (l.running_mean, l.running_var)]  # noqa: E731
    assert len(stats(on)) == len(stats(plain)) > 100 and _same(stats(on), stats(plain))
    assert not torch.equal(on.arena.W, plain.arena.W)            # the SAM step did update the weights


def _subprocess(code, timeout=1800):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("which", ["alexnet_bf16", "alexnet_tf32", "wrn_adam"])
def test_graph_step_equals_eager_and_manual_composition(which):
    _subprocess("""
import test_gpu_sam as t
print('launches, norms', t.model_check(%r))
print('OK')
""" % which)


def test_resnet50_running_statistics_unchanged_by_pass_two():
    _subprocess("""
import test_gpu_sam as t
t.stats_check()
print('OK')
""")
