"""Stochastic depth on the H100: ``drop_path_draw_kernel`` against ``reference.drop_path_draw`` bit for bit, its device counter and
CUDA-graph replays, the batch-norm kernels and the scaled add with a drop row against fp64 torch autograd of the formula, native
ResNet50 / Wide_ResNet with drop-path against their CPU reference path replaying the device tables, bit-identity under
TMPI_DETERMINISTIC=1 (in a subprocess) of graph replay with eager steps and of a table forced to ones with no key, launch counts, and
validation / inference that never drop."""
import math
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

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.ops import drop_path, precision  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

DEV = "cuda:0"


def rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


# --------------------------------------------------------------------------- the draw
@pytest.mark.parametrize("p,L,B,rank,step,seed", [(0.1, 16, 64, 0, 0, 0x5EED), (0.5, 50, 37, 3, 2 ** 33 + 5, 2 ** 40 + 3),
                                                  (0.3, 12, 128, 1, 7, 1), (0.9, 2, 1, 0, 3, 12345), (0.2, 1, 8, 2, 1, 0),
                                                  (0.99, 4, 256, 7, 2 ** 63 - 2, 2 ** 64 - 1)])
def test_draw_kernel_matches_reference(p, L, B, rank, step, seed):
    from theanompi_b200.ops import cuda_impl
    old = ops.rng_state()["seed"]
    ops.seed_dropout(seed)
    try:
        dp = drop_path.DropPath(p, L, B, rank, DEV)
        st = torch.full((1,), step, dtype=torch.int64, device=DEV)
        got = cuda_impl.drop_path_draw(dp, st, dp.table).cpu()
        want = ref.drop_path_draw(dp.rates, seed, rank, step, B)
        assert torch.equal(got, want)
    finally:
        ops.seed_dropout(old)


def test_draw_reads_the_device_counter_and_graph_replays_draw_anew():
    from theanompi_b200.ops import cuda_impl
    ops.seed_dropout(9)
    dp = drop_path.DropPath(0.5, 6, 64, 0, DEV)
    st = torch.full((1,), 100, dtype=torch.int64, device=DEV)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):                                   # warm-up outside the capture
        cuda_impl.drop_path_draw(dp, st, dp.table)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        cuda_impl.drop_path_draw(dp, st, dp.table)
        torch.ops.aten.add_(st, 1)
    tabs = []
    for _ in range(3):
        g.replay()
        torch.cuda.synchronize()
        tabs.append(dp.table.cpu().clone())
    for k, t in enumerate(tabs):
        assert torch.equal(t, ref.drop_path_draw(dp.rates, 9, 0, 100 + k, 64)), k    # drawn before the add
    assert not torch.equal(tabs[0], tabs[1]) and not torch.equal(tabs[1], tabs[2])


# --------------------------------------------------------------------------- kernels with a row
def _row(B, g, p=0.4):
    keep = float(np.float32(1.0 / (1.0 - p)))
    s = torch.where(torch.rand(B, device=DEV, generator=g) < p, 0.0, keep).float()
    if B > 1:
        s[0], s[-1] = 0.0, keep                                  # at least one dropped and one kept sample
    return s.contiguous()


@pytest.mark.parametrize("B,HW,C", [(1, 49, 256), (8, 49, 2048), (37, 49, 256), (64, 49, 2048), (8, 3136, 256), (37, 3136, 256),
                                    (64, 3136, 256), (8, 196, 1024)])
@pytest.mark.parametrize("mode", ["bf16", "tf32"])
def test_batch_norm_with_drop_matches_fp64(mode, B, HW, C):
    """y = relu(s·bn(x) + res) and its gradients against fp64 autograd of the formula on the same (rounded) inputs, the ReLU mask
    taken from the kernel's own output; the tolerances of test_gpu_kernels.py's batch-norm test."""
    old = precision.precision()
    precision.set_precision(mode)
    try:
        dt = precision.act_dtype()
        g = torch.Generator(device=DEV).manual_seed(B * 131 + HW + C)
        shape = (B, HW, 1, C) if HW != 49 else (B, 7, 7, C)
        x = (torch.randn(shape, device=DEV, generator=g) * 2 + 0.5).to(dt).requires_grad_(True)
        res = torch.randn(shape, device=DEV, generator=g).to(dt).requires_grad_(True)
        gam = (torch.rand(C, device=DEV, generator=g) + 0.5).requires_grad_(True)
        bet = torch.randn(C, device=DEV, generator=g).requires_grad_(True)
        s = _row(B, g)
        rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
        y = ops.batch_norm(x, gam, bet, rm, rv, True, 0.1, 1e-5, True, res, drop=s)
        dy = torch.randn(shape, device=DEV, generator=g).to(dt)
        y.backward(dy)
        xd, rd, gd, bd = (t.detach().double().requires_grad_(True) for t in (x, res, gam, bet))
        m = xd.mean((0, 1, 2))
        v = ((xd - m) ** 2).mean((0, 1, 2))
        z = s.double().view(B, 1, 1, 1) * ((xd - m) / torch.sqrt(v + 1e-5) * gd + bd) + rd
        z.backward(dy.double() * (y.detach() > 0).double())
        tol = 2e-2 if mode == "bf16" else 1e-4
        assert rel_err(y, torch.relu(z.detach())) < tol
        assert rel_err(x.grad, xd.grad) < 3 * tol
        assert rel_err(gam.grad, gd.grad) < 3 * tol and rel_err(bet.grad, bd.grad) < 3 * tol
        assert rel_err(res.grad, rd.grad) < tol
        assert rel_err(rm, 0.1 * xd.detach().reshape(-1, C).mean(0)) < 1e-3     # whole-batch statistics
    finally:
        precision.set_precision(old)


def _bn_once(x, res, gam, bet, dy, s):
    xx, rr = x.clone().requires_grad_(True), res.clone().requires_grad_(True)
    gg, bb = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
    y = ops.batch_norm(xx, gg, bb, None, None, True, 0.1, 1e-5, True, rr, drop=s)
    y.backward(dy)
    return [t.clone() for t in (y, xx.grad, rr.grad, gg.grad, bb.grad)]


def bn_twice():
    """Two identical batch-norm forward / backward passes with a drop row at a ResNet50 shape: are all five outputs bit-equal?"""
    g = torch.Generator(device=DEV).manual_seed(5)
    B, C = 64, 256
    x = torch.randn(B, 28, 28, C, device=DEV, generator=g).bfloat16()
    res = torch.randn(B, 28, 28, C, device=DEV, generator=g).bfloat16()
    dy = torch.randn(B, 28, 28, C, device=DEV, generator=g).bfloat16()
    gam, bet = torch.rand(C, device=DEV, generator=g) + 0.5, torch.randn(C, device=DEV, generator=g)
    s = _row(B, g)
    a, b = _bn_once(x, res, gam, bet, dy, s), _bn_once(x, res, gam, bet, dy, s)
    return all(torch.equal(p, q) for p, q in zip(a, b))


def test_deterministic_mode_is_bit_reproducible():
    _subprocess("""
import test_gpu_drop_path as t
assert t.bn_twice()
print('OK')
""")


@pytest.mark.parametrize("shape", [(128, 32, 32, 64), (128, 16, 16, 128), (128, 8, 8, 256), (37, 8, 8, 16), (1, 4, 4, 8)])
@pytest.mark.parametrize("mode", ["bf16", "tf32"])
def test_scaled_add_and_branch_gradient(mode, shape):
    """WRN's merge y = s·a + b and its gradients (s·dy, dy) against fp64, the tolerance of test_gpu_kernels.py's add."""
    old = precision.precision()
    precision.set_precision(mode)
    try:
        dt = precision.act_dtype()
        g = torch.Generator(device=DEV).manual_seed(shape[0] * shape[3])
        a = torch.randn(shape, device=DEV, generator=g).to(dt).requires_grad_(True)
        b = torch.randn(shape, device=DEV, generator=g).to(dt).requires_grad_(True)
        s = _row(shape[0], g)
        y = ops.add(a, b, drop=s)
        dy = torch.randn(shape, device=DEV, generator=g).to(dt)
        y.backward(dy)
        sv = s.double().view(-1, 1, 1, 1)
        tol = 2e-2 if mode == "bf16" else 1e-4
        assert rel_err(y, sv * a.detach().double() + b.detach().double()) < tol
        assert rel_err(a.grad, sv * dy.double()) < tol and torch.equal(b.grad, dy)
        assert torch.all(a.grad[s == 0] == 0)
    finally:
        precision.set_precision(old)


# --------------------------------------------------------------------------- models
IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))
RESNET = ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50", dict(batch_size=8, file_batch_size=8, blocks=(1, 1, 1, 1),
                                                                                no_paraload=True, **IMNET))
WRN = ("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
       dict(batch_size=16, file_batch_size=32, depth=10, widen=2, data_kwargs=dict(n_synthetic=256, synthetic=True)))


def _model(mod, cls, dev, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device=dev, **cfg))
    m.rand_crop = False
    layers2.Dropout.SetDropoutOff(); layers2.Crop.SetRandCropOff()
    m.compile_iter_fns("avg")
    return m


def _train(m, steps, dev, tables=None, recs=None):
    """``steps`` training steps: the recorded costs, the drop table and the mix record of every step (``tables`` / ``recs``: replay
    these instead of drawing)."""
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device=dev)
    seen_t, seen_r = [], []
    if tables is not None:
        it = iter(tables)
        m.drop_path.draw = lambda: m.drop_path.table.copy_(next(it))
    if recs is not None:
        ir = iter(recs)
        m.mixer.draw = lambda: m.mixer.rec.copy_(next(ir))
    for i in range(steps):
        m.train_iter(i, rec)
        seen_t.append(m.drop_path.table.cpu().clone())
        if m.mixer is not None:
            seen_r.append(m.mixer.rec.cpu().clone())
    if dev != "cpu":
        torch.cuda.synchronize()
    return [float(c) for c in rec.train_info["cost"]], seen_t, seen_r


MODELS = {
    "resnet50_sgd": (RESNET, dict(drop_path_rate=0.5, learning_rate=0.05), 4),
    "resnet50_lars_accum4": (RESNET, dict(drop_path_rate=0.5, optimizer="lars", learning_rate=0.5, grad_accum=4), 8),
    "wrn_adam": (WRN, dict(drop_path_rate=0.6), 3),
    "resnet50_mixup_smoothing": (RESNET, dict(drop_path_rate=0.5, learning_rate=0.05, label_smoothing=0.1,
                                              mixup=dict(alpha=1.0, seed=3)), 4),
}


@pytest.mark.parametrize("which", list(MODELS))
def test_models_match_cpu_reference(which):
    """The native model with drop-path against the same model on the CPU reference ops, same weights and batches, the CPU replaying
    the tables (and mix records) the device drew: every step's loss within the tolerance of test_gpu_mixup.py's model comparison."""
    from theanompi_b200.models import layers2
    (mod, cls, cfg), extra, steps = MODELS[which]
    losses, tables, recs = {}, None, None
    try:
        for dev in ("cuda:0", "cpu"):
            m = _model(mod, cls, dev, cuda_graph=False, **dict(cfg, **extra))
            losses[dev], seen_t, seen_r = _train(m, steps, dev, tables, recs)
            if tables is None:
                tables, recs = seen_t, (seen_r or None)
            m.cleanup()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(which, losses)
    assert any(bool((t == 0).any()) for t in tables)                 # something was dropped
    assert len({tuple(t.reshape(-1).tolist()) for t in tables}) == steps
    for a, b in zip(losses["cpu"], losses["cuda:0"]):
        assert math.isfinite(b) and abs(a - b) < 0.08 * max(1.0, abs(a)), losses


def runs(spec, runs_, steps=5):
    """[(name, cuda_graph, extra config, force_ones)] of the model ``spec`` ('resnet' / 'wrn'): name → (W, U, last loss, graph used)."""
    from theanompi_b200.ops import cuda_impl
    mod, cls, cfg = RESNET if spec == "resnet" else WRN
    out = {}
    for name, graph, extra, ones in runs_:
        cuda_impl._STEP.clear()
        ops.seed_dropout(0x5EED)
        m = _model(mod, cls, DEV, cuda_graph=graph, **dict(cfg, **extra))
        if ones:
            m.drop_path.thresh.zero_(); m.drop_path.keep.fill_(1.0)   # the kernel runs and writes a table of ones
        from theanompi_b200.utils.recorder import Recorder
        rec = Recorder(None, 10 ** 6, "t", False, device=DEV)
        for i in range(steps):
            m.train_iter(i, rec)
        torch.cuda.synchronize()
        used = bool(m.captured_steps())
        out[name] = (m.arena.W.clone(), m.arena.U.clone(), float(rec.train_info["cost"][-1]), used)
        m.cleanup()
        del m
    return out


def _subprocess(code, timeout=900):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("spec", ["resnet", "wrn"])
def test_no_key_zero_and_forced_ones_are_bit_identical(spec):
    _subprocess("""
import test_gpu_drop_path as t
for graph in (True, False):
    o = t.runs(%r, [("absent", graph, {}, False), ("zero", graph, dict(drop_path_rate=0.0), False),
                    ("ones", graph, dict(drop_path_rate=0.4), True)])
    wa, ua, la, ga = o["absent"]
    for k in ("zero", "ones"):
        w, u, l, g = o[k]
        print(graph, k, la, l, g)
        assert g == ga == graph and l == la and t.torch.equal(w, wa) and t.torch.equal(u, ua), k
print('OK')
""" % spec)


@pytest.mark.parametrize("spec", ["resnet", "wrn"])
def test_graph_replay_equals_eager_steps(spec):
    _subprocess("""
import test_gpu_drop_path as t
o = t.runs(%r, [("eager", False, dict(drop_path_rate=0.5), False), ("graph", True, dict(drop_path_rate=0.5), False),
                ("plain", True, {}, False)])
(we, ue, le, ge), (wg, ug, lg, gg), (wp, up, lp, gp) = o["eager"], o["graph"], o["plain"]
print('losses eager', le, 'graph', lg, 'plain', lp)
assert gg and not ge and le == lg and t.torch.equal(we, wg) and t.torch.equal(ue, ug)
assert not t.torch.equal(wg, wp)                      # the captured step really drops
print('OK')
""" % spec)


def test_launch_counts():
    """ResNet50: one launch more per step (the draw; the rows ride on the batch-norm launches).  Wide_ResNet depth 10 (L = 3 blocks):
    the draw plus one branch-gradient launch for each of the L − 1 blocks with p_l > 0, so L more."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    try:
        for spec, (mod, cls, cfg) in (("resnet", RESNET), ("wrn", WRN)):
            for name, extra in (("absent", {}), ("zero", dict(drop_path_rate=0.0)), ("drop", dict(drop_path_rate=0.5))):
                m = _model(mod, cls, DEV, cuda_graph=False, **dict(cfg, **extra))
                for _ in range(2):
                    torch.cuda.synchronize()
                    native.reset_launch_count()
                    m.forward_backward(0)
                    torch.cuda.synchronize()
                    counts[spec, name] = native.launch_count()
                m.cleanup()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(counts)
    for spec, extra_launches in (("resnet", 1), ("wrn", 3)):
        assert counts[spec, "zero"] == counts[spec, "absent"]
        assert counts[spec, "drop"] == counts[spec, "absent"] + extra_launches, counts


def val_inf_same(spec):
    """Train with drop_path_rate = 0.7, then validate and infer twice from the same weights and running statistics: with the model's
    drop-path, and after switching it off.  Are the costs and class probabilities bit-equal?"""
    mod, cls, cfg = RESNET if spec == "resnet" else WRN
    m = _model(mod, cls, DEV, **dict(cfg, drop_path_rate=0.7))
    _train(m, 3, DEV)
    m.compile_inference()
    x = m.shared_x[:m.batch_size].clone()
    stats = [(b.running_mean.clone(), b.running_var.clone()) for b in m._bn_layers()]

    def outputs():
        for b, (rm, rv) in zip(m._bn_layers(), stats):       # validation runs batch norm in training mode: it moves them
            b.running_mean.copy_(rm); b.running_var.copy_(rv)
        c = [float(v) for v in m.val_fn(0)]
        p = m.inf_fn(x).clone()
        torch.cuda.synchronize()
        return c, p
    c1, p1 = outputs()
    m.drop_path_rate = 0.0
    m.check_drop_path()
    c0, p0 = outputs()
    print(spec, c1, c0)
    m.cleanup()
    return c1 == c0 and torch.equal(p1, p0)


@pytest.mark.parametrize("spec", ["resnet", "wrn"])
def test_validation_and_inference_never_drop(spec):
    _subprocess("""
import test_gpu_drop_path as t
assert t.val_inf_same(%r)
print('OK')
""" % spec)
