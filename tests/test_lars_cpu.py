"""LARS on the CPU: the reference update against a naive per-tensor implementation of its formulas, a model that learns with it,
BSP over two gloo ranks against one process on the summed gradient, the refusal of the fused exchange and checkpoint / resume."""
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
from theanompi_b200.parallel.arena import G_W, FlatArena  # noqa: E402
from theanompi_b200.utils.opt import FlatLARS  # noqa: E402

SHAPES = [("W", (300, 70)), ("b", (300,)), ("gamma", (96,)), ("W", (64, 3, 3, 16)), ("b", (17,)), ("W", (50, 30)), ("W", (40, 41))]
ZERO_W, ZERO_G = 5, 6                  # an all-zero weight tensor and a tensor whose gradient is always zero


def lars_arena(device="cpu", shadow=False, big=False):
    """Weight decay, a bias lr multiplier, a batch-norm gamma group, sizes that are not multiples of 1024, one all-zero weight and one
    all-zero gradient; ``big`` adds AlexNet's fc6 (9216 x 4096, 36,864 blocks: more than the kernels' grid)."""
    g = torch.Generator().manual_seed(7)
    shapes = SHAPES + ([("W", (4096, 9216))] if big else [])
    params = []
    for name, shape in shapes:
        p = torch.nn.Parameter(torch.randn(*shape, generator=g) * 0.05)
        p.pname = name
        params.append(p)
    with torch.no_grad():
        params[ZERO_W].zero_()
    wt = ["W" if n == "W" else "b" for n, _ in shapes]
    return FlatArena(params, wt, device, weight_decay=5e-4, shadow=shadow), g


def fill_grad(a, g):
    """Random gradients on the real elements (the padding stays zero, as the backward kernels leave it), zero for ZERO_G."""
    a.G.zero_()
    for i, v in enumerate(a.views("G")):
        if i != ZERO_G:
            v.copy_(torch.randn(v.shape, generator=g) * 0.1)


def naive_lars(ws, gs, us, groups, lr, mu, nesterov, eta, wd, bias_mult, inv_k):
    """The formulas written out per tensor in fp64."""
    trust = []
    for i, (w, g, u) in enumerate(zip(ws, gs, us)):
        g = g * inv_k
        wn, gn = float(w.norm()), float(g.norm())
        is_w = groups[i] == G_W
        d = wd if is_w else 0.0
        t = eta * wn / (gn + d * wn) if (is_w and wn > 0 and gn > 0) else 1.0
        trust.append(t)
        ge = t * (g + d * w)
        u.mul_(mu).add_(ge)
        m = 1.0 if groups[i] in (0, 2) else bias_mult
        w.sub_(lr * m * (ge + mu * u if nesterov else u))
    return trust


@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("k", [1, 2])
def test_reference_lars_matches_naive_formulas(nesterov, k):
    a, g = lars_arena()
    opt = FlatLARS(a, mu=0.9, nesterov=nesterov, eta=0.02)
    a.hyper[0] = 0.5
    ws = [v.double().clone() for v in a.views("W")]
    us = [v.double().clone() for v in a.views("U")]
    for s in range(5):
        fill_grad(a, g)
        gs = [v.double().clone() for v in a.views("G")]
        want_t = naive_lars(ws, gs, us, a.group_of, 0.5, 0.9, nesterov, 0.02, 5e-4, 2.0, 1.0 / k)
        opt.step(k=k)
        np.testing.assert_allclose(opt.trust.numpy(), np.array(want_t), rtol=1e-6)
        if s == 0:                             # the gradient step moves the zero weights away from zero
            assert float(opt.trust[ZERO_W]) == 1.0
        assert float(opt.trust[ZERO_G]) == 1.0
        assert float(opt.trust[0]) != 1.0 and float(opt.trust[1]) == 1.0 and float(opt.trust[2]) == 1.0
    for got, want in ((a.views("W"), ws), (a.views("U"), us)):
        for x, y in zip(got, want):
            np.testing.assert_allclose(x.double().numpy(), y.numpy(), rtol=1e-6, atol=1e-6 * float(y.abs().max()) + 1e-12)


def test_filters_update_only_their_groups():
    a, g = lars_arena()
    opt = FlatLARS(a, eta=0.02)
    a.hyper[0] = 0.5
    fill_grad(a, g)
    ex = a.exchanged_mask()
    for flag in ("only_local", "only_exchanged"):
        w0 = [v.clone() for v in a.views("W")]
        opt.step(**{flag: True})
        for i, (v, v0) in enumerate(zip(a.views("W"), w0)):
            assert (not torch.equal(v, v0)) == (ex[i] != (flag == "only_local")), (flag, i)


def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=1.0, optimizer="lars",
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    return Cifar10_model(cfg)


def test_cifar10_model_learns_with_lars():
    from theanompi_b200.utils.recorder import Recorder
    m = _cifar(batch_size=64, file_batch_size=64, data_kwargs=dict(n_synthetic=1024, synthetic=True))
    m.compile_iter_fns("avg")
    assert isinstance(m.lars, FlatLARS)
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params)
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(40):
        m.train_iter(i, rec)
    costs = [float(c) for c in rec.train_info["cost"]]
    assert costs[-1] < 1.5 and costs[-1] < costs[0], costs
    wt = [g == G_W for g in m.arena.group_of]
    t = m.lars.trust
    assert bool(torch.isfinite(t).all()) and bool((t[wt] > 0).all()) and bool((t[wt] != 1).all())


def test_bsp_lars_two_ranks_equals_one_process_on_the_summed_gradient(tmp_path):
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT="29811", OMP_NUM_THREADS="2", PYTHONPATH=ROOT,
               TMPI_TEST_OUT=str(tmp_path))
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_lars_checks.py"), "bsp_lars"],
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
    got = torch.load(tmp_path / "bsp_lars.pt")
    m = _cifar()
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    try:
        m.compile_iter_fns("avg")
        w0 = m.arena.W.clone()
        d = m.data
        for step in range(6):
            if step == 0:
                d.shuffle_data("train", common_seed=m.epoch)
            gsum = None
            for r in range(2):
                m.x_in.copy_(torch.from_numpy(np.ascontiguousarray(d.train_img_shuffle[2 * step + r])))
                m.y_in.copy_(torch.from_numpy(np.asarray(d.train_labels_shuffle[2 * step + r])))
                m._fwd_bwd_eager()
                gsum = m.arena.G.clone() if gsum is None else gsum + m.arena.G
            m.arena.G.copy_(gsum)
            m.lars.step(k=2)
    finally:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn()
    assert float((m.arena.W - w0).abs().max()) > 1e-3              # the comparison is not between two unmoved models
    err = float((got["W"] - m.arena.W).abs().max())
    assert err < 2e-5, err


def test_fused_exchange_is_refused():
    m = _cifar(size=2)
    with pytest.raises(ValueError, match="split strategy"):
        m.compile_iter_fns("cdd", fused_tail=lambda: None)
    m = _cifar(size=2, optimizer="adam")
    with pytest.raises(ValueError, match="'sgd' or 'lars'"):
        m.compile_iter_fns("cdd")


def test_checkpoint_resume_continues_bit_identically(tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    try:
        a = _cifar()
        a.compile_iter_fns("avg")
        d = a.data
        d.shuffle_data("train", common_seed=0)
        batches = [(torch.from_numpy(np.ascontiguousarray(d.train_img_shuffle[i])), torch.from_numpy(np.asarray(d.train_labels_shuffle[i])))
                   for i in range(6)]

        def steps(m, bs):
            Dropout.SetDropoutOff(); Crop.SetRandCropOff()           # also the layers of a model built since
            for x, y in bs:
                m.shared_x.copy_(x)
                m.shared_y.copy_(y)
                m.train_iter_fn(0)

        steps(a, batches[:3])
        f = str(tmp_path / "ck.pt")
        save_checkpoint(a, f)
        steps(a, batches[3:])
        layers2.reseed(999)
        b = _cifar()
        b.compile_iter_fns("avg")
        load_checkpoint(b, f)
        steps(b, batches[3:])
    finally:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn()
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)
    assert torch.equal(a.lars.trust, b.lars.trust)
