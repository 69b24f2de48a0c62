"""LAMB on the CPU: the reference update against a naive per-tensor implementation of its formulas, the group filters and the step
counter, a model that learns with it, BSP over two gloo ranks against one process on the summed gradient, the refusal of the fused
exchange, Wide_ResNet on the split exchange and checkpoint / resume."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from test_lars_cpu import SHAPES, ZERO_G, ZERO_W, fill_grad  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.parallel.arena import G_W, FlatArena  # noqa: E402
from theanompi_b200.utils.opt import FlatLAMB  # noqa: E402

WD = 5e-4


def lamb_arena(device="cpu", shadow=False, big=False, wd=WD):
    """The LARS test arena (weight decay, a bias lr multiplier, a gamma group, sizes that are not multiples of 1024, one all-zero
    weight and one all-zero gradient) with weight decay ``wd``; ``big`` adds AlexNet's fc6 (36,864 blocks: more than the grid)."""
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
    return FlatArena(params, wt, device, weight_decay=wd, shadow=shadow), g


def naive_lamb(ws, gs, ms, vs, groups, lr, t, wd, bias_mult, inv_k, b1=0.9, b2=0.999, eps=1e-6):
    """The formulas written out per tensor in fp64, with b1 and b2 rounded to fp32 as the optimizer takes them (1 − b2 would
    otherwise differ by 1.3e-5 relative)."""
    b1, b2 = float(np.float32(b1)), float(np.float32(b2))
    trust, norms = [], []
    for i, (w, g, m, v) in enumerate(zip(ws, gs, ms, vs)):
        g = g * inv_k
        m.mul_(b1).add_((1 - b1) * g)
        v.mul_(b2).add_((1 - b2) * g * g)
        is_w = groups[i] == G_W
        r = (m / (1 - b1 ** t)) / ((v / (1 - b2 ** t)).sqrt() + eps) + (wd if is_w else 0.0) * w
        wn, rn = float(w.norm()), float(r.norm())
        tr = wn / rn if (is_w and wn > 0 and rn > 0) else 1.0
        trust.append(tr)
        norms.append((wn, rn))
        w.sub_(lr * (1.0 if groups[i] in (0, 2) else bias_mult) * tr * r)
    return trust, norms


@pytest.mark.parametrize("wd", [WD, 0.0])
@pytest.mark.parametrize("k", [1, 2])
def test_reference_lamb_matches_naive_formulas(k, wd):
    a, g = lamb_arena(wd=wd)
    opt = FlatLAMB(a)
    a.hyper[0] = 0.01
    ws = [v.double().clone() for v in a.views("W")]
    ms = [torch.zeros_like(w) for w in ws]
    vs = [torch.zeros_like(w) for w in ws]
    for s in range(5):
        fill_grad(a, g)
        gs = [v.double().clone() for v in a.views("G")]
        want_t, want_n = naive_lamb(ws, gs, ms, vs, a.group_of, 0.01, s + 1, wd, 2.0, 1.0 / k)
        opt.step(k=k)
        assert int(opt.t) == s + 1
        np.testing.assert_allclose(opt.trust.numpy(), np.array(want_t), rtol=1e-5)
        np.testing.assert_allclose(opt.norms.numpy(), np.array(want_n), rtol=1e-5)
        if s == 0:                             # the step moves the zero weights away from zero
            assert float(opt.trust[ZERO_W]) == 1.0
        # a zero gradient leaves r = wd·W: ratio 1 / wd, so the step is the decoupled decay lr·W; without decay r = 0, ratio 1
        assert float(opt.trust[ZERO_G]) == (pytest.approx(1.0 / wd, rel=1e-5) if wd else 1.0)
        assert float(opt.trust[0]) != 1.0 and float(opt.trust[1]) == 1.0 and float(opt.trust[2]) == 1.0
    for got, want in ((a.views("W"), ws), (a.views("U"), ms), (opt_views(a, opt.V), vs)):
        for x, y in zip(got, want):
            np.testing.assert_allclose(x.double().numpy(), y.numpy(), rtol=1e-5, atol=1e-6 * float(y.abs().max()) + 1e-12)


def opt_views(a, buf):
    """``buf`` (a flat buffer laid out as the arena) cut into the parameters' shapes."""
    return [buf[o:o + s].view(p.shape) for o, s, p in zip(a.offsets, a.sizes, a.params)]


def test_filters_update_only_their_groups():
    a, g = lamb_arena()
    opt = FlatLAMB(a)
    a.hyper[0] = 0.01
    fill_grad(a, g)
    ex = a.exchanged_mask()
    for flag, t_after in (("only_local", 0), ("only_exchanged", 1)):
        before = [[v.clone() for v in vs] for vs in (a.views("W"), a.views("U"), opt_views(a, opt.V))]
        opt.step(**{flag: True})
        assert int(opt.t) == t_after
        for vs, vs0 in zip((a.views("W"), a.views("U"), opt_views(a, opt.V)), before):
            for i, (v, v0) in enumerate(zip(vs, vs0)):
                if i != ZERO_G or flag == "only_local":   # a zero gradient leaves M and V at zero
                    assert (not torch.equal(v, v0)) == (ex[i] != (flag == "only_local")), (flag, i)


def test_split_step_equals_one_step():
    """A batch-norm-only pass followed by the exchanged-groups pass advances the step counter once and equals one whole step."""
    (a, g), (b, _) = lamb_arena(), lamb_arena()
    oa, ob = FlatLAMB(a), FlatLAMB(b)
    a.hyper[0] = b.hyper[0] = 0.01
    for _ in range(3):
        fill_grad(a, g)
        b.G.copy_(a.G)
        oa.step(only_local=True)
        oa.step(only_exchanged=True)
        ob.step()
    assert int(oa.t) == int(ob.t) == 3
    for x, y in ((a.W, b.W), (a.U, b.U), (oa.V, ob.V), (oa.trust, ob.trust), (oa.norms, ob.norms)):
        assert torch.equal(x, y)


def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.01, optimizer="lamb",
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    return Cifar10_model(cfg)


def test_cifar10_model_learns_with_lamb():
    from theanompi_b200.utils.recorder import Recorder
    m = _cifar(batch_size=64, file_batch_size=64, data_kwargs=dict(n_synthetic=1024, synthetic=True))
    m.compile_iter_fns("avg")
    assert isinstance(m.lamb, FlatLAMB)
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params)
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(40):
        m.train_iter(i, rec)
    costs = [float(c) for c in rec.train_info["cost"]]
    assert costs[-1] < 1.5 and costs[-1] < costs[0], costs
    assert int(m.lamb.t) == 40
    wt = [g == G_W for g in m.arena.group_of]
    t = m.lamb.trust
    assert bool(torch.isfinite(t).all()) and bool((t[wt] > 0).all()) and bool((t[wt] != 1).all())


def test_bsp_lamb_two_ranks_equals_one_process_on_the_summed_gradient(tmp_path):
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT="29813", OMP_NUM_THREADS="2", PYTHONPATH=ROOT,
               TMPI_TEST_OUT=str(tmp_path))
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_lamb_checks.py"), "bsp_lamb"],
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
    got = torch.load(tmp_path / "bsp_lamb.pt")
    assert got["t"] == 6
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
            m.lamb.step(k=2)
    finally:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn()
    assert float((m.arena.W - w0).abs().max()) > 1e-3              # the comparison is not between two unmoved models
    err = float((got["W"] - m.arena.W).abs().max())
    assert err < 2e-5, err


def test_fused_exchange_is_refused_and_wide_resnet_takes_the_split_exchange():
    m = _cifar(size=2)
    with pytest.raises(ValueError, match="optimizer='lamb'.*split strategy"):
        m.compile_iter_fns("cdd", fused_tail=lambda: None)
    m = _cifar(size=2, optimizer="adam")
    with pytest.raises(ValueError, match="'lamb', 'sgd' or 'lars'"):
        m.compile_iter_fns("cdd")
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    w = Wide_ResNet(dict(verbose=False, rank=0, size=2, device="cpu", batch_size=8, file_batch_size=8, depth=10, widen=1,
                         optimizer="lamb", data_kwargs=dict(n_synthetic=64, synthetic=True)))
    w.compile_iter_fns("cdd")
    assert w.sync_type == "cdd" and isinstance(w.lamb, FlatLAMB) and getattr(w, "adam", None) is None
    assert len(w.vels) == len(w.vels2) == sum(w.arena.exchanged_mask())


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
        assert int(b.lamb.t) == 3
        steps(b, batches[3:])
    finally:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn()
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U) and torch.equal(a.lamb.V, b.lamb.V)
    assert int(a.lamb.t) == int(b.lamb.t) == 6
    assert torch.equal(a.lamb.trust, b.lamb.trust)
