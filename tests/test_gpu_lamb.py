"""LAMB on one H100: the moment / norm kernels against fp64 torch, the update against ``reference.lamb_flat``, run-to-run and
CUDA-graph bit identity, and the native models training with ``optimizer='lamb'``."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from test_lamb_cpu import WD, lamb_arena  # noqa: E402
from test_lars_cpu import ZERO_G, ZERO_W, fill_grad  # noqa: E402

pytestmark = pytest.mark.gpu

STEPS = 5
LR = 0.01


def test_trust_kernels_match_fp64_norms():
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.parallel.arena import G_W
    a, g = lamb_arena("cuda:0", big=True)            # fc6: 36,864 blocks, more than the grid
    fill_grad(a, g)
    n, dev = len(a.sizes), "cuda:0"
    gen = torch.Generator(device=dev).manual_seed(3)
    m0 = torch.randn(a.U.shape, device=dev, generator=gen) * 1e-2
    v0 = torch.rand(a.U.shape, device=dev, generator=gen) * 1e-4
    for i, (o, s) in enumerate(zip(a.offsets, a.sizes)):    # the padding holds zeros, as in a trained arena
        m0[o + s:o + -(-s // 1024) * 1024] = 0
        v0[o + s:o + -(-s // 1024) * 1024] = 0
    a.U.copy_(m0)
    v = v0.clone()
    step = torch.full((1,), 2, dtype=torch.int64, device=dev)     # bias corrections of step 3
    w0, gr0 = a.W.clone(), a.G.clone()
    partial = torch.zeros(a.n_blocks, 2, device=dev)
    norms, trust = torch.zeros(n, 2, device=dev), torch.zeros(n, device=dev)
    b1, b2, eps, inv_k = 0.9, 0.999, 1e-6, 0.5
    cuda_impl.lamb_trust(a, a.G, a.U, v, step, b1, b2, eps, inv_k, 0, partial, norms, trust)
    torch.cuda.synchronize()
    assert torch.equal(a.W, w0) and torch.equal(a.G, gr0) and int(step) == 2
    fb1, fb2 = float(np.float32(b1)), float(np.float32(b2))
    ge = gr0.double() * inv_k
    want_m = fb1 * m0.double() + (1 - fb1) * ge
    want_v = fb2 * v0.double() + (1 - fb2) * ge * ge
    for got, want in ((a.U, want_m), (v, want_v)):
        np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=1e-5, atol=1e-6 * float(want.abs().max()))
    c1, c2 = 1 / (1 - fb1 ** 3), 1 / (1 - fb2 ** 3)
    # r from the kernel's own updated moments, in fp64
    r_all = (a.U.double() * c1) / ((v.double() * c2).sqrt() + eps)
    for i, (o, s, grp) in enumerate(zip(a.offsets, a.sizes, a.group_of)):
        w = w0[o:o + s].double()
        r = r_all[o:o + s] + (WD if grp == G_W else 0.0) * w
        wn, rn = float(w.norm()), float(r.norm())
        assert float(norms[i, 0]) == pytest.approx(wn, rel=1e-5, abs=1e-30), i
        assert float(norms[i, 1]) == pytest.approx(rn, rel=1e-5, abs=1e-30), i
        want = wn / rn if (grp == G_W and wn > 0 and rn > 0) else 1.0
        assert float(trust[i]) == pytest.approx(want, rel=1e-5), i
    assert float(trust[ZERO_W]) == 1.0


def _steps(prec, k=1):
    """STEPS LAMB steps on the CUDA arena and on its CPU twin (same seed, same gradients)."""
    from theanompi_b200.utils.opt import FlatLAMB
    a, g = lamb_arena("cuda:0", shadow=prec == "bf16")
    c, _ = lamb_arena("cpu")
    oa, oc = FlatLAMB(a), FlatLAMB(c)
    a.hyper[0] = c.hyper[0] = LR
    for _ in range(STEPS):
        fill_grad(c, g)
        a.G.copy_(c.G)
        oa.step(k=k)
        oc.step(k=k)
    torch.cuda.synchronize()
    return a, oa, c, oc


@pytest.mark.parametrize("prec,k", [("bf16", 1), ("bf16", 2), ("tf32", 1), ("tf32", 2)])
def test_steps_match_reference(prec, k):
    a, oa, c, oc = _steps(prec, k)
    assert int(oa.t) == int(oc.t) == STEPS
    np.testing.assert_allclose(oa.trust.cpu().numpy(), oc.trust.numpy(), rtol=1e-5)
    np.testing.assert_allclose(oa.norms.cpu().numpy(), oc.norms.numpy(), rtol=1e-5)
    assert float(oa.trust[ZERO_G]) == pytest.approx(1.0 / WD, rel=1e-5)
    for x, y in ((a.W, c.W), (a.U, c.U), (oa.V, oc.V)):
        np.testing.assert_allclose(x.cpu().numpy(), y.numpy(), rtol=1e-5, atol=1e-6 * float(y.abs().max()))
    assert torch.equal(a.G.cpu(), c.G)                 # the gradient is left as it was
    if prec == "bf16":
        assert torch.equal(a.H, a.W.to(torch.bfloat16))
    else:
        assert a.H is None


def test_split_step_equals_one_step():
    """The batch-norm-only pass and the exchanged-groups pass advance the device counter once and equal one whole step."""
    from theanompi_b200.utils.opt import FlatLAMB
    (a, g), (b, _) = lamb_arena("cuda:0", shadow=True), lamb_arena("cuda:0", shadow=True)
    oa, ob = FlatLAMB(a), FlatLAMB(b)
    a.hyper[0] = b.hyper[0] = LR
    for _ in range(3):
        fill_grad(a, g)
        b.G.copy_(a.G)
        oa.step(only_local=True)
        oa.step(only_exchanged=True)
        ob.step()
    torch.cuda.synchronize()
    assert int(oa.t) == int(ob.t) == 3
    for x, y in ((a.W, b.W), (a.U, b.U), (oa.V, ob.V), (a.H, b.H), (oa.trust, ob.trust), (oa.norms, ob.norms)):
        assert torch.equal(x, y)


def test_steps_are_bit_reproducible():
    r1, r2 = _steps("bf16")[:2], _steps("bf16")[:2]
    for x, y in ((r1[0].W, r2[0].W), (r1[0].U, r2[0].U), (r1[1].V, r2[1].V), (r1[0].H, r2[0].H), (r1[1].trust, r2[1].trust),
                 (r1[1].norms, r2[1].norms), (r1[1].t, r2[1].t)):
        assert torch.equal(x, y)


def test_graph_replay_equals_eager_step():
    from theanompi_b200.utils.opt import FlatLAMB
    (a, g), (b, _) = lamb_arena("cuda:0", shadow=True), lamb_arena("cuda:0", shadow=True)
    oa, ob = FlatLAMB(a), FlatLAMB(b)
    fill_grad(a, g)
    b.G.copy_(a.G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ob.step(k=2)
    torch.cuda.current_stream().wait_stream(s)
    for lr in (LR, LR / 4):                           # the graph reads lr and the step counter from the device
        a.hyper[0] = b.hyper[0] = lr
        oa.step(k=2)
        graph.replay()
        torch.cuda.synchronize()
        for x, y in ((a.W, b.W), (a.U, b.U), (oa.V, ob.V), (a.H, b.H), (oa.trust, ob.trust), (oa.norms, ob.norms), (oa.t, ob.t)):
            assert torch.equal(x, y)
    assert int(ob.t) == 2


IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))


def _run(modelfile, modelclass, cfg, steps):
    import importlib
    from theanompi_b200.models import layers2
    from theanompi_b200.utils.recorder import Recorder
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear()
    base = dict(verbose=False, rank=0, size=1, device="cuda:0")
    base.update(cfg)
    m = getattr(importlib.import_module(modelfile), modelclass)(base)
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, modelclass, False, device="cuda:0")
    w0 = m.arena.W.clone()
    for i in range(steps):
        m.train_iter(i, rec)
    torch.cuda.synchronize()
    costs = [float(c) for c in rec.train_info["cost"]]
    assert all(math.isfinite(c) for c in costs), costs
    assert not torch.equal(w0, m.arena.W), "weights did not move"
    m.cleanup()
    return costs, m


def _check_trust(m, steps):
    from theanompi_b200.parallel.arena import G_W
    from theanompi_b200.utils.opt import FlatLAMB
    assert isinstance(m.lamb, FlatLAMB) and int(m.lamb.t) == steps
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params)
    t = m.lamb.trust.cpu()
    wt = torch.tensor([g == G_W for g in m.arena.group_of])
    assert bool(torch.isfinite(t).all()) and bool((t[wt] > 0).all()), t


def test_lamb_does_not_arm_the_fc_epilogue():
    from theanompi_b200.models import layers2
    from theanompi_b200.models.alex_net import AlexNet
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear()
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=32, file_batch_size=32, optimizer="lamb", **IMNET))
    m.compile_iter_fns("avg")
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params)
    m.cleanup()


def test_alexnet_lamb_graph_and_eager_agree():
    from theanompi_b200.ops import cuda_impl
    runs = []
    for graph in (False, True):
        cuda_impl._STEP.clear()
        costs, m = _run("theanompi_b200.models.alex_net", "AlexNet",
                        dict(batch_size=32, file_batch_size=32, cuda_graph=graph, optimizer="lamb", learning_rate=LR, **IMNET), steps=5)
        assert ("step" in m.captured_steps()) == graph
        _check_trust(m, 5)
        runs.append(costs)
    assert abs(runs[0][-1] - runs[1][-1]) < 0.15, runs


def test_cifar10_model_learns_with_lamb():
    # cuda_graph "auto": the model's random crops are drawn on the host every step, so it runs eager (AlexNet covers the graph)
    costs, m = _run("theanompi_b200.models.cifar10", "Cifar10_model",
                    dict(batch_size=64, file_batch_size=64, learning_rate=LR, optimizer="lamb",
                         data_kwargs=dict(n_synthetic=1024, synthetic=True)), steps=40)
    _check_trust(m, 40)
    assert costs[-1] < 1.5 and costs[-1] < costs[0], costs


def test_wide_resnet_trains_with_lamb():
    costs, m = _run("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
                    dict(batch_size=16, file_batch_size=16, depth=10, widen=2, optimizer="lamb", learning_rate=LR,
                         data_kwargs=dict(n_synthetic=128, synthetic=True)), steps=3)
    _check_trust(m, 3)
    assert getattr(m, "adam", None) is None
