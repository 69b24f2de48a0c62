"""LARS on one H100: the norm kernels against fp64 torch norms, the update against ``reference.lars_flat``, run-to-run and CUDA-graph
bit identity, and the native models training with ``optimizer='lars'``."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from test_lars_cpu import ZERO_G, ZERO_W, fill_grad, lars_arena  # noqa: E402

pytestmark = pytest.mark.gpu

STEPS = 5


def test_norm_kernels_match_fp64_norms():
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.parallel.arena import G_W
    a, g = lars_arena("cuda:0", big=True)            # fc6: 36,864 blocks, more than the grid
    fill_grad(a, g)
    n = len(a.sizes)
    partial = torch.zeros(a.n_blocks, 2, device="cuda:0")
    norms, trust = torch.zeros(n, 2, device="cuda:0"), torch.zeros(n, device="cuda:0")
    cuda_impl.lars_trust(a, a.G, 0.5, 0.02, partial, norms, trust)
    torch.cuda.synchronize()
    for i, (w, gg) in enumerate(zip(a.views("W"), a.views("G"))):
        wn, gn = float(w.double().norm()), float(gg.double().norm()) * 0.5
        assert float(norms[i, 0]) == pytest.approx(wn, rel=1e-5, abs=1e-30), i
        assert float(norms[i, 1]) == pytest.approx(gn, rel=1e-5, abs=1e-30), i
        want = 0.02 * wn / (gn + 5e-4 * wn) if (a.group_of[i] == G_W and wn > 0 and gn > 0) else 1.0
        assert float(trust[i]) == pytest.approx(want, rel=1e-5), i
    assert float(trust[ZERO_W]) == 1.0 and float(trust[ZERO_G]) == 1.0


def _steps(prec, nesterov=False, k=1):
    """STEPS LARS steps on the CUDA arena and on its CPU twin (same seed, same gradients)."""
    from theanompi_b200.utils.opt import FlatLARS
    a, g = lars_arena("cuda:0", shadow=prec == "bf16")
    c, _ = lars_arena("cpu")
    oa, oc = FlatLARS(a, 0.9, nesterov, 0.02), FlatLARS(c, 0.9, nesterov, 0.02)
    a.hyper[0] = c.hyper[0] = 0.5
    for _ in range(STEPS):
        fill_grad(c, g)
        a.G.copy_(c.G)
        oa.step(k=k)
        oc.step(k=k)
    torch.cuda.synchronize()
    return a, oa, c, oc


@pytest.mark.parametrize("prec,nesterov,k", [("bf16", False, 1), ("bf16", True, 2), ("tf32", False, 2), ("tf32", True, 1)])
def test_steps_match_reference(prec, nesterov, k):
    a, oa, c, oc = _steps(prec, nesterov, k)
    np.testing.assert_allclose(oa.trust.cpu().numpy(), oc.trust.numpy(), rtol=1e-5)
    np.testing.assert_allclose(oa.norms.cpu().numpy(), oc.norms.numpy(), rtol=1e-5)
    for x, y in ((a.W, c.W), (a.U, c.U)):
        np.testing.assert_allclose(x.cpu().numpy(), y.numpy(), rtol=1e-5, atol=1e-6 * float(y.abs().max()))
    if prec == "bf16":
        assert torch.equal(a.H, a.W.to(torch.bfloat16))
    else:
        assert a.H is None


def test_steps_are_bit_reproducible():
    r1, r2 = _steps("bf16")[:2], _steps("bf16")[:2]
    for x, y in ((r1[0].W, r2[0].W), (r1[0].U, r2[0].U), (r1[0].H, r2[0].H), (r1[1].trust, r2[1].trust), (r1[1].norms, r2[1].norms)):
        assert torch.equal(x, y)


def test_graph_replay_equals_eager_step():
    from theanompi_b200.utils.opt import FlatLARS
    (a, g), (b, _) = lars_arena("cuda:0", shadow=True), lars_arena("cuda:0", shadow=True)
    oa, ob = FlatLARS(a, 0.9, True, 0.02), FlatLARS(b, 0.9, True, 0.02)
    fill_grad(a, g)
    b.G.copy_(a.G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ob.step(k=2)
    torch.cuda.current_stream().wait_stream(s)
    for lr in (0.5, 0.125):                           # the graph reads lr from the device
        a.hyper[0] = b.hyper[0] = lr
        oa.step(k=2)
        graph.replay()
        torch.cuda.synchronize()
        for x, y in ((a.W, b.W), (a.U, b.U), (a.H, b.H), (oa.trust, ob.trust), (oa.norms, ob.norms)):
            assert torch.equal(x, y)


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


def _check_trust(m):
    from theanompi_b200.parallel.arena import G_W
    from theanompi_b200.utils.opt import FlatLARS
    assert isinstance(m.lars, FlatLARS)
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params)
    t = m.lars.trust.cpu()
    wt = torch.tensor([g == G_W for g in m.arena.group_of])
    assert bool(torch.isfinite(t).all()) and bool((t[wt] > 0).all()), t


def test_default_sgd_arms_the_fc_epilogue_and_lars_does_not():
    from theanompi_b200.models import layers2
    from theanompi_b200.models.alex_net import AlexNet
    for opt, armed in (("sgd", True), ("lars", False)):
        layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear()
        m = AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=32, file_batch_size=32, optimizer=opt, **IMNET))
        m.compile_iter_fns("avg")
        assert any(getattr(p, "sgd_epilogue", None) is not None for p in m.arena.params) == armed, opt
        m.cleanup()


def test_alexnet_lars_graph_and_eager_agree():
    from theanompi_b200.ops import cuda_impl
    runs = []
    for graph in (False, True):
        cuda_impl._STEP.clear()
        costs, m = _run("theanompi_b200.models.alex_net", "AlexNet",
                        dict(batch_size=32, file_batch_size=32, cuda_graph=graph, optimizer="lars", learning_rate=2.0, **IMNET), steps=5)
        assert ("step" in m.captured_steps()) == graph
        _check_trust(m)
        runs.append(costs)
    assert abs(runs[0][-1] - runs[1][-1]) < 0.15, runs


def test_cifar10_model_learns_with_lars():
    # cuda_graph "auto": the model's random crops are drawn on the host every step, so it runs eager (AlexNet covers the graph)
    costs, m = _run("theanompi_b200.models.cifar10", "Cifar10_model",
                    dict(batch_size=64, file_batch_size=64, learning_rate=1.0, optimizer="lars",
                         data_kwargs=dict(n_synthetic=1024, synthetic=True)), steps=40)
    _check_trust(m)
    assert costs[-1] < 1.5 and costs[-1] < costs[0], costs
