"""Global gradient-norm clipping on one H100: the norm kernels against an fp64 torch norm, the five clipped rules against the CPU
reference, bit identity with the unclipped kernel below the threshold, skipped steps on a NaN gradient, CUDA-graph and run-to-run
bit identity, and AlexNet, the LSTM and NativeWGAN training with ``grad_clip``."""
import math
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from test_grad_clip_cpu import RULES, clip_arena, fill_grad, make_opt, opt_state  # noqa: E402

pytestmark = pytest.mark.gpu

STEPS = 5
LR = 0.01


def _real_norm(a, g):
    return math.sqrt(sum(float((g[o:o + s].double() ** 2).sum()) for o, s in zip(a.offsets, a.sizes)))


def test_norm_kernels_match_fp64_norm():
    from theanompi_b200.ops import cuda_impl
    a, g = clip_arena("cuda:0", big=True)                 # fc6: 36,864 blocks, more than the grid
    gen = torch.Generator(device="cuda:0").manual_seed(5)
    a.G.copy_(torch.randn(a.G.shape, device="cuda:0", generator=gen) * 1e3)       # garbage in the padding
    for v in a.views("G"):
        v.copy_(torch.randn(v.shape, device="cuda:0", generator=gen) * 0.01)
    g0 = a.G.clone()
    partial = torch.zeros(a.n_blocks, device="cuda:0")
    rec = torch.zeros(4, device="cuda:0")
    skipped = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    want = _real_norm(a, g0)
    for c in (0.5 * want, 2.0 * want):
        cuda_impl.grad_clip_norm(a, a.G, c, partial, rec, skipped)
        torch.cuda.synchronize()
        assert float(rec[0]) == pytest.approx(want, rel=1e-5)
        assert float(rec[1]) == pytest.approx(min(1.0, c / (want + 1e-6)), rel=1e-5)
        assert int(rec[2:3].view(torch.int32)) == 1 and int(skipped) == 0
    assert float(rec[1]) == 1.0
    assert torch.equal(a.G, g0)
    a.G[a.offsets[-1] + 12345] = float("inf")
    cuda_impl.grad_clip_norm(a, a.G, 1.0, partial, rec, skipped)
    a.G[a.offsets[2] + 3] = float("nan")
    cuda_impl.grad_clip_norm(a, a.G, 1.0, partial, rec, skipped)
    torch.cuda.synchronize()
    assert int(rec[2:3].view(torch.int32)) == 0 and int(skipped) == 2 and math.isnan(float(rec[0]))


def _steps(rule, prec, c, lr=LR):
    """STEPS clipped steps on the CUDA arena and on its CPU twin (same gradients)."""
    a, g = clip_arena("cuda:0", shadow=prec == "bf16")
    h, _ = clip_arena("cpu")
    oa, oh = make_opt(rule, a), make_opt(rule, h)
    for o in (oa, oh):
        if c is not None:
            o.set_grad_clip(c)
    a.hyper[0] = h.hyper[0] = lr
    for _ in range(STEPS):
        fill_grad(h, g)
        a.G.copy_(h.G)
        oa.step()
        oh.step()
    torch.cuda.synchronize()
    return a, oa, h, oh


@pytest.mark.parametrize("prec", ["bf16", "tf32"])
@pytest.mark.parametrize("rule", RULES)
def test_clipped_steps_match_reference(rule, prec):
    # Adam: the kernel's bias corrections use the fast __powf, whose error on 1 − b2^t is amplified in the first steps (with or
    # without clipping), so it is held to a norm-wise tolerance at the lr of test_gpu_kernels.py::test_adam_flat_matches_torch;
    # the clipping itself is checked bit for bit below.  The other rules are held to an elementwise tolerance.
    a, oa, h, oh = _steps(rule, prec, 2.0, lr=1e-3 if rule == "adam" else LR)
    assert float(oa.grad_norm) > 2.0                      # the clip is active
    assert float(oa.grad_norm) == pytest.approx(float(oh.grad_norm), rel=1e-5)
    assert float(oa._clip_rec[1]) == pytest.approx(float(oh._clip_rec[1]), rel=1e-5)
    for x, y in zip(opt_state(oa), opt_state(oh)):
        if x.dtype == torch.bfloat16:
            continue
        if rule == "adam":
            err = float((x.cpu().double() - y.double()).norm() / y.double().norm().clamp_min(1e-30))
            assert err < 5e-5, err
        else:
            np.testing.assert_allclose(x.cpu().numpy(), y.numpy(), rtol=1e-5, atol=1e-6 * float(y.abs().max()))
    assert torch.equal(a.G.cpu(), h.G)                   # the gradient is not scaled in place
    if prec == "bf16":
        assert torch.equal(a.H, a.W.to(torch.bfloat16))
    else:
        assert a.H is None


@pytest.mark.parametrize("rule", ["adam", "rmsprop", "adadelta", "rmsprop_centered"])
def test_clipped_step_is_the_unclipped_kernel_on_the_scaled_gradient(rule):
    """The rules that scale the loaded gradient (SGD folds s into inv_k instead): the clipped step equals, bit for bit, the
    unclipped kernel on s·G rounded to fp32."""
    (a, g), (b, _) = clip_arena("cuda:0", shadow=True), clip_arena("cuda:0", shadow=True)
    oa, ob = make_opt(rule, a), make_opt(rule, b)
    oa.set_grad_clip(2.0)
    a.hyper[0] = b.hyper[0] = LR
    for _ in range(STEPS):
        fill_grad(a, g)
        oa.step()
        b.G.copy_(a.G * oa._clip_rec[1])
        ob.step()
    torch.cuda.synchronize()
    assert float(oa._clip_rec[1]) < 1.0
    for x, y in zip(opt_state(oa), opt_state(ob)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("rule", RULES)
def test_above_the_norm_the_step_is_bit_identical_to_the_unclipped_kernel(rule):
    (a, oa, _, _), (b, ob, _, _) = _steps(rule, "bf16", 1e6), _steps(rule, "bf16", None)
    assert float(oa._clip_rec[1]) == 1.0
    for x, y in zip(opt_state(oa), opt_state(ob)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("rule", RULES)
def test_nan_gradient_leaves_every_buffer_bit_identical(rule):
    a, g = clip_arena("cuda:0", shadow=True)
    opt = make_opt(rule, a)
    opt.set_grad_clip(1.0)
    a.hyper[0] = LR
    fill_grad(a, g)
    opt.step()
    before = opt_state(opt)
    fill_grad(a, g)
    a.G[a.offsets[3] + 7] = float("nan")
    opt.step()
    torch.cuda.synchronize()
    for x, y in zip(opt_state(opt), before):
        assert torch.equal(x, y)
    assert int(opt.skipped) == 1 and int(opt._clip_rec[2:3].view(torch.int32)) == 0
    if opt.t is not None:
        assert int(opt.t) == 1                            # the counter did not advance


@pytest.mark.parametrize("rule", ["sgd", "adam"])
def test_graph_replay_equals_eager_step_and_runs_are_bit_identical(rule):
    (a, g), (b, _) = clip_arena("cuda:0", shadow=True), clip_arena("cuda:0", shadow=True)
    oa, ob = make_opt(rule, a), make_opt(rule, b)
    oa.set_grad_clip(2.0)
    ob.set_grad_clip(2.0)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            ob.step()
    torch.cuda.current_stream().wait_stream(s)
    for step, lr in enumerate((LR, LR / 4, LR)):          # the graph reads lr, the gradient and the counters from the device
        fill_grad(a, g)
        if step == 2:
            a.G[100] = float("nan")
        b.G.copy_(a.G)
        a.hyper[0] = b.hyper[0] = lr
        oa.step()
        graph.replay()
        torch.cuda.synchronize()
        for x, y in zip(opt_state(oa) + [oa._clip_rec, oa.skipped], opt_state(ob) + [ob._clip_rec, ob.skipped]):
            assert torch.equal(x.nan_to_num(), y.nan_to_num())
    assert int(ob.skipped) == 1
    r1, r2 = _steps(rule, "bf16", 2.0)[:2], _steps(rule, "bf16", 2.0)[:2]
    for x, y in zip(opt_state(r1[1]) + [r1[1]._clip_rec], opt_state(r2[1]) + [r2[1]._clip_rec]):
        assert torch.equal(x, y)


IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))


def _alexnet(**kw):
    from theanompi_b200.models import layers2
    from theanompi_b200.models.alex_net import AlexNet
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear()
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=32, file_batch_size=32, learning_rate=LR, **IMNET, **kw))
    m.compile_iter_fns("avg")
    return m


def test_fc_epilogue_is_not_armed_while_clipping():
    m = _alexnet(grad_clip=1.0)
    assert all(getattr(p, "sgd_epilogue", None) is None for p in m.arena.params)
    m.cleanup()
    m = _alexnet()                                          # the default path still arms it
    assert any(getattr(p, "sgd_epilogue", None) is not None for p in m.arena.params)
    m.cleanup()


def test_alexnet_with_grad_clip_graph_and_eager_agree():
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.recorder import Recorder
    runs = []
    for graph in (False, True):
        cuda_impl._STEP.clear()
        m = _alexnet(grad_clip=1.0, cuda_graph=graph)
        rec = Recorder(None, 10 ** 6, "AlexNet", False, device="cuda:0")
        w0 = m.arena.W.clone()
        for i in range(6):
            m.train_iter(i, rec)
        torch.cuda.synchronize()
        costs = [float(c) for c in rec.train_info["cost"]]
        assert ("step" in m.captured_steps()) == graph
        assert all(math.isfinite(c) for c in costs) and not torch.equal(w0, m.arena.W)
        assert float(m.clip_opt.grad_norm) > 0 and int(m.clip_opt.skipped) == 0
        runs.append(costs)
        m.cleanup()
    assert abs(runs[0][-1] - runs[1][-1]) < 0.15, runs


@pytest.mark.parametrize("optimizer", ["adadelta", "rmsprop", "sgd"])
def test_lstm_bucket_graphs_with_grad_clip(optimizer):
    from theanompi_b200.models import layers2
    from theanompi_b200.models.lstm import LSTM
    from theanompi_b200.utils.recorder import Recorder
    layers2.reseed(); layers2.Dropout.layers.clear()
    m = LSTM(dict(verbose=False, rank=0, size=1, device="cuda:0", dim_proj=64, optimizer=optimizer, grad_clip=0.5,
                  data_kwargs=dict(n_synthetic=512, n_words=500)))
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "LSTM", False, device="cuda:0")
    n = 600 if optimizer == "adadelta" else 8
    for i in range(n):
        m.train_iter(i, rec)
    torch.cuda.synchronize()
    c = [float(v) for v in rec.train_info["cost"]]
    assert all(math.isfinite(v) for v in c)
    assert m.captured_steps()           # the clipped step runs inside the bucket graphs
    assert m.opt.max_norm == 0.5 and int(m.opt.skipped) == 0 and math.isfinite(float(m.opt.grad_norm))
    if optimizer == "adadelta":                           # the separable corpus (test_gpu_lstm.py): the loss comes down
        first, last = sum(c[:50]) / 50, sum(c[-50:]) / 50
        assert last < 0.5 * first, (first, last)


def test_native_wgan_trains_with_grad_clip():
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN
    from theanompi_b200.utils.recorder import Recorder
    m = NativeWGAN(dict(verbose=False, rank=0, size=1, device="cuda:0", critic_runs=10, grad_clip=5.0,
                        data_kwargs=dict(n_synthetic=256)))
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "gan", False, device="cuda:0")
    w0, g0 = m.arena.W.clone(), m.gen_arena.W.clone()
    c = 0
    for _ in range(3):
        c = m.train_iter(c, rec)
    torch.cuda.synchronize()
    scores = [float(s) for s in m.critic_scores]
    assert all(math.isfinite(s) for s in scores)
    assert not torch.equal(w0, m.arena.W) and not torch.equal(g0, m.gen_arena.W)
    assert m.captured_steps()
    assert int(m.opt_c.skipped) == int(m.opt_g.skipped) == 0
    # the critic loss (fake − real) goes down: its recorded negation, the Wasserstein estimate, goes up
    assert sum(scores[-5:]) / 5 > sum(scores[:5]) / 5, scores
