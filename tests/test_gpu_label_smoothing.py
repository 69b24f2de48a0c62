"""Label smoothing on the H100: the smoothing instantiation of softmax_xent_kernel against the fp64 torch oracle in bf16 and fp32,
bit-identity of ε = 0 with an absent key and of graph replay with eager steps under TMPI_DETERMINISTIC=1 (in a subprocess), native
models with ε = 0.1 against their CPU reference path, the launch count, and a two-GPU fused BSP run."""
import math
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from theanompi_b200.ops import precision  # noqa: E402


# --------------------------------------------------------------------------- kernel
@pytest.mark.parametrize("eps", [0.1, 0.5, 1.0])
@pytest.mark.parametrize("C", [2, 10, 1000, 1001])
@pytest.mark.parametrize("B", [1, 37, 128])
@pytest.mark.parametrize("mode", ["bf16", "tf32"])
def test_kernel_matches_fp64_cross_entropy(mode, B, C, eps):
    """weight · F.cross_entropy(label_smoothing=ε) and its gradient times weight · grad_scale, in fp64 on the same logits.  bf16
    logits: loss within 1e-3, dlogits within 2e-2 of the largest (test_gpu_kernels.py::test_softmax_xent); fp32 logits (the tf32
    mode): 1e-4 relative.  err1 / err5 are bit-equal to the ε = 0 launch."""
    from theanompi_b200.ops import cuda_impl
    old = precision.precision()
    precision.set_precision(mode)
    try:
        g = torch.Generator(device="cuda").manual_seed(B * 7919 + C)
        lg = (torch.randn(B, C, device="cuda", generator=g) * 3).to(precision.act_dtype())
        lab = torch.randint(0, C, (B,), device="cuda", generator=g)
        weight, grad_scale = 0.3, 0.25
        loss, e1, e5, dl = cuda_impl.softmax_xent(lg, lab, weight=weight, grad_scale=grad_scale, label_smoothing=eps)
        _, e1_0, e5_0, _ = cuda_impl.softmax_xent(lg, lab, weight=weight, grad_scale=grad_scale)
        torch.cuda.synchronize()
    finally:
        precision.set_precision(old)
    x = lg.double().requires_grad_(True)
    want = weight * F.cross_entropy(x, lab, label_smoothing=eps)
    want.backward()
    dwant = x.grad * grad_scale
    err_loss = abs(float(loss) - float(want.detach()))
    err_dl = float((dl.double() - dwant).abs().max()) / float(dwant.abs().max())
    if mode == "bf16":
        assert err_loss < 1e-3 and err_dl < 2e-2, (err_loss, err_dl)
    else:
        assert err_loss < 1e-4 * max(1.0, abs(float(want.detach()))) and err_dl < 1e-4, (err_loss, err_dl)
    assert torch.equal(e1, e1_0) and torch.equal(e5, e5_0)


# --------------------------------------------------------------------------- models
IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))
ALEX = ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, no_paraload=True, **IMNET))


def _model(mod, cls, dev, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device=dev, **cfg))
    m.rand_crop = False
    layers2.Dropout.SetDropoutOff(); layers2.Crop.SetRandCropOff()
    m.compile_iter_fns("avg")
    return m


def _train(m, steps, dev):
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device=dev)
    for i in range(steps):
        m.train_iter(i, rec)
    if dev != "cpu":
        torch.cuda.synchronize()
    return [float(c) for c in rec.train_info["cost"]]


def alexnet_runs(runs, steps=6):
    """AlexNet-128b bf16, ``runs`` = [(name, cuda_graph, extra config)]: name → (W, U, losses, graph captured)."""
    from theanompi_b200.ops import cuda_impl
    mod, cls, cfg = ALEX
    out = {}
    for name, graph, extra in runs:
        cuda_impl._STEP.clear()
        m = _model(mod, cls, "cuda:0", cuda_graph=graph, **dict(cfg, **extra))
        losses = _train(m, steps, "cuda:0")
        out[name] = (m.arena.W.clone(), m.arena.U.clone(), losses, "step" in m.captured_steps())
        m.cleanup()
        del m
    return out


def _subprocess(code, timeout=900):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


def test_zero_epsilon_graph_steps_equal_an_absent_key():
    _subprocess("""
import test_gpu_label_smoothing as t
o = t.alexnet_runs([("absent", True, {}), ("zero", True, dict(label_smoothing=0.0))])
(wa, ua, la, ga), (wz, uz, lz, gz) = o["absent"], o["zero"]
print('losses', la, lz, 'graphs', ga, gz)
assert ga and gz and la[-1] == lz[-1]
assert t.torch.equal(wa, wz) and t.torch.equal(ua, uz)
print('OK')
""")


def test_smoothed_graph_replay_equals_eager_steps():
    _subprocess("""
import test_gpu_label_smoothing as t
o = t.alexnet_runs([("eager", False, dict(label_smoothing=0.1)), ("graph", True, dict(label_smoothing=0.1)),
                    ("plain", True, {})])
(we, ue, le, ge), (wg, ug, lg, gg), (wp, up, lp, gp) = o["eager"], o["graph"], o["plain"]
print('losses eager', le, 'graph', lg, 'plain', lp, 'max |dW| graph/eager %g' % float((wg - we).abs().max()))
assert gg and not ge and le[-1] == lg[-1]
assert t.torch.equal(we, wg) and t.torch.equal(ue, ug)
assert not t.torch.equal(wg, wp)                      # the captured step really smooths
print('OK')
""")


MODELS = {
    "alexnet": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=8, file_batch_size=16, **IMNET), 3),
    "googlenet": ("theanompi_b200.models.googlenet", "GoogLeNet", dict(batch_size=8, file_batch_size=16, no_paraload=True, **IMNET), 3),
    "resnet50_lars_accum4": ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50",
                             dict(batch_size=8, file_batch_size=8, blocks=(1, 1, 1, 1), no_paraload=True, optimizer="lars",
                                  learning_rate=0.5, grad_accum=4, **IMNET), 8),
    "wrn_adam": ("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
                 dict(batch_size=16, file_batch_size=32, depth=10, widen=2, data_kwargs=dict(n_synthetic=256, synthetic=True)), 3),
}


@pytest.mark.parametrize("which", list(MODELS))
def test_models_match_cpu_reference(which, monkeypatch):
    """ε = 0.1, the native model against the same model on the CPU reference ops, same weights and batches: every step's smoothed
    loss within the tolerance of test_gpu_models.py's residual-net comparison.  GoogLeNet trains with dropout on so that its two
    auxiliary heads contribute (smoothed, weight 0.3); dropout is the identity in both runs because the two paths draw different
    masks."""
    from theanompi_b200 import ops
    from theanompi_b200.models import layers2
    mod, cls, cfg, steps = MODELS[which]
    monkeypatch.setattr(ops, "dropout", lambda x, p_drop, training, layer_id=0: x)
    losses = {}
    try:
        for dev in ("cpu", "cuda:0"):
            m = _model(mod, cls, dev, cuda_graph=False, label_smoothing=0.1, **cfg)
            if which == "googlenet":
                m.shared_lr.set_value(2e-4)           # its default lr diverges within three steps without dropout
                layers2.Dropout.SetDropoutOn()
                assert layers2.Dropout.layers[0].flag_on
            losses[dev] = _train(m, steps, dev)
            m.cleanup()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(which, losses)
    assert len(losses["cpu"]) == len(losses["cuda:0"]) == steps
    for a, b in zip(losses["cpu"], losses["cuda:0"]):
        assert math.isfinite(b) and abs(a - b) < 0.08 * max(1.0, abs(a)), losses


def test_lstm_two_buckets_matches_cpu_reference(monkeypatch):
    """The LSTM with ε = 0.1 over batches alternating between the 16- and 48-step buckets (one graph each on the GPU) against the
    CPU reference path, dropout taken out; the tolerance of test_gpu_lstm.py's bf16 comparison."""
    import numpy as np
    from theanompi_b200 import ops
    from theanompi_b200.models import layers2
    from theanompi_b200.models.lstm import LSTM
    monkeypatch.setattr(ops, "dropout", lambda x, p_drop, training, layer_id=0: x)
    rs = np.random.RandomState(0)
    batches = []
    for i in range(8):
        L = 10 if i % 2 == 0 else 40
        batches.append((rs.randint(2, 500, (16, L)).astype(np.int64), np.ones((16, L), np.float32), rs.randint(0, 2, 16).astype(np.int64)))
    costs, graphs = {}, None
    for dev in ("cpu", "cuda:0"):
        layers2.reseed()
        m = LSTM(dict(verbose=False, rank=0, size=1, device=dev, dim_proj=64, label_smoothing=0.1,
                      data_kwargs=dict(n_synthetic=64, n_words=500)))
        m.compile_iter_fns("avg")
        m._train_it = iter(batches)
        costs[dev] = _train(m, len(batches), dev)
        if dev != "cpu":
            graphs = sorted(m.captured_steps())
    print(costs, graphs)
    assert graphs == [16, 48], graphs
    for a, b in zip(costs["cpu"], costs["cuda:0"]):
        assert abs(a - b) < 0.02 * max(1.0, abs(a)), costs


def test_launch_count_does_not_change():
    """A step with ε = 0.1 runs as many native launches as one with ε = 0: AlexNet k = 1 and each grad_accum micro-step kind of
    ResNet50."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    try:
        mod, cls, cfg = ALEX
        for eps in (0.0, 0.1):
            m = _model(mod, cls, "cuda:0", cuda_graph=False, label_smoothing=eps, **dict(cfg, batch_size=16, file_batch_size=16))
            for _ in range(2):
                torch.cuda.synchronize()
                native.reset_launch_count()
                m.forward_backward(0)
                torch.cuda.synchronize()
                counts[("alexnet", eps)] = native.launch_count()
        mod, cls, cfg, _ = MODELS["resnet50_lars_accum4"]
        for eps in (0.0, 0.1):
            m = _model(mod, cls, "cuda:0", cuda_graph=False, label_smoothing=eps, **cfg)
            for _ in range(4):
                kind = m.micro_step_kind()
                torch.cuda.synchronize()
                native.reset_launch_count()
                m.forward_backward(0)
                torch.cuda.synchronize()
                counts[(kind, eps)] = native.launch_count()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(counts)
    for key in ("alexnet", "first", "mid", "last"):
        assert counts[(key, 0.1)] == counts[(key, 0.0)] > 10, counts


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_fused_bsp_two_gpus(tmp_path, monkeypatch):
    """BSP sync_type='cdd' over the fused exchange on two GPUs with label_smoothing = 0.1 in rule.model_config."""
    import theanompi_b200 as tm
    monkeypatch.chdir(tmp_path)
    tm.BSP.sync_type, tm.BSP.exch_strategy = "cdd", "fused"
    rule = tm.BSP()
    rule.model_config = dict(batch_size=64, file_batch_size=64, n_epochs=1, learning_rate=0.001, max_batches=12, printFreq=4,
                             label_smoothing=0.1, data_kwargs=dict(n_synthetic=2048, synthetic=True))
    rule.init(devices=["cuda0", "cuda1"], modelfile="theanompi_b200.models.cifar10", modelclass="Cifar10_model")
    try:
        assert rule.proc.wait(timeout=300) == 0
    except subprocess.TimeoutExpired:
        rule.proc.kill()
        raise
