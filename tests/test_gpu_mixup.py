"""Mixup / CutMix on the H100: ``mix_draw_kernel`` against ``reference.mix_draw`` over thousands of draws in one launch,
``mix_batch_kernel`` (vector and scalar paths) and the mixing ``softmax_xent`` instantiation against the reference, native models with
Mixup and CutMix against their CPU reference path driven by the records the device wrote, bit-identity under TMPI_DETERMINISTIC=1 (in a
subprocess) of steps without the key and of graph replay with eager steps, the launch count, and a two-GPU fused BSP run."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from theanompi_b200.ops import mixup, precision  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

CONFIGS = [dict(alpha=0.2), dict(alpha=1.0), dict(alpha=4.0), dict(cutmix_alpha=0.2), dict(cutmix_alpha=1.0), dict(cutmix_alpha=4.0),
           dict(alpha=1.0, prob=0.7), dict(alpha=0.4, cutmix_alpha=1.0), dict(alpha=0.4, cutmix_alpha=1.0, switch_prob=0.2, prob=0.6),
           dict(cutmix_alpha=2.0, prob=0.9), dict(alpha=16.0, cutmix_alpha=16.0, seed=2 ** 40 + 3)]


# --------------------------------------------------------------------------- mix_draw
@pytest.mark.parametrize("hw", [(32, 32), (227, 227)])
@pytest.mark.parametrize("k", range(len(CONFIGS)))
def test_draw_kernel_matches_reference(k, hw):
    """4096 draws in one launch (step counter values 1000 + t, rank 3): mode and centre equal to the reference's, λ within 2 fp32
    ulp, and the box the host recomputes from the device's own raw λ and centre equal to the device's box."""
    from theanompi_b200.ops import cuda_impl
    cfg = mixup.check_config(CONFIGS[k])
    n, start, rank = 4096, 1000 + 7919 * k, 3
    step = torch.full((1,), start, dtype=torch.int64, device="cuda")
    dev = mixup.decode(cuda_impl.mix_draw(cfg, rank, hw, step, n=n))
    want = ref.mix_draw(cfg, cfg["seed"], rank, np.arange(start, start + n), hw)
    assert np.array_equal(dev["mode"], want["mode"])
    for f in ("cy", "cx", "H", "W"):
        assert np.array_equal(dev[f], want[f]), f
    ulp = np.spacing(np.abs(want["lam"]).astype(np.float32))
    assert (np.abs(dev["lam"] - want["lam"]) <= 2 * ulp).all()
    assert np.allclose(dev["lam_raw"], want["lam_raw"], rtol=1e-12, atol=1e-15)
    H, W = hw
    cut = dev[dev["mode"] == mixup.MIX_CUTMIX]
    r = np.sqrt(1.0 - cut["lam_raw"])
    ch, cw = (H * r).astype(np.int64), (W * r).astype(np.int64)
    y0, y1 = np.clip(cut["cy"] - ch // 2, 0, H), np.clip(cut["cy"] + ch // 2, 0, H)
    x0, x1 = np.clip(cut["cx"] - cw // 2, 0, W), np.clip(cut["cx"] + cw // 2, 0, W)
    assert np.array_equal(cut["y0"], y0) and np.array_equal(cut["y1"], y1)
    assert np.array_equal(cut["x0"], x0) and np.array_equal(cut["x1"], x1)
    assert np.array_equal(cut["lam"], (1.0 - (y1 - y0) * (x1 - x0) / float(H * W)).astype(np.float32))
    assert np.array_equal(dev[dev["mode"] == mixup.MIX_MIXUP]["lam"], dev[dev["mode"] == mixup.MIX_MIXUP]["lam_raw"].astype(np.float32))


def test_draw_reads_the_device_counter():
    """The training step's launch (n = 1) draws the record of the current device counter value."""
    from theanompi_b200.ops import cuda_impl
    cfg = mixup.check_config(dict(alpha=1.0))
    step = torch.full((1,), 41, dtype=torch.int64, device="cuda")
    out = torch.zeros(mixup.RECORD_BYTES, dtype=torch.uint8, device="cuda")
    cuda_impl.mix_draw(cfg, 0, (32, 32), step, out=out)
    a = float(mixup.decode(out)["lam_raw"])
    step += 1
    cuda_impl.mix_draw(cfg, 0, (32, 32), step, out=out)
    b = float(mixup.decode(out)["lam_raw"])
    want = ref.mix_draw(cfg, 0, 0, np.array([41, 42]), (32, 32))["lam_raw"]
    assert np.allclose([a, b], want, rtol=1e-12) and a != b


# --------------------------------------------------------------------------- mix_batch
def _ulp_close(a, b):
    """Elementwise: equal, or one unit in the last place apart (same storage type)."""
    it = torch.int16 if a.dtype == torch.bfloat16 else torch.int32
    ai, bi = a.contiguous().view(it).long(), b.contiguous().view(it).long()
    return bool(((a == b) | ((ai - bi).abs() <= 1)).all())


@pytest.mark.parametrize("hw", [(227, 227), (32, 32)])
@pytest.mark.parametrize("B", [1, 2, 37, 128])
@pytest.mark.parametrize("mode", ["bf16", "tf32"])
def test_mix_batch_kernel_matches_reference(mode, B, hw):
    """227·227·3 rows take the scalar path (309,174 bytes in bf16), 32·32·3 rows the 16-byte vector path.  CutMix and the unmixed
    record are bit-exact, Mixup within one ulp of the activation dtype."""
    from theanompi_b200.ops import cuda_impl
    dt = torch.bfloat16 if mode == "bf16" else torch.float32
    H, W = hw
    g = torch.Generator(device="cuda").manual_seed(B * H)
    x = (torch.randn(B, H, W, 3, device="cuda", generator=g) * 30).to(dt)
    cut = mixup.check_config(dict(cutmix_alpha=1.0))
    recs = {"none": ref.mix_draw(mixup.check_config(dict(alpha=1.0, prob=0.0)), 0, 0, 5, hw),
            "mixup": ref.mix_draw(mixup.check_config(dict(alpha=1.0)), 0, 0, 5, hw)}
    cuts = ref.mix_draw(cut, 0, 0, np.arange(64), hw)
    recs["cutmix"] = cuts[np.argmin(np.abs(cuts["lam"] - 0.6))]              # a box of about 40 % of the image, off-centre
    recs["cutmix_edge"] = cuts[np.argmax((cuts["y0"] == 0) | (cuts["x1"] == W))]
    for name, r in recs.items():
        y = x.clone()
        rec = mixup.encode(r).cuda()
        assert cuda_impl.mix_batch(y, rec) is y
        want = ref.mix_batch(x.cpu(), r)
        got = y.cpu()
        if name == "mixup":
            assert _ulp_close(got, want), name
        else:
            assert torch.equal(got, want), name
        if name == "none":
            assert torch.equal(y, x)


# --------------------------------------------------------------------------- softmax_xent(mix=)
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("C", [2, 10, 1000, 1001])
@pytest.mark.parametrize("B", [1, 37, 128])
@pytest.mark.parametrize("mode", ["bf16", "tf32"])
def test_mixing_softmax_matches_fp64_cross_entropy(mode, B, C, eps):
    """weight · F.cross_entropy against the mixed probability target q and its gradient times weight · grad_scale, fp64 on the same
    logits, with the label-smoothing test's tolerances; err1 / err5 bit-equal to the plain launch on the larger-weight label."""
    from theanompi_b200.ops import cuda_impl
    old = precision.precision()
    precision.set_precision(mode)
    try:
        g = torch.Generator(device="cuda").manual_seed(B * 7919 + C)
        lg = (torch.randn(B, C, device="cuda", generator=g) * 3).to(precision.act_dtype())
        lab = torch.randint(0, C, (B,), device="cuda", generator=g)
        weight, grad_scale = 0.3, 0.25
        for r in (ref.mix_draw(mixup.check_config(dict(alpha=1.0)), 0, 0, 2, (32, 32)),
                  ref.mix_draw(mixup.check_config(dict(cutmix_alpha=1.0)), 0, 0, 3, (32, 32)),
                  ref.mix_draw(mixup.check_config(dict(alpha=1.0, prob=0.0)), 0, 0, 3, (32, 32))):
            rec = mixup.encode(r).cuda()
            loss, e1, e5, dl = cuda_impl.softmax_xent(lg, lab, weight=weight, grad_scale=grad_scale, label_smoothing=eps, mix=rec)
            lam = ref.mix_lambda(r)
            ye = lab if lam >= 0.5 else lab.flip(0)
            _, e1_0, e5_0, _ = cuda_impl.softmax_xent(lg, ye)
            torch.cuda.synchronize()
            x = lg.double().requires_grad_(True)
            soft = lambda t: (1 - eps) * F.one_hot(t, C).double() + eps / C      # noqa: E731
            want = weight * F.cross_entropy(x, lam * soft(lab) + (1 - lam) * soft(lab.flip(0)))
            want.backward()
            dwant = x.grad * grad_scale
            err_loss = abs(float(loss) - float(want.detach()))
            err_dl = float((dl.double() - dwant).abs().max()) / float(dwant.abs().max())
            if mode == "bf16":
                assert err_loss < 1e-3 and err_dl < 2e-2, (int(r["mode"]), err_loss, err_dl)
            else:
                assert err_loss < 1e-4 * max(1.0, abs(float(want.detach()))) and err_dl < 1e-4, (int(r["mode"]), err_loss, err_dl)
            assert torch.equal(e1, e1_0) and torch.equal(e5, e5_0)
    finally:
        precision.set_precision(old)


# --------------------------------------------------------------------------- models
IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))
ALEX = ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, no_paraload=True, **IMNET))
MIXES = {"mixup": dict(alpha=1.0, seed=3), "cutmix": dict(cutmix_alpha=1.0, seed=4)}


def _model(mod, cls, dev, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device=dev, **cfg))
    m.rand_crop = False
    layers2.Dropout.SetDropoutOff(); layers2.Crop.SetRandCropOff()
    m.compile_iter_fns("avg")
    return m


def _train(m, steps, dev, recs=None):
    """``steps`` training steps: the recorded costs, and the mix record of every step (``recs``: replay these records instead of
    drawing)."""
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device=dev)
    seen = []
    if recs is not None:
        it = iter(recs)
        m.mixer.draw = lambda: m.mixer.rec.copy_(next(it))
    for i in range(steps):
        m.train_iter(i, rec)
        if m.mixer is not None:
            seen.append(m.mixer.rec.cpu().clone())
    if dev != "cpu":
        torch.cuda.synchronize()
    return [float(c) for c in rec.train_info["cost"]], seen


def alexnet_runs(runs, steps=6):
    """AlexNet-128b bf16, ``runs`` = [(name, cuda_graph, extra config)]: name → (W, U, losses, graph captured)."""
    from theanompi_b200.ops import cuda_impl
    mod, cls, cfg = ALEX
    out = {}
    for name, graph, extra in runs:
        cuda_impl._STEP.clear()
        m = _model(mod, cls, "cuda:0", cuda_graph=graph, **dict(cfg, **extra))
        losses, _ = _train(m, steps, "cuda:0")
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


def test_steps_without_the_key_are_unchanged():
    _subprocess("""
import test_gpu_mixup as t
o = t.alexnet_runs([("absent", True, {}), ("none", True, dict(mixup=None)), ("eager", False, {})])
(wa, ua, la, ga), (wn, un, ln, gn), (we, ue, le, ge) = o["absent"], o["none"], o["eager"]
print('losses', la, ln, le, 'graphs', ga, gn, ge)
assert ga and gn and not ge and la[-1] == ln[-1] == le[-1]
assert t.torch.equal(wa, wn) and t.torch.equal(ua, un) and t.torch.equal(wa, we) and t.torch.equal(ua, ue)
print('OK')
""")


def test_mixed_graph_replay_equals_eager_steps():
    _subprocess("""
import test_gpu_mixup as t
runs = []
for k, mx in t.MIXES.items():
    runs += [(k + "_eager", False, dict(mixup=mx)), (k + "_graph", True, dict(mixup=mx))]
o = t.alexnet_runs(runs + [("plain", True, {})])
wp = o["plain"][0]
for k in t.MIXES:
    (we, ue, le, ge), (wg, ug, lg, gg) = o[k + "_eager"], o[k + "_graph"]
    print(k, 'losses eager', le, 'graph', lg, 'max |dW| graph/eager %g' % float((wg - we).abs().max()))
    assert gg and not ge and le[-1] == lg[-1]
    assert t.torch.equal(we, wg) and t.torch.equal(ue, ug)
    assert not t.torch.equal(wg, wp)                      # the captured step really mixes
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
    "cifar10": ("theanompi_b200.models.cifar10", "Cifar10_model",
                dict(batch_size=32, file_batch_size=32, learning_rate=0.01, data_kwargs=dict(n_synthetic=512, synthetic=True)), 3),
}


@pytest.mark.parametrize("kind", list(MIXES))
@pytest.mark.parametrize("which", list(MODELS))
def test_models_match_cpu_reference(which, kind, monkeypatch):
    """The native model with Mixup / CutMix against the same model on the CPU reference ops, same weights and batches, the CPU
    replaying the records the device drew: every step's mixed loss within the tolerance of test_gpu_models.py's residual-net
    comparison.  GoogLeNet trains with dropout on so that its two auxiliary heads contribute; dropout is the identity in both runs
    because the two paths draw different masks."""
    from theanompi_b200 import ops
    from theanompi_b200.models import layers2
    mod, cls, cfg, steps = MODELS[which]
    monkeypatch.setattr(ops, "dropout", lambda x, p_drop, training, layer_id=0: x)
    losses, recs = {}, None
    try:
        for dev in ("cuda:0", "cpu"):
            m = _model(mod, cls, dev, cuda_graph=False, mixup=MIXES[kind], **cfg)
            if which == "googlenet":
                m.shared_lr.set_value(2e-4)           # its default lr diverges within three steps without dropout
                layers2.Dropout.SetDropoutOn()
                assert layers2.Dropout.layers[0].flag_on
            losses[dev], seen = _train(m, steps, dev, recs)
            if recs is None:
                recs = seen
            m.cleanup()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    modes = [int(mixup.decode(r)["mode"]) for r in recs]
    print(which, kind, modes, losses)
    assert set(modes) == {mixup.MIX_MIXUP if kind == "mixup" else mixup.MIX_CUTMIX}
    assert len(losses["cpu"]) == len(losses["cuda:0"]) == steps
    for a, b in zip(losses["cpu"], losses["cuda:0"]):
        assert math.isfinite(b) and abs(a - b) < 0.08 * max(1.0, abs(a)), losses


def test_launch_count():
    """AlexNet-128b (1000 classes) runs 55 native launches per step without mixup and 57 with it: the draw and the mix; the loss keeps
    its two."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    try:
        for name, extra in (("off", {}), ("mixup", dict(mixup=MIXES["mixup"])), ("cutmix", dict(mixup=MIXES["cutmix"]))):
            m = _model("theanompi_b200.models.alex_net", "AlexNet", "cuda:0", cuda_graph=False, batch_size=128, file_batch_size=128,
                       no_paraload=True, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True), **extra)
            layers2.Dropout.SetDropoutOn()                        # a training step: its two dropout layers launch too
            for _ in range(2):
                torch.cuda.synchronize()
                native.reset_launch_count()
                m.forward_backward(0)
                torch.cuda.synchronize()
                counts[name] = native.launch_count()
            m.cleanup()
    finally:
        layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(counts)
    assert counts["off"] == 55 and counts["mixup"] == counts["cutmix"] == 57, counts


@pytest.mark.multigpu
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_fused_bsp_two_gpus(tmp_path, monkeypatch):
    """BSP sync_type='cdd' over the fused exchange on two GPUs with Mixup and CutMix in rule.model_config."""
    import theanompi_b200 as tm
    monkeypatch.chdir(tmp_path)
    tm.BSP.sync_type, tm.BSP.exch_strategy = "cdd", "fused"
    rule = tm.BSP()
    rule.model_config = dict(batch_size=64, file_batch_size=64, n_epochs=1, learning_rate=0.001, max_batches=12, printFreq=4,
                             mixup=dict(alpha=0.2, cutmix_alpha=1.0), data_kwargs=dict(n_synthetic=2048, synthetic=True))
    rule.init(devices=["cuda0", "cuda1"], modelfile="theanompi_b200.models.cifar10", modelclass="Cifar10_model")
    try:
        assert rule.proc.wait(timeout=300) == 0
    except subprocess.TimeoutExpired:
        rule.proc.kill()
        raise
