"""Knowledge distillation (``config['distill']``) on the CPU reference path: ``reference.softmax_xent_kd`` against the torch expression
(cross-entropy plus temperature-scaled KL divergence) in fp64, the model step against a manual composition (the teacher's eval forward on
x_in, the reference loss, the student's backward and optimizer) for an AlexNet and a small ResNet50 student, an unchanged teacher and
unchanged student draws, the teacher on the mixed batch, one teacher forward per SAM step, grad_accum's 1/n, label smoothing on the hard
term only, every refusal, the key off, checkpoints and BSP 'avg' / 'cdd' on two gloo ranks.

Also the child process of the two-rank test: ``python tests/test_distill_cpu.py bsp <avg|cdd> <checkpoint>`` with RANK / WORLD_SIZE set."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import BatchNormal, Crop, Dropout  # noqa: E402
from theanompi_b200.ops import functional, mixup, reference as ref  # noqa: E402
from theanompi_b200.ops.distill import check_config  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402

IMNET = dict(n_class=16, no_paraload=True, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
ALEX = "theanompi_b200.models.alex_net:AlexNet"
R50 = "theanompi_b200.models.lasagne_model_zoo.resnet50:ResNet50"
R152 = "theanompi_b200.models.lasagne_model_zoo.resnet152_outdated:ResNet152"
SMALL = (1, 1, 1, 1)


def _clear():
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear(); BatchNormal.layers.clear()


def _alex(rank=0, size=1, **kw):
    from theanompi_b200.models.alex_net import AlexNet
    _clear()
    cfg = dict(verbose=False, rank=rank, size=size, device="cpu", batch_size=4, file_batch_size=4, learning_rate=0.01, **IMNET)
    cfg.update(kw)
    m = AlexNet(cfg)
    m.rand_crop = False                                  # the serial loader's random crops come from numpy's global generator
    return m


def _r50(rank=0, size=1, **kw):
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    _clear()
    cfg = dict(verbose=False, rank=rank, size=size, device="cpu", batch_size=4, file_batch_size=4, learning_rate=0.05, blocks=SMALL,
               **IMNET)
    cfg.update(kw)
    m = ResNet50(cfg)
    m.rand_crop = False
    return m


def _rec():
    return Recorder(None, 10 ** 6, "c", False, device="cpu")


def _train(m, n=1):
    """``n`` training steps that leave the momentum and the batch-norm statistics non-trivial."""
    m.compile_iter_fns("avg")
    rec = _rec()
    for i in range(n):
        m.train_iter(i, rec)
    return m


@pytest.fixture(scope="module")
def ckpts(tmp_path_factory):
    """Checkpoints of a trained AlexNet (16 classes) and a trained small ResNet50, written by save_checkpoint."""
    from theanompi_b200.utils.helper_funcs import save_checkpoint
    d = tmp_path_factory.mktemp("teachers")
    step = functional._RNG["step"]
    out = {"alex": str(d / "ckpt_3.pt"), "r50": str(d / "ckpt_5.pt")}
    save_checkpoint(_train(_alex(learning_rate=0.02), 2), out["alex"])
    save_checkpoint(_train(_r50(), 2), out["r50"])
    functional._RNG["step"] = step
    _clear()
    return out


def _state(m):
    a = m.arena
    return [a.W.clone(), a.U.clone(), a.G.clone()] + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)]


def _assert_equal_lists(a, b, what=""):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i, float((x.double() - y.double()).abs().max()))


# ------------------------------------------------------------------ the reference against the torch expression
def _torch_loss(z, y, t, alpha, T, eps, lam):
    """The distillation loss as torch writes it: the (smoothed, mixed) cross-entropy and the batch-mean KL divergence."""
    hard = F.cross_entropy(z, y, label_smoothing=eps)
    if lam != 1.0:
        hard = lam * hard + (1.0 - lam) * F.cross_entropy(z, y.flip(0), label_smoothing=eps)
    kl = F.kl_div(F.log_softmax(z / T, 1), F.log_softmax(t / T, 1), reduction="batchmean", log_target=True)
    return (1.0 - alpha) * hard + alpha * T * T * kl


def _record(mode, lam):
    """A mix record (ops/mixup.py layout) of ``mode`` with effective weight ``lam``."""
    r = np.zeros((), dtype=mixup.RECORD)
    r["mode"], r["lam"], r["lam_raw"], r["H"], r["W"] = mode, lam, lam, 8, 8
    return mixup.encode(r)


MIXES = {"none": None, "mixup": (mixup.MIX_MIXUP, 0.7), "cutmix": (mixup.MIX_CUTMIX, 0.375)}


@pytest.mark.parametrize("mix", list(MIXES))
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("T", [1.0, 2.0, 4.0])
@pytest.mark.parametrize("alpha", [0.3, 1.0])
@pytest.mark.parametrize("B,C", [(4, 5), (8, 16), (6, 1000), (3, 37)])
def test_reference_equals_the_torch_expression(B, C, alpha, T, eps, mix):
    g = torch.Generator().manual_seed(B * 1000 + C)
    z = (torch.randn(B, C, generator=g, dtype=torch.float64) * 3).requires_grad_()
    t = torch.randn(B, C, generator=g, dtype=torch.float64) * 3
    y = torch.randint(0, C, (B,), generator=g)
    rec = None if MIXES[mix] is None else _record(*MIXES[mix])
    lam = 1.0 if rec is None else ref.mix_lambda(rec)
    loss, err1, err5, d = ref.softmax_xent_kd(z.detach(), y, t, alpha, T, label_smoothing=eps, mix=rec)
    want = _torch_loss(z, y, t, alpha, T, eps, lam)
    (grad,) = torch.autograd.grad(want, z)
    assert loss.dtype == torch.float64 and abs(float(loss) - float(want)) <= 1e-12 * max(1.0, abs(float(want)))
    assert float((d - grad).abs().max()) <= 1e-15 * max(1.0, float(grad.abs().max())) * C
    ye = y if lam >= 0.5 else y.flip(0)
    assert float(err1) == float((z.argmax(1) != ye).double().mean())
    assert float(err5) == 1.0 - float((z.topk(min(5, C), 1).indices == ye[:, None]).any(1).double().mean())
    # fp32: the same computation rounded to fp32
    l32, _, _, d32 = ref.softmax_xent_kd(z.detach().float(), y, t.float(), alpha, T, label_smoothing=eps, mix=rec)
    assert l32.dtype == torch.float32 and abs(float(l32) - float(want)) <= 1e-5 * max(1.0, abs(float(want)))
    assert float((d32.double() - grad).abs().max()) <= 1e-6


@pytest.mark.parametrize("T", [1.0, 2.0, 4.0])
def test_pure_function_matching_of_itself_is_zero(T):
    z = torch.randn(8, 100, dtype=torch.float64) * 5
    y = torch.randint(0, 100, (8,))
    for eps in (0.0, 0.1):
        loss, _, _, d = ref.softmax_xent_kd(z, y, z.clone(), 1.0, T, label_smoothing=eps)
        assert abs(float(loss)) <= 1e-13 and float(d.abs().max()) <= 1e-17


def test_label_smoothing_reaches_the_hard_term_only():
    g = torch.Generator().manual_seed(5)
    z, t = torch.randn(8, 20, generator=g, dtype=torch.float64), torch.randn(8, 20, generator=g, dtype=torch.float64)
    y = torch.randint(0, 20, (8,), generator=g)
    pure = [ref.softmax_xent_kd(z, y, t, 1.0, 2.0, label_smoothing=e) for e in (0.0, 0.3)]
    assert float(pure[0][0]) == float(pure[1][0]) and torch.equal(pure[0][3], pure[1][3])
    a, b = (ref.softmax_xent_kd(z, y, t, 0.5, 2.0, label_smoothing=e) for e in (0.0, 0.3))
    hard = [float(F.cross_entropy(z, y, label_smoothing=e)) for e in (0.0, 0.3)]
    assert abs((float(b[0]) - float(a[0])) - 0.5 * (hard[1] - hard[0])) <= 1e-12


def test_grad_accum_scales_the_gradient():
    z = torch.randn(4, 10).requires_grad_()
    t, y = torch.randn(4, 10), torch.randint(0, 10, (4,))
    grads = []
    for scale in (1.0, 0.25):
        z.grad = None
        with ops.accum.mode(False, scale):
            loss, _, _ = ops.softmax_xent_kd(z, y, t, 0.4, 3.0)
        loss.backward()
        grads.append(z.grad.clone())
    assert torch.equal(grads[1], grads[0] * 0.25)


# ------------------------------------------------------------------ the model step against a manual composition
def _load_teacher(m, builder, path, **kw):
    """The teacher built and loaded by hand (after the student, so that the student's layer ids are its own), in eval mode."""
    from theanompi_b200.utils.helper_funcs import load_checkpoint
    n_d, n_b = len(Dropout.layers), len(BatchNormal.layers)
    rng = layers2.rng
    t = builder(batch_size=m.batch_size, file_batch_size=m.batch_size, clear=False, **kw)
    layers2.rng = rng
    del Dropout.layers[n_d:], BatchNormal.layers[n_b:]
    load_checkpoint(t, path)
    for l in t.layers:
        if isinstance(l, Dropout):
            l.flag_on = False
        if isinstance(l, BatchNormal):
            l.training = False
    return t


def _manual_step_fn(m, teacher, alpha, T):
    """The train_iter_fn of a student built without the key that does, from the model's own pieces: the draws and the mix, the
    teacher's eval forward on x_in, the student's forward, the reference loss, its backward, the step tail."""
    def step(subb=0):
        B = m.batch_size
        m.x_in.copy_(m.shared_x[subb * B:(subb + 1) * B])
        m.y_in.copy_(m.shared_y[subb * B:(subb + 1) * B])
        m.n_updates += 1
        m._schedule_lr()
        rec = None
        if m.mixer is not None:
            rec = m.mixer.draw()
            m.mix_input(rec)
        if m.drop_path is not None:
            m.drop_path.draw()
        with torch.no_grad():
            t = teacher.forward(m.x_in).clone()
        m._drop_on = m.drop_path is not None
        z = m.forward(m.x_in)
        m._drop_on = False
        loss, err, _, d = ref.softmax_xent_kd(z.detach(), m.y_in, t, alpha, T, label_smoothing=m.label_smoothing, mix=rec)
        z.backward(d)
        if m._tail is not None:                             # BSP 'cdd': get_vel runs the exchange's pre() instead
            with torch.no_grad():
                m._tail()
        m._after_step()
        return loss, err
    return step


def _builder(which):
    def b(clear=True, **kw):
        if not clear:
            from theanompi_b200.models.alex_net import AlexNet
            from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
            cls = AlexNet if which == "alex" else ResNet50
            base = dict(verbose=False, rank=0, size=1, device="cpu", **IMNET)
            if which == "r50":
                base["blocks"] = SMALL
            base.update(kw)
            m = cls(base)
            m.rand_crop = False
            return m
        return (_alex if which == "alex" else _r50)(**kw)
    return b


CASES = {
    "alex": ("alex", ALEX, {}, dict(alpha=0.7, temperature=4.0), {}),
    "alex_smooth_mix": ("alex", ALEX, {}, dict(alpha=0.5, temperature=2.0),
                        dict(label_smoothing=0.1, mixup=dict(alpha=0.8, cutmix_alpha=1.0))),
    "r50_drop_path_lars": ("r50", R152, dict(blocks=list(SMALL)), dict(alpha=1.0, temperature=1.0),
                           dict(drop_path_rate=0.2, optimizer="lars")),
}


@pytest.mark.parametrize("case", list(CASES))
def test_model_step_equals_manual_composition(case, ckpts):
    which, teacher, tcfg, kd, kw = CASES[case]
    build = _builder(which)
    dist = dict(teacher=teacher, checkpoint=ckpts[which], config=tcfg, **kd)
    on = build(distill=dist, **kw)
    on.compile_iter_fns("avg")
    man = build(**kw)
    man.compile_iter_fns("avg")
    t = _load_teacher(man, build, ckpts[which])
    man.train_iter_fn = _manual_step_fn(man, t, kd["alpha"], kd["temperature"])
    rec = _rec()
    for i in range(3):
        step = functional._RNG["step"]
        on.train_iter(i, rec)
        functional._RNG["step"] = step                       # the manual model draws the same step
        man.train_iter(i, rec)
        _assert_equal_lists(_state(on), _state(man), (case, i))


def test_teacher_unchanged_and_student_draws_unchanged(ckpts):
    cfg = dict(mixup=dict(alpha=1.0, cutmix_alpha=1.0), drop_path_rate=0.3, learning_rate=0.05)
    on = _r50(distill=dict(teacher=R50, checkpoint=ckpts["r50"], config=dict(blocks=SMALL), alpha=0.5, temperature=2.0), **cfg)
    on.compile_iter_fns("avg")
    t = on.distiller.teacher
    assert all(l not in BatchNormal.layers for l in t._bn_layers()) and all(l in BatchNormal.layers for l in on._bn_layers())
    sd = torch.load(ckpts["r50"], map_location="cpu", weights_only=False)
    assert torch.equal(t.arena.W, sd["arena"]["W"]) and torch.equal(t.arena.U, sd["arena"]["U"])
    off = _r50(**cfg)
    off.compile_iter_fns("avg")
    seen = {"on": [], "off": []}
    for key, m in (("on", on), ("off", off)):
        draw, dp = m.mixer.draw, m.drop_path.draw
        m.mixer.draw = lambda draw=draw, key=key: (seen[key].append(draw().clone()), seen[key][-1])[1]
        m.drop_path.draw = lambda dp=dp, key=key, m=m: (dp(), seen[key].append(m.drop_path.table.clone()))[0]
    rec = _rec()
    for i in range(3):
        step = functional._RNG["step"]
        on.train_iter(i, rec)
        functional._RNG["step"] = step
        off.train_iter(i, rec)
    _assert_equal_lists(seen["on"], seen["off"], "draws")
    assert len(seen["on"]) == 6
    assert torch.equal(t.arena.W, sd["arena"]["W"]) and torch.equal(t.arena.U, sd["arena"]["U"])
    assert not t.arena.G.any()
    for l, (mu, var) in zip(t._bn_layers(), sd["extra_state"]["bn"]):
        assert torch.equal(l.running_mean, mu) and torch.equal(l.running_var, var)


def test_teacher_layers_leave_the_class_lists(ckpts):
    on = _alex(distill=dict(teacher=ALEX, checkpoint=ckpts["alex"]))
    ids = [l.layer_id for l in Dropout.layers]
    state = layers2.rng.get_state()
    on.compile_iter_fns("avg")
    assert [l.layer_id for l in Dropout.layers] == ids == [0, 1] and Dropout.layers[0] in on.layers
    after = layers2.rng.get_state()
    assert np.array_equal(state[1], after[1]) and state[2] == after[2]
    Dropout.SetDropoutOn(); BatchNormal.SetTrainOn()
    d = on.distiller
    kd = d.target(on.x_in)
    assert all(not l.flag_on for l in d._dropouts) and len(d._dropouts) == 2
    assert all(l.flag_on for l in Dropout.layers)
    with torch.no_grad():
        again = d.teacher.forward(on.x_in)
    assert torch.equal(kd.logits, again)                     # eval: no dropout mask, the same logits


def test_teacher_sees_the_mixed_batch_and_sam_runs_it_once(ckpts):
    dist = dict(teacher=R50, checkpoint=ckpts["r50"], config=dict(blocks=SMALL))
    m = _r50(distill=dist, mixup=dict(alpha=1.0), sam=dict(rho=0.05))
    m.compile_iter_fns("avg")
    seen, kds = [], []
    fwd = m.distiller.teacher.forward
    m.distiller.teacher.forward = lambda x: (seen.append(x.clone()), fwd(x))[1]
    tp = m._train_pass
    m._train_pass = lambda rec, kd=None: (kds.append(kd), tp(rec, kd))[1]
    rec = _rec()
    for i in range(2):
        del seen[:], kds[:]
        m.train_iter(i, rec)
        assert len(seen) == 1 and len(kds) == 2 and kds[0] is kds[1] and kds[0] is not None
        assert torch.equal(seen[0], m.x_in)                    # x_in holds the batch as mixed in place
        assert not torch.equal(seen[0], m.shared_x[:m.batch_size])


def test_grad_accum_window_trains(ckpts):
    dist = dict(teacher=R50, checkpoint=ckpts["r50"], config=dict(blocks=SMALL), alpha=0.5, temperature=2.0)
    m = _r50(distill=dist, grad_accum=2, batch_size=2)
    m.compile_iter_fns("avg")
    calls = []
    fwd = m.distiller.teacher.forward
    m.distiller.teacher.forward = lambda x: (calls.append(1), fwd(x))[1]
    w0 = m.arena.W.clone()
    rec = _rec()
    for i in range(2):
        m.train_iter(i, rec)
    assert len(calls) == 2 and m.n_updates == 1 and not torch.equal(w0, m.arena.W) and torch.isfinite(m.arena.W).all()


# ------------------------------------------------------------------ the key
@pytest.mark.parametrize("bad", [
    "on", [1], True, dict(teacher=ALEX, checkpoint="x", foo=1), dict(checkpoint="x"), dict(teacher="alex_net.AlexNet", checkpoint="x"),
    dict(teacher=":AlexNet", checkpoint="x"), dict(teacher=ALEX), dict(teacher=ALEX, checkpoint=""),
    dict(teacher=ALEX, checkpoint="x", alpha=True), dict(teacher=ALEX, checkpoint="x", alpha=0.0),
    dict(teacher=ALEX, checkpoint="x", alpha=1.5), dict(teacher=ALEX, checkpoint="x", alpha=float("nan")),
    dict(teacher=ALEX, checkpoint="x", alpha="0.5"), dict(teacher=ALEX, checkpoint="x", temperature=0.0),
    dict(teacher=ALEX, checkpoint="x", temperature=-1.0), dict(teacher=ALEX, checkpoint="x", temperature=float("inf")),
    dict(teacher=ALEX, checkpoint="x", temperature=False), dict(teacher=ALEX, checkpoint="x", config=[1]),
    dict(teacher=ALEX, checkpoint="x", config=dict(batch_size=8)), dict(teacher=ALEX, checkpoint="x", config=dict(blocks=[0, 1])),
    dict(teacher=ALEX, checkpoint="x", config=dict(n_class=10))])
def test_malformed_values_are_refused(bad):
    with pytest.raises(ValueError, match="distill"):
        check_config(bad)


def test_refusals_at_compile_iter_fns(ckpts, tmp_path):
    good = dict(teacher=R50, checkpoint=ckpts["r50"], config=dict(blocks=SMALL))
    cases = [
        (dict(good, alpha=2.0), "distill\\['alpha'\\]"),
        (dict(good, teacher="theanompi_b200.models.nope:ResNet50"), "cannot be imported"),
        (dict(good, teacher="theanompi_b200.models.lasagne_model_zoo.resnet50:Nope"), "cannot be imported"),
        (dict(good, teacher="theanompi_b200.models.lasagne_model_zoo.resnet50:ResNet50Torch"), "is not supported"),
        (dict(good, teacher="theanompi_b200.models.keras_model_zoo.wresnet:Wide_ResNet"), "is not supported"),
        (dict(good, teacher=ALEX, config={}), "takes \\(H, W, C\\)"),
        (dict(good, checkpoint=str(tmp_path / "missing.pt")), "no checkpoint"),
        (dict(good, config=dict(blocks=(1, 1, 2, 1))), "does not match the layout"),
        (dict(good, config=dict(batch_size=2)), "distill\\['config'\\]"),
    ]
    for dist, msg in cases:
        m = _r50(distill=dist)
        with pytest.raises(ValueError, match=msg):
            m.compile_iter_fns("avg")
    empty = tmp_path / "ckpt_0.pt"
    torch.save({"epoch": 0}, str(empty))
    m = _r50(distill=dict(good, checkpoint=str(empty)))
    with pytest.raises(ValueError, match="does not match the layout"):
        m.compile_iter_fns("avg")
    m = _alex(distill=dict(teacher=ALEX, checkpoint=ckpts["alex"]), n_class=10)
    with pytest.raises(ValueError, match="does not match the layout"):
        m.compile_iter_fns("avg")


def test_unsupported_models_are_refused(ckpts):
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet, Wide_ResNetTorch
    from theanompi_b200.models.lasagne_model_zoo.lsgan import NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.wgan import WGAN, NativeWGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    from theanompi_b200.models.torch_base import TorchModelBase
    for cls in (AlexNet_sc, Cifar10_model, Wide_ResNet, Wide_ResNetTorch, NativeWGAN, NativeLSGAN, WGAN, LSTM, LSTMTorch, ResNet50Torch,
                TorchModelBase):
        assert cls.supports_distill is False, cls
    dist = dict(teacher=ALEX, checkpoint=ckpts["alex"])
    _clear()
    models = [Cifar10_model(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, distill=dist,
                                 data_kwargs=dict(n_synthetic=640, synthetic=True))),
              Wide_ResNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=8, file_batch_size=8, depth=10, widen=1, distill=dist,
                               data_kwargs=dict(n_synthetic=64, synthetic=True))),
              NativeWGAN(dict(verbose=False, rank=0, size=1, device="cpu", distill=dist, data_kwargs=dict(n_synthetic=128))),
              LSTM(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, distill=dist,
                        data_kwargs=dict(n_synthetic=96, n_words=200))),
              LSTMTorch(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, distill=dist,
                             data_kwargs=dict(n_synthetic=64, n_words=200)))]
    for m in models:
        with pytest.raises(ValueError, match="distill is not supported"):
            m.compile_iter_fns("avg")


def test_defaults_and_json_round_trip(ckpts):
    assert check_config(dict(teacher=ALEX, checkpoint="c.pt")) == dict(teacher=ALEX, checkpoint="c.pt", alpha=0.5, temperature=1.0,
                                                                      config={})
    cfg = dict(teacher=R152, checkpoint=ckpts["r50"], alpha=0.9, temperature=3, config=dict(blocks=SMALL))
    back = json.loads(json.dumps(dict(distill=cfg)))["distill"]
    assert back["config"]["blocks"] == [1, 1, 1, 1]
    want = dict(cfg, temperature=3.0, config=dict(blocks=SMALL))
    assert check_config(back) == want
    assert check_config(dict(cfg, alpha=np.float32(0.25), temperature=np.int64(2)))["alpha"] == 0.25
    m = _r50(distill=back)
    m.compile_iter_fns("avg")
    d = m.distiller
    assert (d.alpha, d.temperature) == (0.9, 3.0) and type(d.teacher).__name__ == "ResNet152" and d.teacher.blocks == SMALL
    assert d.teacher.arena.allocator is None and d.teacher.use_graph is False


def test_key_off_builds_nothing_and_trains_the_same():
    off = _r50()
    none = _r50(distill=None)
    for m in (off, none):
        m.compile_iter_fns("avg")
        assert m.distiller is None
    rec = _rec()
    for i in range(2):
        step = functional._RNG["step"]
        off.train_iter(i, rec)
        functional._RNG["step"] = step
        none.train_iter(i, rec)
        _assert_equal_lists(_state(off), _state(none), i)
    assert "distill" not in off.extra_state()


def test_checkpoint_carries_no_teacher_and_resume_continues(ckpts, tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    cfg = dict(distill=dict(teacher=R50, checkpoint=ckpts["r50"], config=dict(blocks=SMALL), alpha=0.6, temperature=2.0))
    rec = _rec()
    first = _r50(**cfg)
    first.compile_iter_fns("avg")
    n = first.data.n_batch_train
    for i in range(n):
        first.train_iter(i, rec)
    first.reset_iter("train")
    path = str(tmp_path / "ckpt_1.pt")
    save_checkpoint(first, path)
    sd = torch.load(path, map_location="cpu", weights_only=False)
    assert set(sd["extra_state"]) == {"bn"} and len(sd["extra_state"]["bn"]) == len(first._bn_layers())
    assert sd["arena"]["W"].numel() == first.arena.W.numel()
    plain = _r50()
    assert set(plain.extra_state()) == set(sd["extra_state"])
    step = functional._RNG["step"]
    for i in range(2):
        first.train_iter(i, rec)
    functional._RNG["step"] = step
    resumed = _r50(**cfg)
    resumed.compile_iter_fns("avg")
    load_checkpoint(resumed, path)
    for i in range(2):
        resumed.train_iter(i, rec)
    _assert_equal_lists(_state(resumed), _state(first))


# ------------------------------------------------------------------ BSP on two gloo ranks
def case_bsp(sync, ckpt):
    """Two ranks, BSP over the split 'ar' strategy, each distilling from its own copy of the teacher: the local step equals the manual
    composition before and after the exchange."""
    from mp_cpu_checks import _proc
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    p = _proc()
    dist = dict(teacher=R50, checkpoint=ckpt, config=dict(blocks=SMALL), alpha=0.5, temperature=2.0)
    on = _r50(rank=p.rank, size=p.size, distill=dist)
    on.compile_iter_fns(sync)
    man = _r50(rank=p.rank, size=p.size)
    man.compile_iter_fns(sync)
    t = _load_teacher(man, _builder("r50"), ckpt)
    fn = _manual_step_fn(man, t, 0.5, 2.0)
    if sync == "avg":
        man.train_iter_fn = fn
    else:
        man.forward_backward = fn
    ex_on = BSP_Exchanger(p.comm, None, "ar", sync, p.ctx, on)
    ex_man = BSP_Exchanger(p.comm, None, "ar", sync, p.ctx, man)
    rec = Recorder(p.comm, 1000, "t", False, device="cpu")
    for u in range(3):
        on.train_iter(u, rec)
        man.train_iter(u, rec)
        _assert_equal_lists(_state(on), _state(man), ("local", u))
        ex_on.exchange(rec)
        ex_man.exchange(rec)
        _assert_equal_lists(_state(on), _state(man), ("exchanged", u))
    p.comm.Barrier()
    print("OK distill bsp", sync, "rank", p.rank)


@pytest.mark.parametrize("sync", ["avg", "cdd"])
def test_bsp_two_gloo_ranks(sync, ckpts):
    port = {"avg": "29881", "cdd": "29882"}[sync]
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=port, OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "bsp", sync, ckpts["r50"]],
                              env=dict(env, RANK=str(r), LOCAL_RANK=str(r)), stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(2)]
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=600)[0])
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0, "rank %d failed:\n%s" % (r, o[-3000:])


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
    import torch.distributed as dist
    globals()["case_" + sys.argv[1]](*sys.argv[2:])
    if dist.is_initialized():
        dist.destroy_process_group()
