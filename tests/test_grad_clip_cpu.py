"""Global gradient-norm clipping on the CPU: the reference norm against a naive fp64 norm, the five clipped flat optimizers against
``torch.nn.utils.clip_grad_norm_`` and ``torch.optim``, the unclipped step below the threshold, skipped steps on a NaN gradient, the
refusals, Cifar10 / LSTM / GAN training with ``grad_clip`` and checkpoint resume."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.parallel.arena import FlatArena  # noqa: E402
from theanompi_b200.utils import opt as O  # noqa: E402

WD = 5e-4
# sizes that are not multiples of the 1024-element arena block: every tensor is followed by padding
SHAPES = [("W", (300, 70)), ("b", (300,)), ("gamma", (96,)), ("W", (64, 3, 3, 16)), ("b", (17,)), ("W", (50, 30))]
RULES = ["sgd", "adam", "rmsprop", "adadelta", "rmsprop_centered"]


def clip_arena(device="cpu", shadow=False, wd=WD, big=False):
    """Weight decay on the weights, bias lr multiplier 1 (so torch.optim param groups can mirror the arena); ``big`` adds AlexNet's
    fc6 (36,864 blocks: more than the kernels' grid)."""
    g = torch.Generator().manual_seed(11)
    params = []
    for name, shape in SHAPES + ([("W", (4096, 9216))] if big else []):
        p = torch.nn.Parameter(torch.randn(*shape, generator=g) * 0.05)
        p.pname = name
        params.append(p)
    wt = ["W" if p.pname == "W" else "b" for p in params]
    return FlatArena(params, wt, device, weight_decay=wd, bias_lr_mult=1.0, shadow=shadow), g


def fill_grad(a, g, scale=1.0, garbage=False):
    """Random gradients on the real elements; the padding holds zeros, or garbage that every norm must ignore."""
    if garbage:
        a.G.copy_(torch.randn(a.G.shape, generator=g) * 1e3)
    else:
        a.G.zero_()
    for v in a.views("G"):
        v.copy_(torch.randn(v.shape, generator=g) * scale)


def make_opt(rule, a):
    return {"sgd": lambda: O.FlatSGD(a, mu=0.9), "adam": lambda: O.FlatAdam(a), "rmsprop": lambda: O.FlatRMSProp(a),
            "adadelta": lambda: O.FlatAdadelta(a), "rmsprop_centered": lambda: O.FlatCenteredRMSProp(a)}[rule]()


def opt_state(opt):
    a = opt.arena
    out = [a.W.clone()] + ([a.U.clone()] if opt.uses_u else []) + [getattr(opt, n).clone() for n in opt.buffers]
    if a.H is not None:
        out.append(a.H.clone())
    if opt.t is not None:
        out.append(opt.t.clone())
    return out


def test_reference_norm_ignores_padding():
    a, g = clip_arena()
    fill_grad(a, g, garbage=True)
    naive = math.sqrt(sum(float((v.double() ** 2).sum()) for v in a.views("G")))
    assert float(a.G.double().norm()) > 10 * naive                      # the padding really holds garbage
    n, s, finite = ref.clip_scale(a.G, a.offsets, a.sizes, 1.0)
    assert finite and n == pytest.approx(naive, rel=1e-12)
    assert s == float(np.float32(1.0 / (naive + 1e-6)))
    n, s, finite = ref.clip_scale(a.G, a.offsets, a.sizes, 10 * naive)
    assert finite and s == 1.0
    a.G[a.offsets[1] + 5] = float("inf")
    assert ref.clip_scale(a.G, a.offsets, a.sizes, 1.0)[1:] == (0.0, False)
    a.G[a.offsets[1] + 5] = float("nan")
    assert ref.clip_scale(a.G, a.offsets, a.sizes, 1.0)[1:] == (0.0, False)


def _torch_twin(rule, a, lr):
    """Copies of the arena's parameters and the matching torch.optim optimizer (None for the centred RMSProp, which has none)."""
    ps = [torch.nn.Parameter(p.detach().clone()) for p in a.params]
    decay = [p for p, grp in zip(ps, a.group_of) if a.group_wd_np[grp] > 0]
    rest = [p for p, grp in zip(ps, a.group_of) if a.group_wd_np[grp] == 0]
    groups = [{"params": decay, "weight_decay": WD}, {"params": rest, "weight_decay": 0.0}]
    mk = {"sgd": lambda: torch.optim.SGD(groups, lr=lr, momentum=0.9),
          "adam": lambda: torch.optim.Adam(groups, lr=lr, betas=(0.9, 0.999), eps=1e-8),
          "rmsprop": lambda: torch.optim.RMSprop(groups, lr=lr, alpha=0.99, eps=1e-8),
          "adadelta": lambda: torch.optim.Adadelta(groups, lr=lr, rho=0.95, eps=1e-6)}
    return ps, (mk[rule]() if rule in mk else None)


@pytest.mark.parametrize("rule", RULES)
def test_clipped_rule_matches_clip_grad_norm_and_torch_optim(rule):
    lr, c = 0.01, 2.0
    a, g = clip_arena()
    opt = make_opt(rule, a)
    opt.set_grad_clip(c)
    a.hyper[0] = lr
    ps, tor = _torch_twin(rule, a, lr)
    if tor is None:                                        # the centred RMSProp: its reference function on torch-clipped gradients
        b, _ = clip_arena()
        twin = O.FlatCenteredRMSProp(b)
        b.hyper[0] = lr
    for step in range(5):
        fill_grad(a, g)
        opt.step()
        assert float(opt.grad_norm) > c and int(opt.skipped) == 0     # the clip is active on every step
        for p, v in zip(ps, a.views("G")):
            p.grad = v.clone()
        total = torch.nn.utils.clip_grad_norm_(ps, c)
        assert float(opt.grad_norm) == pytest.approx(float(total), rel=1e-6)
        if tor is not None:
            tor.step()
        else:
            for v, p in zip(b.views("G"), ps):
                v.copy_(p.grad)
            twin.step()
            for p, w in zip(ps, b.views("W")):
                p.data.copy_(w)
    for w, p in zip(a.views("W"), ps):
        torch.testing.assert_close(w, p.detach(), rtol=2e-5, atol=1e-7)


@pytest.mark.parametrize("rule", RULES)
def test_below_the_threshold_the_step_is_the_unclipped_step(rule):
    (a, g), (b, _) = clip_arena(), clip_arena()
    oa, ob = make_opt(rule, a), make_opt(rule, b)
    oa.set_grad_clip(1e6)
    a.hyper[0] = b.hyper[0] = 0.01
    for _ in range(3):
        fill_grad(a, g)
        b.G.copy_(a.G)
        oa.step()
        ob.step()
        assert float(oa._clip_rec[1]) == 1.0
    for x, y in zip(opt_state(oa), opt_state(ob)):
        assert torch.equal(x, y)


@pytest.mark.parametrize("rule", RULES)
def test_nan_gradient_skips_the_step(rule):
    a, g = clip_arena()
    opt = make_opt(rule, a)
    opt.set_grad_clip(1.0)
    a.hyper[0] = 0.01
    fill_grad(a, g)
    opt.step()
    before = opt_state(opt)
    fill_grad(a, g)
    a.G[a.offsets[3] + 7] = float("nan")
    g0 = a.G.clone()
    opt.step()
    for x, y in zip(opt_state(opt), before):
        assert torch.equal(x, y)
    assert int(opt.skipped) == 1 and math.isnan(float(opt.grad_norm))
    assert torch.equal(a.G.isnan(), g0.isnan()) and torch.equal(a.G.nan_to_num(), g0.nan_to_num())     # G is not modified
    fill_grad(a, g)
    opt.step()                                             # the next finite step updates again
    assert not torch.equal(a.W, before[0]) and int(opt.skipped) == 1
    if opt.t is not None:
        assert int(opt.t) == 2


def test_lars_and_lamb_refuse_clipping():
    a, _ = clip_arena()
    for cls in (O.FlatLARS, O.FlatLAMB):
        with pytest.raises(ValueError, match="sgd, adam, rmsprop"):
            cls(a).set_grad_clip(1.0)
    for name in ("lars", "lamb"):
        m = _cifar(optimizer=name)
        with pytest.raises(ValueError, match="grad_clip does not combine with optimizer='%s'.*sync_type='avg'" % name):
            m.compile_iter_fns("avg")


def test_fused_tail_and_torch_twins_are_refused():
    m = _cifar(size=2)
    with pytest.raises(ValueError, match="fused exchange strategy.*sync_type='avg' with a split strategy"):
        m.compile_iter_fns("avg", fused_tail=lambda: None)
    from theanompi_b200.models.lasagne_model_zoo.wgan import WGAN
    from theanompi_b200.models.lstm import LSTMTorch
    twins = [WGAN(dict(verbose=False, rank=0, size=1, device="cpu", grad_clip=5.0, data_kwargs=dict(n_synthetic=128))),
             LSTMTorch(dict(verbose=False, rank=0, size=1, device="cpu", grad_clip=5.0, dim_proj=16, batch_size=8,
                            data_kwargs=dict(n_synthetic=64, n_words=200)))]
    for t in twins:
        with pytest.raises(ValueError, match="not supported by the torch twins"):
            t.compile_iter_fns("avg")


def test_cdd_with_two_gloo_ranks_is_refused_and_avg_clips(tmp_path):
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT="29837", OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, os.path.join(ROOT, "tests", "mp_grad_clip_checks.py"), "cdd_refused_avg_clips"],
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


def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.01, grad_clip=1.0,
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    return Cifar10_model(cfg)


def test_cifar10_model_learns_with_grad_clip():
    from theanompi_b200.utils.recorder import Recorder
    m = _cifar(batch_size=64, file_batch_size=64, learning_rate=0.05, data_kwargs=dict(n_synthetic=1024, synthetic=True))
    m.compile_iter_fns("avg")
    assert isinstance(m.clip_opt, O.FlatSGD) and m.clip_opt.max_norm == 1.0
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    for i in range(40):
        m.train_iter(i, rec)
    costs = [float(c) for c in rec.train_info["cost"]]
    assert costs[-1] < 1.5 and costs[-1] < costs[0], costs
    assert int(m.clip_opt.skipped) == 0 and math.isfinite(float(m.clip_opt.grad_norm))


@pytest.mark.parametrize("optimizer", ["adadelta", "rmsprop", "sgd"])
def test_lstm_trains_with_grad_clip(optimizer):
    from theanompi_b200.models.lstm import LSTM
    from theanompi_b200.utils.recorder import Recorder
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=32, batch_size=8, optimizer=optimizer, grad_clip=0.05,
               data_kwargs=dict(n_synthetic=64, n_words=200))
    m = LSTM(cfg)
    m.compile_iter_fns("avg")
    assert m.opt.max_norm == 0.05
    rec = Recorder(None, 10 ** 6, "l", False, device="cpu")
    w0 = m.arena.W.clone()
    for i in range(4):
        m.train_iter(i, rec)
    assert all(math.isfinite(float(c)) for c in rec.train_info["cost"])
    assert not torch.equal(w0, m.arena.W)
    assert float(m.opt.grad_norm) > 0.05 and float(m.opt._clip_rec[1]) < 1.0


def test_native_gan_clips_critic_and_generator_separately():
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN
    from theanompi_b200.utils.recorder import Recorder
    m = NativeWGAN(dict(verbose=False, rank=0, size=1, device="cpu", critic_runs=2, grad_clip=5.0, data_kwargs=dict(n_synthetic=128)))
    m.compile_iter_fns("avg")
    rec = Recorder(None, 10 ** 6, "g", False, device="cpu")
    w0, g0 = m.arena.W.clone(), m.gen_arena.W.clone()
    c = 0
    for _ in range(2):
        c = m.train_iter(c, rec)
    assert not torch.equal(w0, m.arena.W) and not torch.equal(g0, m.gen_arena.W)
    assert m.opt_c.max_norm == m.opt_g.max_norm == 5.0
    # each optimizer's norm is the one of its own arena's gradient (the generator's G still holds its last gradient)
    n_g = ref.clip_scale(m.gen_arena.G, m.gen_arena.offsets, m.gen_arena.sizes, 5.0)[0]
    assert float(m.opt_g.grad_norm) == pytest.approx(n_g, rel=1e-6)
    assert int(m.opt_c.skipped) == int(m.opt_g.skipped) == 0
    assert "skipped" in m.extra_state()["rms_c"]


def test_checkpoint_resume_continues_bit_identically(tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    try:
        a = _cifar(grad_clip=0.5)
        a.compile_iter_fns("avg")
        d = a.data
        d.shuffle_data("train", common_seed=0)
        batches = [(torch.from_numpy(np.ascontiguousarray(d.train_img_shuffle[i])), torch.from_numpy(np.asarray(d.train_labels_shuffle[i])))
                   for i in range(6)]

        def steps(m, bs):
            Dropout.SetDropoutOff(); Crop.SetRandCropOff()
            for x, y in bs:
                m.shared_x.copy_(x)
                m.shared_y.copy_(y)
                m.train_iter_fn(0)

        steps(a, batches[:3])
        a.clip_opt.skipped.fill_(2)                        # a counter value the resumed model must carry on from
        f = str(tmp_path / "ck.pt")
        save_checkpoint(a, f)
        steps(a, batches[3:])
        layers2.reseed(999)
        b = _cifar(grad_clip=0.5)
        b.compile_iter_fns("avg")
        load_checkpoint(b, f)
        assert int(b.clip_opt.skipped) == 2
        steps(b, batches[3:])
    finally:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn()
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)
    assert torch.equal(a.clip_opt.grad_norm, b.clip_opt.grad_norm) and int(a.clip_opt.skipped) == int(b.clip_opt.skipped) == 2
