"""Sharpness-aware minimization (``config['sam']``) on the CPU reference path: ``reference.sam_*`` against the PyTorch SAM wrapper's
``first_step`` / ``second_step`` (davda54/sam, the version that keeps ``old_p``) over random arenas with padding, the model step against a
manual composition of the model's own pieces (SGD and Adam, with and without grad_clip), frozen running statistics in the second pass,
the same input in both passes, a non-finite norm, the key's refusals, the key off, checkpoint resume, and BSP 'avg' / 'cdd' on two gloo
ranks.

Also the child process of the two-rank test: ``python tests/test_sam_cpu.py bsp <avg|cdd>`` with RANK / WORLD_SIZE set."""
import json
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
from theanompi_b200.ops import functional, reference as ref  # noqa: E402
from theanompi_b200.utils.opt import Sam  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402


def _wrn(rank=0, size=1, **kw):
    """A Wide-ResNet 10-1 (seven batch-norm layers) on 8-image CIFAR batches, trained with momentum SGD."""
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    layers2.reseed()
    cfg = dict(verbose=False, rank=rank, size=size, device="cpu", batch_size=8, file_batch_size=8, depth=10, widen=1, optimizer="sgd",
               learning_rate=0.05, data_kwargs=dict(n_synthetic=64, synthetic=True))
    cfg.update(kw)
    m = Wide_ResNet(cfg)
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    return m


def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.05,
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    return Cifar10_model(cfg)


@pytest.fixture(autouse=True)
def no_dropout():
    yield
    Dropout.SetDropoutOn(); Crop.SetRandCropOn()


def _rec():
    return Recorder(None, 10 ** 6, "c", False, device="cpu")


def _state(m):
    a = m.arena
    out = [a.W.clone(), a.U.clone(), a.G.clone()] + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)]
    adam = getattr(m, "adam", None)
    return out + ([adam.V.clone(), adam.t.clone()] if adam is not None else [])


def _assert_equal_lists(a, b, what=""):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i, float((x.double() - y.double()).abs().max()))


# ------------------------------------------------------------------ the reference functions against the SAM wrapper
class _TorchSam(object):
    """davda54/sam's first_step / second_step over a list of tensors with their gradients (the base optimizer's step left out)."""

    def __init__(self, params, rho, adaptive):
        self.params, self.rho, self.adaptive = params, rho, adaptive
        self.old_p = {}

    def grad_norm(self):
        return torch.norm(torch.stack([((torch.abs(p) if self.adaptive else 1.0) * p.grad).norm(p=2) for p in self.params]), p=2)

    @torch.no_grad()
    def first_step(self, grad_norm=None):
        grad_norm = self.grad_norm() if grad_norm is None else grad_norm
        scale = self.rho / (grad_norm + 1e-12)
        for p in self.params:
            self.old_p[p] = p.data.clone()
            e_w = (torch.pow(p, 2) if self.adaptive else 1.0) * p.grad * scale.to(p)
            p.add_(e_w)

    @torch.no_grad()
    def second_step(self):
        for p in self.params:
            p.data = self.old_p[p]


def _arena(seed, sizes=(1000, (3, 7, 5), 4097, (64, 33), 1, (16, 3, 3, 8))):
    from theanompi_b200.parallel.arena import FlatArena
    g = torch.Generator().manual_seed(seed)
    params = [torch.randn(s if isinstance(s, tuple) else (s,), generator=g) for s in sizes]
    a = FlatArena(params, device="cpu", shadow=True)
    assert any(n % 1024 for n in a.sizes)                                 # padding after partial last blocks
    a.G.copy_(torch.randn(a.numel, generator=g) * 1e-2)
    pad = torch.ones(a.numel, dtype=torch.bool)
    for o, s in zip(a.offsets, a.sizes):
        pad[o:o + s] = False
    a.W[pad] = 3.0                                                        # padding that a perturbation would move
    a.G[pad] = 5.0
    a.refresh_shadow()
    return a, pad


@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("rho", [0.01, 0.05, 0.5, 2.0])
@pytest.mark.parametrize("seed", [0, 1])
def test_reference_matches_the_sam_wrapper(adaptive, rho, seed):
    a, pad = _arena(seed)
    views = [a.W[o:o + s].clone() for o, s in zip(a.offsets, a.sizes)]
    for v, o, s in zip(views, a.offsets, a.sizes):
        v.grad = a.G[o:o + s].clone()
    tsam = _TorchSam(views, rho, adaptive)
    tn = tsam.grad_norm()
    n = ref.sam_norm(a.W, a.G, a.offsets, a.sizes, adaptive)
    # the fp64 sum of the reference against torch's fp32 per-tensor norms: both within a few fp32 ulps of the exact norm
    assert abs(float(n) - float(tn)) <= 4e-6 * float(tn), (float(n), float(tn))
    s, finite = ref.sam_scale(n, rho)
    assert finite and s == float(np.float32(rho) * (1.0 / (np.float32(n) + np.float32(1e-12))))
    w0, h0 = a.W.clone(), a.H.clone()
    P = torch.full_like(a.W, float("nan"))
    ref.sam_perturb(a.W, a.G, P, s, finite, a.offsets, a.sizes, adaptive, w_half=a.H)
    tsam.first_step(grad_norm=torch.tensor(float(n), dtype=torch.float32))        # the same norm: bit-identical perturbed weights
    for v, o, sz in zip(views, a.offsets, a.sizes):
        assert torch.equal(a.W[o:o + sz], v), (o, sz)
    assert torch.equal(P, w0)
    assert torch.equal(a.W[pad], w0[pad]), "the padding moved"
    assert torch.equal(a.H, a.W.to(torch.bfloat16)) and not torch.equal(a.H, h0)
    ref.sam_restore(a.W, P, w_half=a.H)
    tsam.second_step()
    assert torch.equal(a.W, w0) and torch.equal(a.H, h0)
    for v, o, sz in zip(views, a.offsets, a.sizes):
        assert torch.equal(a.W[o:o + sz], v)


def test_reference_non_finite_norm_leaves_the_weights():
    a, _ = _arena(3)
    a.G[7] = float("nan")
    n = ref.sam_norm(a.W, a.G, a.offsets, a.sizes)
    s, finite = ref.sam_scale(n, 0.05)
    assert not np.isfinite(n) and not finite and s == 0.0
    w0, h0 = a.W.clone(), a.H.clone()
    P = torch.zeros_like(a.W)
    ref.sam_perturb(a.W, a.G, P, s, finite, a.offsets, a.sizes, w_half=a.H)
    assert torch.equal(a.W, w0) and torch.equal(P, w0) and torch.equal(a.H, h0)


# ------------------------------------------------------------------ the model step against a manual composition
def _manual_step_fn(m, rho, adaptive):
    """The train_iter_fn of a model built without the key that does, from the model's own pieces: pass 1 (draws, forward, backward),
    the reference perturbation, pass 2 with running statistics frozen, the restore and the step tail."""
    a = m.arena

    def step(subb=0):
        B = m.batch_size
        m.x_in.copy_(m.shared_x[subb * B:(subb + 1) * B])
        m.y_in.copy_(m.shared_y[subb * B:(subb + 1) * B])
        m.n_updates += 1
        m._schedule_lr()
        out = m._fwd_bwd_eager()
        n = ref.sam_norm(a.W, a.G, a.offsets, a.sizes, adaptive)
        s, finite = ref.sam_scale(n, rho)
        P = torch.empty_like(a.W)
        ref.sam_perturb(a.W, a.G, P, s, finite, a.offsets, a.sizes, adaptive, w_half=a.H)
        with m.bn_stats_frozen():
            m._train_pass(None)
        ref.sam_restore(a.W, P, w_half=a.H)
        with torch.no_grad():
            m._tail()
        m._after_step()
        return out
    return step


@pytest.mark.parametrize("opt", ["sgd", "adam"])
@pytest.mark.parametrize("clip", [None, 0.5])
@pytest.mark.parametrize("adaptive", [False, True])
def test_model_step_equals_manual_composition(opt, clip, adaptive):
    rho = 0.5 if adaptive else 0.05
    kw = dict(optimizer=opt, grad_clip=clip, learning_rate=0.05 if opt == "sgd" else 1e-3)
    on = _wrn(sam=dict(rho=rho, adaptive=adaptive), **kw)
    on.compile_iter_fns("avg")
    man = _wrn(**kw)
    man.compile_iter_fns("avg")
    man.train_iter_fn = _manual_step_fn(man, rho, adaptive)
    rec = _rec()
    for i in range(4):
        on.train_iter(i, rec)
        man.train_iter(i, rec)
        _assert_equal_lists(_state(on), _state(man), (opt, clip, adaptive, i))
        assert np.isfinite(float(on.sam_norm)) and float(on.sam_norm) > 0
    assert on.sam_opt.rho == rho and on.sam_opt.adaptive is adaptive


def test_running_statistics_are_those_of_pass_one():
    on, plain = _wrn(sam=dict(rho=0.1)), _wrn()
    for m in (on, plain):
        m.compile_iter_fns("avg")
    B = plain.batch_size

    def pass_one(subb=0):                                       # pass 1 alone
        plain.x_in.copy_(plain.shared_x[:B]); plain.y_in.copy_(plain.shared_y[:B])
        return plain._fwd_bwd_eager()
    plain.train_iter_fn = pass_one
    on.train_iter(0, _rec())
    plain.train_iter(0, _rec())
    stats = lambda m: [t for l in m._bn_layers() for t in (l.running_mean, l.running_var)]  # noqa: E731
    _assert_equal_lists(stats(on), stats(plain))
    assert not torch.equal(stats(on)[0], torch.zeros_like(stats(on)[0]))
    assert all(l.update_stats for l in on._bn_layers())


def test_both_passes_see_the_same_input():
    m = _wrn(sam=dict(rho=0.05), mixup=dict(alpha=0.8, cutmix_alpha=1.0), cifar_augment=dict(pad=4, cutout=8),
             drop_path_rate=0.2)
    m.compile_iter_fns("avg")
    seen, rows = [], []
    fwd, drop_row = m.stem.forward, m.drop_row
    m.stem.forward = lambda x: (seen.append(x.clone()), fwd(x))[1]
    m.drop_row = lambda l: (rows.append(drop_row(l)), rows[-1])[1]
    rec = _rec()
    for i in range(3):
        del seen[:], rows[:]
        m.train_iter(i, rec)
        assert len(seen) == 2 and torch.equal(seen[0], seen[1]), i
        half = len(rows) // 2
        assert len(rows) == 2 * len(m.body) and any(r is not None for r in rows)
        assert all((x is None and y is None) or torch.equal(x, y) for x, y in zip(rows[:half], rows[half:]))
        assert not torch.equal(seen[0], ((m.x_in.float() - m._mean) / 64.0))      # augmented and mixed


@pytest.mark.parametrize("model", ["wrn", "wrn_cifar_augment"])
def test_the_mix_is_applied_once_per_pass(model):
    """Without cifar_augment x_in is mixed in place once (a second mix would mix the mixed batch); with it the record is handed to the
    second forward again."""
    extra = dict(cifar_augment=dict(pad=4, cutout=0)) if model == "wrn_cifar_augment" else {}
    m = _wrn(sam=dict(rho=0.05), mixup=dict(alpha=1.0), **extra)
    m.compile_iter_fns("avg")
    seen = []
    fwd = m.stem.forward
    m.stem.forward = lambda x: (seen.append(x.clone()), fwd(x))[1]
    step = functional._RNG["step"]                              # the CPU draws' step counter: the plain model draws the same step
    m.train_iter(0, _rec())
    functional._RNG["step"] = step
    plain = _wrn(mixup=dict(alpha=1.0), **extra)
    plain.compile_iter_fns("avg")
    first = []
    fwd2 = plain.stem.forward
    plain.stem.forward = lambda x: (first.append(x.clone()), fwd2(x))[1]
    plain.train_iter(0, _rec())
    assert torch.equal(seen[0], first[0]) and torch.equal(seen[1], first[0])


def test_non_finite_norm_runs_pass_two_at_w():
    m = _wrn(sam=dict(rho=0.05))
    m.compile_iter_fns("avg")
    passes = []
    train_pass = m._train_pass

    def poisoned(rec):
        if not passes:
            out = train_pass(rec)
            m.arena.G[5] = float("nan")
        else:
            passes.append(m.arena.W.clone())
            out = train_pass(rec)
        passes.append(None)
        return out
    m._train_pass = poisoned
    w0 = m.arena.W.clone()
    m.train_iter(0, _rec())
    assert torch.equal(passes[1], w0), "the weights were perturbed by a NaN norm"
    assert not np.isfinite(float(m.sam_norm)) and int(m.sam_opt.rec[2:3].view(torch.int32)) == 0


# ------------------------------------------------------------------ the key
@pytest.mark.parametrize("bad", [
    [0.05], "on", True, 0.05, dict(rho=0.05, foo=1), dict(rho=True), dict(rho=float("nan")), dict(rho=float("inf")), dict(rho=0.0),
    dict(rho=-0.1), dict(rho="0.05"), dict(rho=None), dict(adaptive=1), dict(adaptive="yes"), dict(adaptive=None)])
def test_malformed_values_are_refused(bad):
    with pytest.raises(ValueError, match="sam"):
        Sam.check_config(bad)
    m = _wrn(sam=bad)
    with pytest.raises(ValueError, match="sam"):
        m.compile_iter_fns("avg")


def test_defaults_and_json_round_trip():
    assert Sam.check_config({}) == dict(rho=0.05, adaptive=False)
    cfg = dict(rho=1.5, adaptive=True)
    back = json.loads(json.dumps(dict(sam=cfg)))["sam"]
    assert Sam.check_config(back) == cfg
    assert Sam.check_config(dict(rho=np.float32(0.25), adaptive=np.bool_(False))) == dict(rho=0.25, adaptive=False)
    m = _wrn(sam=back)
    m.compile_iter_fns("avg")
    assert (m.sam_opt.rho, m.sam_opt.adaptive) == (1.5, True) and m.sam_opt.P.shape == m.arena.W.shape


def test_unsupported_models_and_options_are_refused():
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.lasagne_model_zoo.lsgan import NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.wgan import WGAN, NativeWGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    from theanompi_b200.models.torch_base import TorchModelBase
    for cls in (AlexNet_sc, Cifar10_model, NativeWGAN, NativeLSGAN, WGAN, LSTM, LSTMTorch, TorchModelBase):
        assert cls.supports_sam is False, cls
    sam = dict(rho=0.05)
    models = [_cifar(sam=sam),
              NativeWGAN(dict(verbose=False, rank=0, size=1, device="cpu", sam=sam, data_kwargs=dict(n_synthetic=128))),
              LSTM(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, sam=sam,
                        data_kwargs=dict(n_synthetic=96, n_words=200))),
              LSTMTorch(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, sam=sam,
                             data_kwargs=dict(n_synthetic=64, n_words=200)))]
    for m in models:
        with pytest.raises(ValueError, match="sam is not supported"):
            m.compile_iter_fns("avg")
    m = _wrn(sam=sam, grad_accum=2, batch_size=4)
    with pytest.raises(ValueError, match="sam does not combine with grad_accum = 2"):
        m.compile_iter_fns("avg")
    for opt in ("sgd", "adam"):
        m = _wrn(rank=0, size=2, sam=sam, optimizer=opt)
        with pytest.raises(ValueError, match="sam does not combine with a fused exchange"):
            m.compile_iter_fns("cdd" if opt == "sgd" else "avg", fused_tail=lambda: None)


def test_key_off_builds_nothing_and_trains_the_same():
    off, none = _wrn(), _wrn(sam=None)
    calls = []
    for m in (off, none):
        m.compile_iter_fns("avg")
        assert m.sam_opt is None and m.sam_norm is None
        tp = m._train_pass
        m._train_pass = lambda rec, tp=tp: (calls.append(1), tp(rec))[1]
    rec = _rec()
    for i in range(3):
        off.train_iter(i, rec)
        none.train_iter(i, rec)
        _assert_equal_lists(_state(off), _state(none), i)
    assert len(calls) == 6                                      # one training pass per step
    assert "sam" not in off.extra_state()


def test_checkpoint_resume_continues_bit_identically(tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    cfg = dict(optimizer="adam", learning_rate=1e-3, sam=dict(rho=0.5, adaptive=True))
    rec = _rec()
    first = _wrn(**cfg)
    first.compile_iter_fns("avg")
    n = first.data.n_batch_train
    for i in range(n):
        first.train_iter(i, rec)
    first.reset_iter("train")
    save_checkpoint(first, str(tmp_path / "ckpt.pt"))
    for i in range(3):
        first.train_iter(i, rec)
    resumed = _wrn(**cfg)
    resumed.compile_iter_fns("avg")
    load_checkpoint(resumed, str(tmp_path / "ckpt.pt"))
    for i in range(3):
        resumed.train_iter(i, rec)
    _assert_equal_lists(_state(resumed), _state(first))


# ------------------------------------------------------------------ BSP on two gloo ranks
def _manual_fb(m, rho):
    """forward_backward of the manual composition for BSP 'cdd', where the step has no tail: get_vel runs pre() after it."""
    a = m.arena

    def fb(subb=0):
        B = m.batch_size
        m.x_in.copy_(m.shared_x[subb * B:(subb + 1) * B])
        m.y_in.copy_(m.shared_y[subb * B:(subb + 1) * B])
        m.n_updates += 1
        out = m._fwd_bwd_eager()
        n = ref.sam_norm(a.W, a.G, a.offsets, a.sizes)
        s, finite = ref.sam_scale(n, rho)
        P = torch.empty_like(a.W)
        ref.sam_perturb(a.W, a.G, P, s, finite, a.offsets, a.sizes, w_half=a.H)
        with m.bn_stats_frozen():
            m._train_pass(None)
        ref.sam_restore(a.W, P, w_half=a.H)
        m._after_step()
        return out
    return fb


def case_bsp(sync):
    """Two ranks, BSP over the split 'ar' strategy, each rank perturbing by its own gradient.  'avg': every rank's local SAM step equals
    its manual composition before the weights are averaged.  'cdd': G after get_vel is the rank's pass-2 gradient, the send buffers
    are built from it, the exchanged sum R is the sum of both ranks' sends, and the weights after post() equal the composition's."""
    from mp_cpu_checks import _proc
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    p = _proc()
    on = _wrn(rank=p.rank, size=p.size, sam=dict(rho=0.05))
    man = _wrn(rank=p.rank, size=p.size)
    on.compile_iter_fns(sync)
    man.compile_iter_fns(sync)
    if sync == "avg":
        man.train_iter_fn = _manual_step_fn(man, 0.05, False)
    else:
        man.forward_backward = _manual_fb(man, 0.05)
    ex_on = BSP_Exchanger(p.comm, None, "ar", sync, p.ctx, on)
    ex_man = BSP_Exchanger(p.comm, None, "ar", sync, p.ctx, man)
    rec = Recorder(p.comm, 1000, "t", False, device="cpu")
    for u in range(3):
        on.train_iter(u, rec)
        man.train_iter(u, rec)
        _assert_equal_lists(_state(on), _state(man), ("local", u))
        if sync == "cdd":
            sends = [torch.cat([v.reshape(-1) for v in m.vels]).clone() for m in (on, man)]
            assert torch.equal(sends[0], sends[1]), u
            both = p.comm.allgather(sends[1])
        ex_on.exchange(rec)
        ex_man.exchange(rec)
        _assert_equal_lists(_state(on), _state(man), ("exchanged", u))
        if sync == "cdd":
            got = torch.cat([v.reshape(-1) for v in on.vels2])
            assert torch.allclose(got, both[0] + both[1], rtol=0, atol=1e-6), u
    p.comm.Barrier()
    print("OK sam bsp", sync, "rank", p.rank)


@pytest.mark.parametrize("sync", ["avg", "cdd"])
def test_bsp_two_gloo_ranks(sync):
    port = {"avg": "29871", "cdd": "29872"}[sync]
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT=port, OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "bsp", sync], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)),
                              stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
             for r in range(2)]
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=300)[0])
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
