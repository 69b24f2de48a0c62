"""Model EMA (``config['model_ema']``) on the CPU reference path: the key's refusals, the average against torch's
``AveragedModel(avg_fn=d·e + (1 − d)·w, use_buffers=True)`` fed the model's weights and batch-norm statistics after every update (with
``every``, ``warmup``, ``grad_accum``, a dropped window and a skipped clipped step), ``ema_weights()``, training unchanged by the key,
checkpoint resume, the recorder's EMA channel, and BSP ``sync_type='cdd'`` on two gloo ranks.

Also the child process of the two-rank test: ``python tests/test_model_ema_cpu.py bsp_cdd`` with RANK / WORLD_SIZE set."""
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
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.utils.opt import ModelEma  # noqa: E402
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


def _snapshot(m):
    """The model's weights and batch-norm statistics, in ModelEma's order."""
    return [m.arena.W.clone()] + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)]


class _Oracle(object):
    """torch's AveragedModel over a module holding the arena's W and every statistics tensor as buffers, fed the model's values after
    every update; torchvision's warm-up resets n_averaged, so the average copies."""

    def __init__(self, m, decay, every, warmup):
        from torch.optim.swa_utils import AveragedModel
        self.net = torch.nn.Module()
        self.net.w = torch.nn.Parameter(torch.zeros(0))
        self.every, self.warmup = every, warmup
        self._load(m)
        self.avg = AveragedModel(self.net, avg_fn=lambda e, w, n: decay * e + (1 - decay) * w, use_buffers=True)
        self.u = 0

    def _load(self, m):
        snap = _snapshot(m)
        self.net.w = torch.nn.Parameter(snap[0])
        for i, t in enumerate(snap[1:]):
            self.net.register_buffer("s%d" % i, t)

    def update(self, m):
        self.u += 1
        if self.u % self.every:
            return
        self._load(m)
        if self.u <= self.warmup:
            self.avg.n_averaged.fill_(0)
        self.avg.update_parameters(self.net)

    def values(self):
        return [self.avg.module.w.detach()] + [getattr(self.avg.module, "s%d" % i) for i in range(len(list(self.net.buffers())))]


def _ema_values(m):
    e, o, out = m.ema, 0, [m.ema.E]
    for n in e.sizes:
        out.append(e.E_bn[o:o + n])
        o += n
    return out


def _assert_equal_lists(a, b, what=""):
    assert len(a) == len(b)
    for i, (x, y) in enumerate(zip(a, b)):
        assert torch.equal(x, y), (what, i, float((x - y).abs().max()))


# ------------------------------------------------------------------ the key
@pytest.mark.parametrize("bad", [
    [0.9], "on", True, dict(decay=0.9, foo=1), dict(decay=True), dict(decay=float("nan")), dict(decay=float("inf")), dict(decay=-0.1),
    dict(decay=1.5), dict(decay="0.9"), dict(decay=None), dict(every=0), dict(every=2.0), dict(every=True), dict(every="2"),
    dict(warmup=-1), dict(warmup=1.5), dict(warmup=False)])
def test_malformed_values_are_refused(bad):
    with pytest.raises(ValueError, match="model_ema"):
        ModelEma.check_config(bad)
    m = _cifar(model_ema=bad)
    with pytest.raises(ValueError, match="model_ema"):
        m.compile_iter_fns("avg")


def test_defaults_and_json_round_trip():
    assert ModelEma.check_config({}) == dict(decay=0.9999, every=1, warmup=0)
    cfg = dict(decay=0.99998, every=32, warmup=0)
    back = json.loads(json.dumps(dict(model_ema=cfg)))["model_ema"]
    assert ModelEma.check_config(back) == cfg
    assert ModelEma.check_config(dict(decay=1, every=np.int64(3))) == dict(decay=1.0, every=3, warmup=0)
    m = _cifar(model_ema=back)
    m.compile_iter_fns("avg")
    assert (m.ema.decay, m.ema.every, m.ema.warmup) == (0.99998, 32, 0)
    assert m.ema.one_minus_decay == float(np.float32(1.0 - 0.99998))


def test_unsupported_models_and_rules_are_refused():
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.lasagne_model_zoo.lsgan import NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.wgan import WGAN, NativeWGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    from theanompi_b200.models.torch_base import TorchModelBase
    for cls in (AlexNet_sc, NativeWGAN, NativeLSGAN, WGAN, LSTM, LSTMTorch, TorchModelBase):
        assert cls.supports_model_ema is False, cls
    ema = dict(decay=0.9)
    models = [NativeWGAN(dict(verbose=False, rank=0, size=1, device="cpu", model_ema=ema, data_kwargs=dict(n_synthetic=128))),
              LSTM(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, model_ema=ema,
                        data_kwargs=dict(n_synthetic=96, n_words=200))),
              LSTMTorch(dict(verbose=False, rank=0, size=1, device="cpu", dim_proj=16, batch_size=8, model_ema=ema,
                             data_kwargs=dict(n_synthetic=64, n_words=200)))]
    for m in models:
        with pytest.raises(ValueError, match="model_ema is not supported"):
            m.compile_iter_fns("avg")
    # two workers: BSP 'avg' (and EASGD / ASGD / GOSGD, which compile with 'avg'), a fused strategy, Wide_ResNet's Adam
    for kw, sync, fused, match in ((dict(), "avg", None, "change in the exchange"), (dict(), "cdd", lambda: None, "fused exchange"),
                                   (dict(optimizer="adam"), "avg", None, "change in the exchange")):
        m = _wrn(rank=0, size=2, model_ema=ema, **kw)
        with pytest.raises(ValueError, match="model_ema"):
            m.compile_iter_fns(sync, fused_tail=fused)
        with pytest.raises(ValueError, match=match):
            m.compile_iter_fns(sync, fused_tail=fused)


def test_key_off_builds_nothing():
    m = _cifar()
    m.compile_iter_fns("avg")
    assert m.ema is None and "model_ema" not in m.extra_state()
    with pytest.raises(RuntimeError, match="model_ema"):
        with m.ema_weights():
            pass


# ------------------------------------------------------------------ the average against AveragedModel
@pytest.mark.parametrize("decay,every,warmup", [(0.0, 1, 0), (0.5, 1, 0), (0.9999, 1, 0), (1.0, 1, 0), (0.0, 3, 0), (0.5, 3, 0),
                                                (0.9999, 3, 0), (1.0, 3, 0), (0.5, 1, 4), (0.9999, 3, 4)])
def test_average_equals_averaged_model(decay, every, warmup):
    m = _wrn(model_ema=dict(decay=decay, every=every, warmup=warmup))
    m.compile_iter_fns("avg")
    oracle = _Oracle(m, decay, every, warmup)
    _assert_equal_lists(_ema_values(m), oracle.values(), "initial")
    rec = _rec()
    for i in range(7):
        m.train_iter(i, rec)
        oracle.update(m)
        _assert_equal_lists(_ema_values(m), oracle.values(), (decay, every, warmup, i))
    assert int(m.ema.state[0]) == 7 and m.ema.n_averaged == int(oracle.avg.n_averaged)


@pytest.mark.parametrize("n", [2, 3])
def test_grad_accum_windows_count_once_and_dropped_window_not(n):
    m = _wrn(batch_size=4, model_ema=dict(decay=0.5, every=1), grad_accum=n)
    m.compile_iter_fns("avg")
    oracle = _Oracle(m, 0.5, 1, 0)
    rec = _rec()
    for i in range(2 * n + 1):                  # two windows and one micro-step of a third
        m.train_iter(i, rec)
        if m.micro_step_kind() == "first" and m.n_updates > oracle.u:
            oracle.update(m)
    assert m.n_updates == 2 and int(m.ema.state[0]) == 2
    m.reset_iter("train")                       # the open window is dropped: it does not count
    for i in range(n):
        m.train_iter(i, rec)
    oracle.update(m)
    assert int(m.ema.state[0]) == 3
    _assert_equal_lists(_ema_values(m), oracle.values())


def test_skipped_clipped_step_counts_and_averages_unchanged_weights():
    m = _wrn(model_ema=dict(decay=0.5, every=1), grad_clip=1.0)
    m.compile_iter_fns("avg")
    oracle = _Oracle(m, 0.5, 1, 0)
    fwd = m._fwd_bwd_eager
    calls = []

    def poisoned():
        out = fwd()
        calls.append(1)
        if len(calls) == 3:
            m.arena.G[5] = float("nan")         # a non-finite gradient norm: the third step is skipped
        return out
    m._fwd_bwd_eager = poisoned
    rec = _rec()
    for i in range(5):
        w = m.arena.W.clone()
        m.train_iter(i, rec)
        assert torch.equal(w, m.arena.W) == (i == 2)
        oracle.update(m)
        _assert_equal_lists(_ema_values(m), oracle.values(), i)
    assert int(m.clip_opt.skipped) == 1 and int(m.ema.state[0]) == 5 and m.ema.n_averaged == 5


# ------------------------------------------------------------------ ema_weights, unchanged training, checkpoints
def test_ema_weights_round_trip_and_training_unchanged():
    plain, ema = _wrn(), _wrn(model_ema=dict(decay=0.5, every=2))
    for m in (plain, ema):
        m.compile_iter_fns("avg")
    rec = _rec()
    for i in range(5):
        plain.train_iter(i, rec)
        ema.train_iter(i, rec)
        before, avg = _snapshot(ema), [t.clone() for t in _ema_values(ema)]
        with ema.ema_weights():
            _assert_equal_lists(_snapshot(ema), avg, "inside")
            _assert_equal_lists(_ema_values(ema), before, "E holds the model")
            ema.val_iter(i, rec)
        ema.reset_iter("val")
        _assert_equal_lists(_snapshot(ema), before, "restored")
        _assert_equal_lists(_snapshot(ema), _snapshot(plain), "training changed by the key")
        assert torch.equal(ema.arena.U, plain.arena.U)


def test_ema_weights_keeps_the_bf16_shadow():
    m = _wrn(model_ema=dict(decay=0.5), _arena_shadow=True)
    m.compile_iter_fns("avg")
    m.ema.E.mul_(0.75)                          # an average that differs from W (the CPU path does not train on the shadow)
    h, e = m.arena.H.clone(), m.ema.E.clone()
    assert torch.equal(h, m.arena.W.to(torch.bfloat16))
    with m.ema_weights():
        assert torch.equal(m.arena.W, e) and torch.equal(m.arena.H, e.to(torch.bfloat16))
    assert torch.equal(m.arena.H, h)


def test_checkpoint_resume_continues_the_average(tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    cfg = dict(decay=0.5, every=2, warmup=1)
    rec = _rec()
    straight = _wrn(model_ema=cfg)
    straight.compile_iter_fns("avg")
    n = straight.data.n_batch_train                             # checkpoint at the end of the first epoch
    for i in range(n):
        straight.train_iter(i, rec)
    straight.reset_iter("train")
    for i in range(4):
        straight.train_iter(i, rec)

    first = _wrn(model_ema=cfg)
    first.compile_iter_fns("avg")
    for i in range(n):
        first.train_iter(i, rec)
    first.reset_iter("train")
    save_checkpoint(first, str(tmp_path / "ckpt.pt"))
    resumed = _wrn(model_ema=cfg)
    resumed.compile_iter_fns("avg")
    load_checkpoint(resumed, str(tmp_path / "ckpt.pt"))
    assert int(resumed.ema.state[0]) == n and resumed.ema.n_averaged == n // 2
    for i in range(4):
        resumed.train_iter(i, rec)
    _assert_equal_lists(_ema_values(resumed), _ema_values(straight))
    _assert_equal_lists(_snapshot(resumed), _snapshot(straight))


def test_recorder_ema_channel_saved_loaded_and_cut(tmp_path):
    r = _rec()
    r.val_error(4, 0.3, 0.2, 0.1)
    r.gather_val_info(); r.print_val_info(4)
    assert "val_info_ema" not in r.info_dict                   # no EMA pass: no channel
    for count, c in ((8, 0.5), (12, 0.4)):
        r.val_error(count, c, 0.2, 0.1)
        with r.ema_channel():
            r.val_error(count, c - 0.1, 0.1, 0.05)
        r.gather_val_info(); r.print_val_info(count)
    assert [v[1] for v in r.info_dict["val_info"]] == [0.3, 0.5, 0.4]
    assert r.info_dict["val_info_ema"] == [[8, 0.4, 0.1, 0.05], [12, pytest.approx(0.3), 0.1, 0.05]]
    r.save(12, 0.1, filepath=str(tmp_path))
    back = _rec()
    back.load(str(tmp_path / "inforec.pkl"))
    assert back.info_dict["val_info_ema"] == r.info_dict["val_info_ema"]
    back.cut(1)
    assert len(back.info_dict["val_info"]) == 1 and len(back.info_dict["val_info_ema"]) == 1


# ------------------------------------------------------------------ BSP 'cdd' on two gloo ranks
def case_bsp_cdd():
    """Two ranks, BSP ``sync_type='cdd'`` over the split 'ar' strategy: after every exchange E equals the reference average replayed on
    this rank's W and statistics, and the average of the exchanged weights is the same on both ranks."""
    from mp_cpu_checks import _proc
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    p = _proc()
    m = _wrn(rank=p.rank, size=p.size, model_ema=dict(decay=0.5, every=2, warmup=2))
    m.compile_iter_fns("cdd")
    ex = BSP_Exchanger(p.comm, None, "ar", "cdd", p.ctx, m)
    want = [t.clone() for t in _ema_values(m)]
    n_av, rec = 0, Recorder(p.comm, 1000, "t", False, device="cpu")
    for u in range(1, 8):
        m.train_iter(u, rec)
        ex.exchange(rec)
        _, n_av, mode = ref.ema_advance(u - 1, n_av, 2, 2)
        ref.ema_update(list(zip(want, _snapshot(m))), mode, 0.5, float(np.float32(1.0 - 0.5)))
        _assert_equal_lists(_ema_values(m), want, u)
    assert int(m.ema.state[0]) == 7 and m.ema.n_averaged == n_av == 3
    # the exchanged weights are the same on both ranks after post(), and so is their average; batch-norm gamma / beta and the running
    # statistics stay local to each rank (they are never exchanged), and so does their average, checked above against the reference
    ex = m.arena.exch_vector()
    ws, es = p.comm.allgather(m.arena.W[ex].clone()), p.comm.allgather(m.ema.E[ex].clone())
    assert torch.equal(ws[0], ws[1]) and torch.equal(es[0], es[1]), "the averages of the two ranks differ"
    p.comm.Barrier()
    print("OK model ema rank", p.rank)


def test_bsp_cdd_two_gloo_ranks():
    env = dict(os.environ, WORLD_SIZE="2", MASTER_ADDR="127.0.0.1", MASTER_PORT="29863", OMP_NUM_THREADS="2", PYTHONPATH=ROOT)
    procs = [subprocess.Popen([sys.executable, os.path.abspath(__file__), "bsp_cdd"], env=dict(env, RANK=str(r), LOCAL_RANK=str(r)),
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
    globals()["case_" + sys.argv[1]]()
    if dist.is_initialized():
        dist.destroy_process_group()
