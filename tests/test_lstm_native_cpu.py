"""The LSTM's flat optimizers (Adadelta, the reference's centred RMSProp) and the native LSTM model on the CPU reference path:
optimizer math against torch / a per-tensor transcription, state round trips, bucket padding, checkpoint resume and the three
optimizers of ``config['optimizer']``."""
import math

import numpy as np
import pytest
import torch

from theanompi_b200 import ops
from theanompi_b200.parallel.arena import FlatArena
from theanompi_b200.utils.opt import FlatAdadelta, FlatCenteredRMSProp

SMALL = dict(dim_proj=32, batch_size=8, data_kwargs=dict(n_synthetic=64, n_words=200))


def _tensors(seed=0):
    g = torch.Generator().manual_seed(seed)
    # sizes that are not multiples of the arena block, so every tensor is followed by padding
    shapes = [(40, 33), (40,), (7, 9, 5), (3,), (1500,)]
    ts = [torch.randn(*s, generator=g) * 0.1 for s in shapes]
    return ts, ["W" if t.dim() > 1 else "b" for t in ts]


def _arena_and_copies(bias_lr_mult=2.0):
    ts, types = _tensors()
    copies = [t.clone() for t in ts]
    a = FlatArena(ts, types, "cpu", bias_lr_mult=bias_lr_mult, shadow=False)
    return a, copies, types


def _grads(a, k):
    g = torch.Generator().manual_seed(100 + k)
    return [torch.randn(p.shape, generator=g) for p in a.params]


def _set_grads(a, grads):
    a.G.zero_()
    for gb, gr in zip(a.views("G"), grads):
        gb.copy_(gr)


def test_flat_adadelta_matches_torch_adadelta():
    a, copies, types = _arena_and_copies(bias_lr_mult=2.0)
    a.hyper[0] = 1.0
    opt = FlatAdadelta(a)
    ps = [c.requires_grad_(True) for c in copies]
    tor = torch.optim.Adadelta([{"params": [p for p, t in zip(ps, types) if t == "W"], "lr": 1.0},
                                {"params": [p for p, t in zip(ps, types) if t == "b"], "lr": 2.0}], rho=0.95, eps=1e-6)
    for k in range(10):
        grads = _grads(a, k)
        _set_grads(a, grads)
        opt.step()
        for p, gr in zip(ps, grads):
            p.grad = gr.clone()
        tor.step()
    for w, p in zip(a.params, ps):
        torch.testing.assert_close(w.detach(), p.detach(), rtol=1e-6, atol=1e-9)
    for u, v, p in zip(a.views("U"), [opt.V[o:o + s].view(p.shape) for o, s, p in zip(a.offsets, a.sizes, a.params)], ps):
        st = tor.state[p]
        torch.testing.assert_close(u, st["acc_delta"], rtol=1e-6, atol=1e-12)
        torch.testing.assert_close(v, st["square_avg"], rtol=1e-6, atol=1e-12)
    assert float(a.W[a.offsets[1] + a.sizes[1]:a.offsets[2]].abs().max()) == 0.0      # padding is never touched by the grads


def test_flat_centered_rmsprop_matches_transcription():
    """Per-tensor transcription of the reference LSTM's rmsprop (``updir_new`` / ``param_up``), fp64, element by element."""
    a, copies, types = _arena_and_copies(bias_lr_mult=2.0)
    lr = 1e-4
    a.hyper[0] = lr
    opt = FlatCenteredRMSProp(a)
    state = [dict(w=c.double().clone(), r=torch.zeros_like(c, dtype=torch.float64), s=torch.zeros_like(c, dtype=torch.float64),
                  m=torch.zeros_like(c, dtype=torch.float64)) for c in copies]
    for k in range(10):
        grads = _grads(a, k)
        _set_grads(a, grads)
        opt.step()
        for st, gr, t in zip(state, grads, types):
            g = gr.double()
            st["r"] = 0.95 * st["r"] + 0.05 * g
            st["s"] = 0.95 * st["s"] + 0.05 * g ** 2
            st["m"] = 0.9 * st["m"] - lr * (2.0 if t == "b" else 1.0) * g / torch.sqrt(st["s"] - st["r"] ** 2 + 1e-4)
            st["w"] = st["w"] + st["m"]
    for w, u, st in zip(a.params, a.views("U"), state):
        torch.testing.assert_close(w.detach().double(), st["w"], rtol=1e-5, atol=1e-7)
        torch.testing.assert_close(u.double(), st["m"], rtol=1e-4, atol=1e-9)


@pytest.mark.parametrize("cls,keys", [(FlatAdadelta, ["V"]), (FlatCenteredRMSProp, ["R", "S"])])
def test_flat_optimizer_state_dict_round_trip(cls, keys):
    a, _, _ = _arena_and_copies()
    a.hyper[0] = 1e-3
    opt = cls(a)
    for k in range(3):
        _set_grads(a, _grads(a, k))
        opt.step()
    sd = opt.state_dict()
    assert sorted(sd) == sorted(keys)
    b, _, _ = _arena_and_copies()
    opt2 = cls(b)
    opt2.load_state_dict(sd)
    for k in keys:
        assert torch.equal(getattr(opt2, k), getattr(opt, k)) and getattr(opt, k).abs().sum() > 0


def _lstm(**kw):
    from theanompi_b200.models import layers2
    from theanompi_b200.models.lstm import LSTM
    layers2.reseed(); layers2.Dropout.layers.clear()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", **SMALL)
    cfg.update(kw)
    m = LSTM(cfg)
    m.compile_iter_fns("avg")
    return m


def _loss_and_grad(m, x, mk, y):
    m.arena.G.zero_()
    c, _, _ = ops.softmax_xent(m.forward_logits(torch.from_numpy(x), torch.from_numpy(mk)), torch.from_numpy(y))
    c.backward()
    return float(c.detach()), m.arena.G.clone()


def test_bucket_padding_leaves_loss_and_gradients_unchanged():
    from theanompi_b200.models.lstm import bucket_len, pad_batch
    assert [bucket_len(t, 500) for t in (1, 16, 17, 79, 499, 500)] == [16, 16, 32, 80, 512, 512]
    with pytest.raises(ValueError):
        bucket_len(513, 500)
    m = _lstm()
    m.training = False                                    # dropout off: the eval-mode scaling is deterministic
    x, mk, y = next(m.data.batches("train", m.batch_size, False))
    T = x.shape[1]
    Tb = bucket_len(T, m.data.maxlen)
    assert Tb > T
    xp, mp = pad_batch(x, mk, Tb)
    assert xp.shape == (m.batch_size, Tb) and not xp[:, T:].any() and not mp[:, T:].any()
    l0, g0 = _loss_and_grad(m, x, mk, y)
    l1, g1 = _loss_and_grad(m, xp, mp, y)
    assert abs(l1 - l0) <= 1e-6 * abs(l0), (l0, l1)
    torch.testing.assert_close(g1, g0, rtol=1e-5, atol=1e-5 * float(g0.abs().max()))


def _fixed_batch_step(m, batch, rng_step):
    from theanompi_b200.utils.recorder import Recorder
    m._train_it = iter([batch])
    ops.rng_state()["step"] = rng_step
    rec = Recorder(None, 10 ** 6, "LSTM", False, device="cpu")
    m.train_iter(0, rec)
    return float(rec.train_info["cost"][0])


@pytest.mark.parametrize("opt", ["adadelta", "rmsprop"])
def test_checkpoint_resume_restores_optimizer_and_early_stopping(opt, tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    from theanompi_b200.utils.recorder import Recorder
    a = _lstm(optimizer=opt)
    rec = Recorder(None, 10 ** 6, "LSTM", False, device="cpu")
    for i in range(3):
        a.train_iter(i, rec)
    a.val_iter(3, rec)
    a.bad_counter = 4
    f = str(tmp_path / "ck.pt")
    save_checkpoint(a, f)
    b = _lstm(optimizer=opt)
    load_checkpoint(b, f)
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)
    for k, v in a.opt.state_dict().items():
        assert torch.equal(v, b.opt.state_dict()[k])
    assert (b.best_err, b.bad_counter) == (a.best_err, a.bad_counter) and a.best_err < 1.0
    batch = next(a.data.batches("train", a.batch_size, True, seed=77))
    rng = ops.rng_state()["step"]
    ca, cb = _fixed_batch_step(a, batch, rng), _fixed_batch_step(b, batch, rng)
    assert ca == cb
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)
    # a checkpoint of another optimizer is refused
    c = _lstm(optimizer="sgd")
    with pytest.raises(ValueError, match="optimizer"):
        load_checkpoint(c, f)


@pytest.mark.parametrize("opt,lr", [("adadelta", 1.0), ("rmsprop", 1e-4), ("sgd", 1e-4)])
def test_each_optimizer_trains_and_validates_on_the_reference_path(opt, lr):
    from theanompi_b200.utils.recorder import Recorder
    m = _lstm(optimizer=opt)
    assert m.shared_lr.get_value() == pytest.approx(lr) and float(m.arena.hyper[0]) == pytest.approx(lr)
    rec = Recorder(None, 10 ** 6, "LSTM", False, device="cpu")
    w0 = m.arena.W.clone()
    for i in range(3):
        m.train_iter(i, rec)
    assert m.val_iter(3, rec) == m.data.n_batch_val
    assert all(math.isfinite(float(v)) for v in rec.train_info["cost"] + rec.val_info["cost"])
    assert not torch.equal(w0, m.arena.W)
    assert _lstm(optimizer=opt, learning_rate=0.5).shared_lr.get_value() == 0.5
    with pytest.raises(ValueError):
        _lstm(optimizer="adam")


def test_synthetic_corpus_lengths():
    from theanompi_b200.models.lstm import IMDB_Data
    d = IMDB_Data(n_synthetic=64, seq_len=(100, 500))
    lens = [len(s) for s in d.train[0] + d.valid[0]]
    assert min(lens) >= 100 and max(lens) < 500 and max(lens) > 300
    d0, d1 = IMDB_Data(n_synthetic=64), IMDB_Data(n_synthetic=64, seq_len=(20, 80))        # the default is unchanged
    assert all(np.array_equal(p, q) for p, q in zip(d0.train[0], d1.train[0]))
    assert all(20 <= len(s) < 80 for s in d0.train[0])
