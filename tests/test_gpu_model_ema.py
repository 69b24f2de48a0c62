"""Model EMA on the H100: ``ema_update`` and ``ema_swap`` bit for bit against ``ops/reference.py`` (partial last blocks, bf16 and
tf32 arenas, d in {0, 0.5, 0.99998, 1}, every mode, batch-norm segments of 64 … 2048 channels, a NaN-fenced skip step), and training
under the CUDA graph with ``TMPI_DETERMINISTIC=1`` (in subprocesses): AlexNet bf16 / tf32, ResNet50 and Wide_ResNet train bit-identically
with and without the key, EMA validation passes included, E equals the reference replayed on the weights of every step, the step has
exactly two more launches, decay 0 validates like the model (one and ten crops), decay 1 keeps the first average, grad_accum averages
once per window, a resumed run continues E and two runs give the same E."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)

from theanompi_b200.ops import reference as ref  # noqa: E402

MODES = {"skip": ref.EMA_SKIP, "copy": ref.EMA_COPY, "average": ref.EMA_AVERAGE}


def _arena(shadow, sizes=(1000, (3, 7, 5), 4097, (64, 33), 1)):
    from theanompi_b200.parallel.arena import FlatArena
    g = torch.Generator().manual_seed(7)
    params = [torch.randn(s if isinstance(s, tuple) else (s,), generator=g) for s in sizes]
    a = FlatArena(params, device="cuda", shadow=shadow)
    assert any(n % 1024 for n in a.sizes)                                 # partial last blocks
    return a


def _table(pairs):
    return torch.tensor([(d.data_ptr(), s.data_ptr(), d.numel()) for d, s in pairs], dtype=torch.int64, device="cuda").view(-1, 3)


def _stats(channels, seed):
    g = torch.Generator().manual_seed(seed)
    return [torch.randn(c, generator=g).cuda() for c in channels for _ in range(2)]


CHANNELS = (64, 128, 256, 512, 1024, 2048, 96)


@pytest.mark.parametrize("shadow", [True, False], ids=["bf16", "tf32"])
@pytest.mark.parametrize("decay", [0.0, 0.5, 0.99998, 1.0])
@pytest.mark.parametrize("mode", list(MODES))
def test_ema_update_matches_reference(shadow, decay, mode):
    from theanompi_b200.ops import cuda_impl
    a = _arena(shadow)
    # E and its statistics part sit inside NaN fences: nothing outside them may change
    fenced = torch.full((a.numel + 2048,), float("nan"), device="cuda")
    E = fenced[1024:-1024]
    E.copy_(torch.randn(a.numel, generator=torch.Generator().manual_seed(3)))
    stats, avg = _stats(CHANNELS, 1), _stats(CHANNELS, 2)
    n_bn = sum(t.numel() for t in avg)
    fenced_bn = torch.full((n_bn + 2048,), float("nan"), device="cuda")
    bn_e = fenced_bn[1024:-1024]
    bn_e.copy_(torch.cat(avg))
    parts, o = [], 0
    for s in stats:
        parts.append(bn_e[o:o + s.numel()]); o += s.numel()
    omd = float(np.float32(1.0 - decay))
    before = [t.clone() for t in (a.W, a.G, a.U, E, bn_e) + tuple(stats)] + ([a.H.clone()] if shadow else [])
    want_e, want_bn = E.clone(), bn_e.clone()
    wparts, o = [], 0
    for s in stats:
        wparts.append(want_bn[o:o + s.numel()]); o += s.numel()
    ref.ema_update([(want_e, a.W)] + list(zip(wparts, stats)), MODES[mode], decay, omd)
    state = torch.tensor([5, 2, MODES[mode]], dtype=torch.int64, device="cuda")
    cuda_impl.ema_update(a, E, state, _table(list(zip(parts, stats))), decay, omd)
    torch.cuda.synchronize()
    assert torch.equal(E, want_e) and torch.equal(bn_e, want_bn)
    after = [a.W, a.G, a.U, E, bn_e] + stats + ([a.H] if shadow else [])
    for i, (x, y) in enumerate(zip(before, after)):
        if i in (3, 4) and mode != "skip":
            continue
        assert torch.equal(x, y), i
    for f in (fenced, fenced_bn):
        assert f[:1024].isnan().all() and f[-1024:].isnan().all()
    assert state.tolist() == [5, 2, MODES[mode]]


def test_ema_advance_matches_reference():
    from theanompi_b200.ops import cuda_impl
    for every, warmup in ((1, 0), (3, 0), (2, 5), (32, 0)):
        state = torch.zeros(3, dtype=torch.int64, device="cuda")
        u, n = 0, 0
        for _ in range(70):
            cuda_impl.ema_advance(state, every, warmup)
            u, n, mode = ref.ema_advance(u, n, every, warmup)
            assert state.tolist() == [u, n, mode], (every, warmup, u)


@pytest.mark.parametrize("shadow", [True, False], ids=["bf16", "tf32"])
def test_ema_swap_twice_is_the_identity(shadow):
    from theanompi_b200.ops import cuda_impl
    a = _arena(shadow)
    if shadow:
        a.refresh_shadow()
    E = torch.randn(a.numel, generator=torch.Generator().manual_seed(5)).cuda()
    stats = _stats(CHANNELS, 1)
    bn_e = torch.cat(_stats(CHANNELS, 2))
    parts, o = [], 0
    for s in stats:
        parts.append(bn_e[o:o + s.numel()]); o += s.numel()
    table = _table(list(zip(parts, stats)))
    w0, e0, bn0, s0 = a.W.clone(), E.clone(), bn_e.clone(), [s.clone() for s in stats]
    h0 = a.H.clone() if shadow else None
    cuda_impl.ema_swap(a, E, table)
    torch.cuda.synchronize()
    assert torch.equal(a.W, e0) and torch.equal(E, w0) and torch.equal(bn_e, torch.cat(s0))
    assert all(torch.equal(s, p) for s, p in zip(stats, torch.split(bn0, [s.numel() for s in stats])))
    if shadow:
        assert torch.equal(a.H, e0.to(torch.bfloat16))
    cuda_impl.ema_swap(a, E, table)
    torch.cuda.synchronize()
    assert torch.equal(a.W, w0) and torch.equal(E, e0) and torch.equal(bn_e, bn0)
    assert all(torch.equal(s, p) for s, p in zip(stats, s0))
    if shadow:
        assert torch.equal(a.H, h0)


# --------------------------------------------------------------------------- models (subprocesses, deterministic mode)
IMNET = dict(n_class=16, data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True))
MODELS = {
    "alexnet_bf16": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=32, file_batch_size=32, no_paraload=True, **IMNET)),
    "alexnet_tf32": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=32, file_batch_size=32, no_paraload=True, dtype="tf32",
                                                                       **IMNET)),
    "resnet50": ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50",
                 dict(batch_size=8, file_batch_size=8, blocks=(1, 1, 1, 1), no_paraload=True, **IMNET)),
    "wrn": ("theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet",
            dict(batch_size=16, file_batch_size=16, depth=10, widen=2, learning_rate=1e-3, data_kwargs=dict(n_synthetic=256, synthetic=True))),
}


def _model(which, **kw):
    import importlib
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import cuda_impl
    mod, cls, cfg = MODELS[which]
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    cuda_impl._STEP.clear()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", **dict(cfg, **kw)))
    m.rand_crop = False
    m.compile_iter_fns("avg")
    return m


def _state(m):
    out = [m.arena.W.clone(), m.arena.U.clone()] + ([m.arena.H.clone()] if m.arena.H is not None else [])
    return out + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)]


def _ema(m):
    return [m.ema.E.clone(), m.ema.E_bn.clone()]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def run(which, n=10, ema=None, val=False, **kw):
    """``n`` training steps under the CUDA graph; with ``val`` an EMA validation pass (and a plain one) after every step.  Returns the
    final state, E, the snapshots of W and the statistics after every step, the validation results and the model."""
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    m = _model(which, model_ema=ema, **kw)
    snaps, vals = [], []
    for i in range(n):
        m.train_iter(i, rec)
        snaps.append([m.arena.W.clone()] + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)])
        if val:
            m.val_iter(i, rec); m.reset_iter("val")
            with m.ema_weights():
                m.val_iter(i, rec); m.reset_iter("val")
            vals.append([float(v) for v in rec.val_info["cost"][-2:]])
    torch.cuda.synchronize()
    return _state(m), (_ema(m) if m.ema is not None else None), snaps, vals, m


def replay(m0_state, snaps, decay, every, warmup=0):
    """The reference average of the per-step snapshots, from the initial weights and statistics ``m0_state``."""
    e = [t.clone() for t in m0_state]
    u = n = 0
    for s in snaps:
        u, n, mode = ref.ema_advance(u, n, every, warmup)
        ref.ema_update(list(zip(e, s)), mode, decay, float(np.float32(1.0 - decay)))
    return [e[0], torch.cat([t.reshape(-1) for t in e[1:]]) if len(e) > 1 else torch.zeros(0, device=e[0].device)]


def model_check(which):
    """Key off vs on (every 3, with EMA validation passes): the same training bit for bit; E against the reference replay; graphs
    captured; two more launches per step."""
    from theanompi_b200.ops import native
    cfg = dict(decay=0.9, every=3)
    off, _, _, _, m_off = run(which)
    m0 = _model(which)
    init = [m0.arena.W.clone()] + [t.clone().cuda() for l in m0._bn_layers() for t in (l.running_mean, l.running_var)]
    on, e, snaps, vals, m_on = run(which, ema=cfg, val=True)
    assert m_on.captured_steps() == {"step"}, m_on.captured_steps()
    assert _same(off, on), "training changed by the key"
    want = replay(init, snaps, 0.9, 3)
    assert _same(e, want), "E differs from the reference replay"
    assert all(np.isfinite(v).all() for v in vals)
    counts = {}
    for key, ema in (("off", None), ("on", cfg)):
        m = _model(which, model_ema=ema, cuda_graph=False)
        from theanompi_b200.utils.recorder import Recorder
        rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
        m.train_iter(0, rec)
        torch.cuda.synchronize()
        native.reset_launch_count()
        m.train_iter(1, rec)
        torch.cuda.synchronize()
        counts[key] = native.launch_count()
    assert counts["on"] == counts["off"] + 2, counts
    return counts


def _subprocess(code, timeout=1200):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("which", list(MODELS))
def test_graph_training_unchanged_and_average_exact(which):
    _subprocess("""
import test_gpu_model_ema as t
print('launches', t.model_check(%r))
print('OK')
""" % which)


def decay_checks():
    """decay 0 validated right after an averaging step validates like the model (1 and 10 crops); decay 1 keeps the first average;
    grad_accum 2 averages once per window; two runs give the same E."""
    for crops in (1, 10):
        _, _, _, vals, _ = run("alexnet_bf16", n=4, ema=dict(decay=0.0, every=2), val=True, val_crops=crops)
        assert vals[1][0] == vals[1][1] and vals[3][0] == vals[3][1], (crops, vals)
    _, e, snaps, _, _ = run("resnet50", n=7, ema=dict(decay=1.0, every=2))
    assert torch.equal(e[0], snaps[1][0]) and torch.equal(e[1], torch.cat([t.reshape(-1) for t in snaps[1][1:]]))
    _, e, snaps, _, m = run("alexnet_bf16", n=6, ema=dict(decay=0.5, every=1), grad_accum=2)
    assert int(m.ema.state[0]) == 3 and m.n_updates == 3
    m0 = _model("alexnet_bf16")
    assert _same(e, replay([m0.arena.W.clone()], snaps[1::2], 0.5, 1))
    _, e2, _, _, _ = run("alexnet_bf16", n=6, ema=dict(decay=0.5, every=1), grad_accum=2)
    assert _same(e, e2), "two deterministic runs differ"


def test_decay_edges_grad_accum_and_determinism():
    _subprocess("""
import test_gpu_model_ema as t
t.decay_checks()
print('OK')
""")


def resume_check(tmp):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    cfg = dict(decay=0.7, every=2)
    a = _model("resnet50", model_ema=cfg)
    n = a.data.n_batch_train
    for i in range(n):
        a.train_iter(i, rec)
    a.reset_iter("train")
    save_checkpoint(a, os.path.join(tmp, "ckpt.pt"))
    for i in range(4):
        a.train_iter(i, rec)
    want = _ema(a) + _state(a)
    b = _model("resnet50", model_ema=cfg)
    load_checkpoint(b, os.path.join(tmp, "ckpt.pt"))
    for i in range(4):
        b.train_iter(i, rec)
    torch.cuda.synchronize()
    assert _same(_ema(b) + _state(b), want), "the resumed average differs"


def test_checkpoint_resume_continues_the_average(tmp_path):
    _subprocess("""
import test_gpu_model_ema as t
t.resume_check(%r)
print('OK')
""" % str(tmp_path))
