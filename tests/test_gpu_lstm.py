"""The native LSTM on one H100, in both precision modes: the flat Adadelta / centred-RMSProp kernels against the CPU reference, the
bucketed step graphs against the eager step, the model against the CPU reference path, one launch per optimizer step, checkpoint
resume, and learning on the separable synthetic corpus."""
import pytest
import torch

from theanompi_b200.ops import native, precision
from theanompi_b200.ops import reference as ref
from theanompi_b200.parallel.arena import FlatArena
from theanompi_b200.utils.opt import FlatAdadelta, FlatCenteredRMSProp

pytestmark = pytest.mark.gpu
DEV = "cuda"
# batch lengths of the graph / eager comparison: buckets 32, 48 and 64 four times each, so each bucket is captured and replayed
LENGTHS = [20, 40, 60, 18, 35, 50, 30, 47, 64, 25, 33, 55]


@pytest.fixture(autouse=True)
def _restore_precision():
    old = precision.precision()
    yield
    precision.set_precision(old)


def _make(dtype, **kw):
    from theanompi_b200.models import layers2
    from theanompi_b200.models.lstm import LSTM
    layers2.reseed(); layers2.Dropout.layers.clear()
    cfg = dict(verbose=False, rank=0, size=1, device="cuda:0", dtype=dtype, dim_proj=64,
               data_kwargs=dict(n_synthetic=256, n_words=500))
    cfg.update(kw)
    m = LSTM(cfg)
    m.compile_iter_fns("avg")
    return m


def _steps(m, n):
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "LSTM", False, device=str(m.device))
    for i in range(n):
        m.train_iter(i, rec)
    return [float(v) for v in rec.train_info["cost"]]


def _reset_dropout_step():
    from theanompi_b200.ops import cuda_impl
    cuda_impl._STEP.clear()


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float(a @ b / (a.norm() * b.norm() + 1e-30))


def _arena(shadow):
    g = torch.Generator(device=DEV).manual_seed(3)
    ps = [torch.randn(512, 128, device=DEV, generator=g) * 0.1, torch.randn(512, device=DEV, generator=g) * 0.1,
          torch.randn(10000, 128, device=DEV, generator=g) * 0.01, torch.randn(2, 128, device=DEV, generator=g) * 0.01,
          torch.randn(2, device=DEV, generator=g) * 0.01]
    return FlatArena(ps, device=DEV, weight_decay=1e-3, bias_lr_mult=2.0, shadow=shadow)


@pytest.mark.parametrize("mode", ["bf16", "tf32"])
@pytest.mark.parametrize("kind", ["adadelta", "rmsprop"])
def test_flat_kernels_match_cpu_reference(kind, mode):
    """Eight steps of the native kernel against ``ops.reference`` on the CPU, with weight decay and a bias lr multiplier; in bf16
    the shadow written in the same pass is the rounded master, in tf32 there is none."""
    precision.set_precision(mode)
    a = _arena(shadow=(mode == "bf16"))
    lr = 1.0 if kind == "adadelta" else 1e-4
    a.hyper[0] = lr
    opt = FlatAdadelta(a) if kind == "adadelta" else FlatCenteredRMSProp(a)
    w, u = a.W.cpu().clone(), torch.zeros(a.numel)
    bufs = [torch.zeros(a.numel) for _ in range(1 if kind == "adadelta" else 2)]
    lrm, wd = a.lr_mult_vector().cpu(), a.wd_vector().cpu()
    g = torch.Generator(device=DEV).manual_seed(7)
    for _ in range(8):
        gr = torch.randn(a.numel, device=DEV, generator=g) * 0.05
        a.G.copy_(gr)
        opt.step()
        if kind == "adadelta":
            ref.adadelta_flat(w, gr.cpu(), u, bufs[0], lrm, wd, lr)
        else:
            ref.rmsprop_centered_flat(w, gr.cpu(), u, bufs[0], bufs[1], lrm, wd, lr)
    torch.cuda.synchronize()
    torch.testing.assert_close(a.W.cpu(), w, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(a.U.cpu(), u, rtol=1e-4, atol=1e-8)
    got = [opt.V] if kind == "adadelta" else [opt.R, opt.S]
    for x, y in zip(got, bufs):               # (the gradient average r cancels to values far below its scale)
        torch.testing.assert_close(x.cpu(), y, rtol=1e-4, atol=1e-6 * float(y.abs().max()))
    if mode == "bf16":
        torch.testing.assert_close(a.H.float(), a.W, rtol=2 ** -8, atol=0)
    else:
        assert a.H is None


@pytest.mark.parametrize("opt", ["adadelta", "rmsprop", "sgd"])
def test_optimizer_step_is_one_native_launch(opt):
    m = _make("tf32", optimizer=opt, cuda_graph=False)
    native.reset_launch_count()
    _steps(m, 1)
    torch.cuda.synchronize()
    assert native.launch_count() > 100                     # the eager step runs on the native kernels
    native.reset_launch_count()
    with torch.no_grad():
        m.opt.step(m.shared_lr.get_value()) if opt == "sgd" else m.opt.step()
    torch.cuda.synchronize()
    assert native.launch_count() == 1


@pytest.mark.parametrize("dtype", ["bf16", "tf32"])
def test_bucket_graphs_and_eager_agree(dtype):
    """12 steps over batches of three length buckets: eager on the unpadded batches vs one graph per bucket on the padded ones.
    The padded steps are no-ops, so the two differ only by summation order (GEMM shapes that depend on T, atomics)."""
    runs = []
    for graph in (False, True):
        _reset_dropout_step()                               # the same dropout masks in both runs
        m = _make(dtype, cuda_graph=graph)
        it = m.data.batches("train", m.batch_size, True, seed=0)
        batches = []
        for T in LENGTHS:                                   # the synthetic batches are longer than 64: cut them to T steps
            x, mk, y = next(it)
            batches.append((x[:, :T].copy(), mk[:, :T].copy(), y))
        m._train_it = iter(batches)
        w0 = m.arena.W.clone()
        runs.append((m, _steps(m, len(LENGTHS)), w0))
    torch.cuda.synchronize()
    (me, ce, w0), (mg, cg, _) = runs
    captured = sorted(mg.captured_steps())
    assert captured == [32, 48, 64] and not me._graphs
    tol = 0.02 if dtype == "bf16" else 0.005
    assert max(abs(a - b) for a, b in zip(ce, cg)) < tol, (ce, cg)
    assert _cos(me.arena.W - w0, mg.arena.W - w0) > 0.98
    if dtype == "bf16":
        assert torch.equal(mg.arena.H.float(), mg.arena.W.to(torch.bfloat16).float())      # the update refreshed the shadow


@pytest.mark.parametrize("dtype", ["bf16", "tf32"])
def test_native_lstm_matches_cpu_reference(dtype, monkeypatch):
    """Three steps of the native model (bucket graphs) and of the same model on the fp32 reference ops (CPU), same weights and
    batches; dropout is taken out because the two paths draw different masks."""
    from theanompi_b200 import ops
    from theanompi_b200.models import layers2
    from theanompi_b200.models.lstm import LSTM
    monkeypatch.setattr(ops, "dropout", lambda x, p_drop, training, layer_id=0: x)
    ms, costs = {}, {}
    for dev in ("cpu", "cuda:0"):
        layers2.reseed()
        ms[dev] = LSTM(dict(verbose=False, rank=0, size=1, device=dev, dtype=dtype, dim_proj=64, data_kwargs=dict(n_synthetic=256, n_words=500)))
        ms[dev].compile_iter_fns("avg")
    w0 = ms["cpu"].arena.W.clone()
    assert torch.equal(ms["cuda:0"].arena.W.cpu(), w0)
    for dev, m in ms.items():
        costs[dev] = _steps(m, 3)
    torch.cuda.synchronize()
    tol = 0.02 if dtype == "bf16" else 0.005
    for a, b in zip(costs["cpu"], costs["cuda:0"]):
        assert abs(a - b) < tol * max(1.0, abs(a)), costs
    cos = _cos(ms["cuda:0"].arena.W.cpu() - w0, ms["cpu"].arena.W - w0)
    assert cos > (0.9 if dtype == "bf16" else 0.95), cos


def test_checkpoint_resume_on_gpu(tmp_path):
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_checkpoint
    a = _make("tf32", optimizer="rmsprop")
    _steps(a, 4)
    a.best_err, a.bad_counter = 0.375, 2
    f = str(tmp_path / "ck.pt")
    save_checkpoint(a, f)
    b = _make("tf32", optimizer="rmsprop")
    load_checkpoint(b, f)
    for x, y in ((a.arena.W, b.arena.W), (a.arena.U, b.arena.U), (a.opt.R, b.opt.R), (a.opt.S, b.opt.S)):
        assert torch.equal(x, y)
    assert (b.best_err, b.bad_counter) == (0.375, 2)
    batch = next(a.data.batches("train", a.batch_size, True, seed=5))
    step = cuda_impl.step_counter(a.device)
    k = int(step)
    for m in (a, b):                                          # the same next batch and dropout step for both, eager
        m.use_graph = False
        m._train_it = iter([batch])
        step.fill_(k)
        _steps(m, 1)
    torch.cuda.synchronize()
    # the embedding gradient is a scatter-add with atomics, so the two continuations may differ in the last bits
    assert float((a.arena.W - b.arena.W).abs().max()) < 1e-5
    assert float((a.opt.S - b.opt.S).abs().max()) <= 1e-6 * float(a.opt.S.abs().max())


def test_adadelta_lowers_the_loss_on_the_separable_corpus():
    """The synthetic corpus marks 30 % of the tokens by class.  On the CPU reference path, same configuration, the mean loss of
    50 steps stays at 0.69 up to step 300, falls to 0.25 over steps 400-449 and to 0.0035 over steps 550-599.  The threshold leaves
    room for the onset to come about 100 steps later."""
    _reset_dropout_step()
    m = _make("bf16", data_kwargs=dict(n_synthetic=512, n_words=500))
    c = _steps(m, 600)
    first, last = sum(c[:50]) / 50, sum(c[-50:]) / 50
    assert first > 0.68 and last < 0.1, (first, last)
