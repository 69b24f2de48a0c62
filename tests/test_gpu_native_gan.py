"""The native GAN models on one H100: the same model on the CPU reference path over the first steps (same weights, batches and
noise), graph vs eager, native launches, and checkpoint resume."""
import pytest
import torch

from theanompi_b200.ops import native, precision

pytestmark = pytest.mark.gpu
ZOO = "theanompi_b200.models.lasagne_model_zoo."
MODELS = [(ZOO + "wgan", "NativeWGAN", dict(critic_runs=2, data_kwargs=dict(n_synthetic=256))),
          (ZOO + "lsgan", "NativeLSGAN", dict(data_kwargs=dict(n_synthetic=256))),
          (ZOO + "lsgan_cifar10", "NativeLSGAN", dict(data_kwargs=dict(n_synthetic=256, synthetic=True)))]


def _make(modelfile, modelclass, cfg, device, dtype, **kw):
    import importlib
    c = dict(verbose=False, rank=0, size=1, device=device, dtype=dtype, **cfg)
    c.update(kw)
    m = getattr(importlib.import_module(modelfile), modelclass)(c)
    m.compile_iter_fns("avg")
    return m


def _steps(m, n):
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "gan", False, device=str(m.device))
    c = 0
    for _ in range(n):
        c = m.train_iter(c, rec)
    return [float(v) for v in rec.train_info["cost"]], [float(v) for v in rec.train_info["error"]]


def _cos(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return float(a @ b / (a.norm() * b.norm() + 1e-30))


@pytest.fixture(autouse=True)
def _restore_precision():
    old = precision.precision()
    yield
    precision.set_precision(old)


@pytest.mark.parametrize("dtype", ["bf16", "tf32"])
@pytest.mark.parametrize("modelfile,modelclass,cfg", MODELS)
def test_native_gan_matches_cpu_reference(modelfile, modelclass, cfg, dtype):
    """Three steps on the GPU (captured graphs) and on the CPU reference ops from the same initial weights, batches and noise:
    the scores agree and the weight updates of both arenas point the same way.  RMSProp's first steps are close to
    lr·sign(g)/sqrt(1 - alpha) for every element, so gradients near zero, whose sign the bf16 / tf32 rounding decides, move by a
    full step in either direction: the update directions are compared by cosine, not elementwise."""
    gm = _make(modelfile, modelclass, cfg, "cuda:0", dtype)
    cm = _make(modelfile, modelclass, cfg, "cpu", dtype)
    assert torch.equal(gm.arena.W.cpu(), cm.arena.W) and torch.equal(gm.gen_arena.W.cpu(), cm.gen_arena.W)
    w0, g0 = cm.arena.W.clone(), cm.gen_arena.W.clone()
    gs, gg = _steps(gm, 3)
    cs, cg = _steps(cm, 3)
    torch.cuda.synchronize()
    tol = 0.1 if dtype == "bf16" else 0.02                   # step k's weights carry k RMSProp-amplified rounding differences
    for seq_g, seq_c in ((gs, cs), (gg, cg)):
        for k, (a, b) in enumerate(zip(seq_g, seq_c)):
            assert abs(a - b) <= tol * (1 + 2 * k) * max(abs(b), 1e-2), (gs, cs, gg, cg)
    cos_min = 0.7 if dtype == "bf16" else 0.85
    assert _cos(gm.arena.W.cpu() - w0, cm.arena.W - w0) > cos_min
    assert _cos(gm.gen_arena.W.cpu() - g0, cm.gen_arena.W - g0) > cos_min


@pytest.mark.parametrize("modelfile,modelclass,cfg", MODELS[:2])
def test_native_gan_graph_and_eager_agree_and_launch_native_kernels(modelfile, modelclass, cfg):
    ms = [_make(modelfile, modelclass, cfg, "cuda:0", "tf32", cuda_graph=g) for g in (False, True)]
    w0 = ms[0].arena.W.clone()
    native.reset_launch_count()
    _steps(ms[0], 1)
    assert native.launch_count() > 20                              # the eager step runs on the native kernels
    _steps(ms[0], 2)
    _steps(ms[1], 3)
    torch.cuda.synchronize()
    assert ms[1].captured_steps() == {"critic", "gen"}
    # bias / BN gradient sums use atomics, whose order differs between runs (see the test above): 0.987 was measured for LSGAN
    assert _cos(ms[0].arena.W - w0, ms[1].arena.W - w0) > 0.95
    assert _cos(ms[0].gen_arena.W, ms[1].gen_arena.W) > 0.9999


def test_native_gan_checkpoint_resume(tmp_path):
    from theanompi_b200.utils.helper_funcs import load_checkpoint, save_model
    modelfile, modelclass, cfg = MODELS[0]
    a = _make(modelfile, modelclass, cfg, "cuda:0", "tf32")
    _steps(a, 2)
    save_model(a, str(tmp_path), False)
    b = _make(modelfile, modelclass, cfg, "cuda:0", "tf32")
    load_checkpoint(b, str(tmp_path / ("ckpt_%d.pt" % a.epoch)))
    for x, y in ((a.arena.W, b.arena.W), (a.opt_c.V, b.opt_c.V), (a.gen_arena.W, b.gen_arena.W), (a.opt_g.V, b.opt_g.V),
                 (a.step, b.step)):
        assert torch.equal(x, y)
    assert b.generator_updates == a.generator_updates
    for m in (a, b):                                              # the same next batches for both, eager
        m._train_gen = m.data.iterate("train", seed=0)
        m.config["critic_runs"] = 1
        m.use_graph = False
    _steps(a, 1)
    _steps(b, 1)
    torch.cuda.synchronize()
    # the bias / batch-norm gradient sums use atomics, so the two continuations differ in the last bits of a few gradients; RMSProp
    # turns a flipped sign of a near-zero gradient into a full step (lr / sqrt(1 - alpha) at most): 99 % of the weights must match
    # to 1e-6 and none may differ by more than two such steps
    d = (b.arena.W - a.arena.W).abs()
    assert float((d > 1e-6).float().mean()) < 1e-2 and float(d.max()) <= 2 * 10 * float(a.shared_lr.get_value()) * 1.01
