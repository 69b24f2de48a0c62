"""Knowledge distillation on the H100.  Kernel: ``softmax_xent_kd`` against the fp64 reference (``reference.softmax_xent_kd`` on the same
dtype-rounded logits), bf16 and fp32, over (B, C) from (8, 16) to (256, 1000), α ∈ {0.3, 1}, T ∈ {1, 2, 4}, ε ∈ {0, 0.1}, no mix / a Mixup /
a CutMix record, with logits up to ±60, per-row loss, per-element dlogits and exact err1 / err5.  Models (in subprocesses,
``TMPI_DETERMINISTIC=1``): AlexNet bf16 and tf32 distilling from an AlexNet, ResNet50 from a ResNet50; the captured step replays bit for
bit like the eager one and like a manual composition, the teacher stays bit-identical, and the launches per step are the student's plus the
teacher's eval forward.  ResNet50 with mixup and SAM runs one teacher forward per step."""
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

from theanompi_b200.ops import mixup, reference as ref  # noqa: E402

# The kernel's fp32 error relative to the exact value of each exponential term and sum: __expf of an argument |x| ≤ 120 loses about
# |x|·log2(e)·2^-24 ≈ 1e-5 to the rounding of x·log2(e) plus 2 ulp; the row sums (4 strided terms per thread, a 5-level warp tree, 8
# warps) add at most about 17·2^-24 ≈ 1e-6.  DELTA = 1e-4 covers both with a margin of about 10.
DELTA = 1e-4


def _record(mode, lam):
    r = np.zeros((), dtype=mixup.RECORD)
    r["mode"], r["lam"], r["lam_raw"], r["H"], r["W"] = mode, lam, lam, 8, 8
    return mixup.encode(r)


MIXES = {"none": None, "mixup": (mixup.MIX_MIXUP, 0.3), "cutmix": (mixup.MIX_CUTMIX, 0.625)}


def _logits(B, C, seed):
    """Student and teacher logits up to ±60: a wide normal spread, clamped; row 0 has t = z, row 1 a shifted copy of z."""
    g = torch.Generator().manual_seed(seed)
    z = (torch.randn(B, C, generator=g) * 15).clamp(-60, 60)
    t = (torch.randn(B, C, generator=g) * 15).clamp(-60, 60)
    t[0] = z[0]
    t[1] = (z[1] + 7.0).clamp(-60, 60)
    z[2 % B] = z[2 % B].round()                                 # ties between logits: the rank rule decides
    return z, t


def _launch(z, t, y, rec, alpha, T, eps, grad_scale=1.0):
    """One softmax_xent_kd launch with a rowstat buffer of our own, so that the per-row losses and errors can be read."""
    from theanompi_b200.ops import native
    B, C = z.shape
    dl = torch.empty_like(z)
    rowstat = torch.empty((B, 3), dtype=torch.float32, device=z.device)
    out3 = torch.empty(3, dtype=torch.float32, device=z.device)
    native.require().softmax_xent_kd(z.data_ptr(), t.data_ptr(), y.data_ptr(), 0 if rec is None else rec.data_ptr(), dl.data_ptr(),
                                     rowstat.data_ptr(), out3.data_ptr(), B, C, float(grad_scale), float(eps), float(alpha), float(T),
                                     int(z.dtype == torch.float32), torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return rowstat.cpu(), out3.cpu(), dl.float().cpu()


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("B,C", [(8, 16), (64, 10), (32, 1000), (128, 1000), (256, 1000)])
def test_kernel_matches_fp64_reference(B, C, dtype):
    z0, t0 = _logits(B, C, B * 7 + C)
    zd, td = z0.to(dtype).cuda(), t0.to(dtype).cuda()
    z, t = zd.double().cpu(), td.double().cpu()               # the values the kernel reads
    y = torch.randint(0, C, (B,), generator=torch.Generator().manual_seed(C)).cuda()
    yc = y.cpu()
    out_rel = 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -23   # rounding of dlogits to the output dtype (nearest: half an ulp)
    for mix, spec in MIXES.items():
        rec = None if spec is None else _record(*spec)
        lam = 1.0 if rec is None else ref.mix_lambda(rec)
        for alpha in (0.3, 1.0):
            for T in (1.0, 2.0, 4.0):
                for eps in (0.0, 0.1):
                    what = (mix, alpha, T, eps)
                    rowstat, out3, dl = _launch(zd, td, y, None if rec is None else rec.cuda(), alpha, T, eps)
                    loss, _, _, d = ref.softmax_xent_kd(z, yc, t, alpha, T, label_smoothing=eps, mix=rec)
                    # per-row loss in fp64, and the bound on each row's error: δ on log se, on on·|z_i − m| and on·|z_j − m|, off·Σ|z − m|;
                    # on the KL term δ·(Σ p_t·|(t − m_t) − (z − m)| / T + 2) (its sum and the two logarithms), times α·T²
                    C_ = z.shape[1]
                    m, mt = z.max(1, keepdim=True).values, t.max(1, keepdim=True).values
                    v, u = z - m, t - mt
                    pt = torch.softmax(t / T, 1)
                    q = (1 - eps) * torch.nn.functional.one_hot(yc, C_).double() + eps / C_
                    if lam != 1.0:
                        q = lam * q + (1 - lam) * ((1 - eps) * torch.nn.functional.one_hot(yc.flip(0), C_).double() + eps / C_)
                    lsm = torch.log_softmax(z, 1)
                    kl = (pt * (torch.log_softmax(t / T, 1) - torch.log_softmax(z / T, 1))).sum(1)
                    rows = (1 - alpha) * -(q * lsm).sum(1) + alpha * T * T * kl
                    yj = yc.flip(0) if lam != 1.0 else yc
                    tol = DELTA * ((1 - alpha) * (1 + v.gather(1, yc[:, None])[:, 0].abs() + v.gather(1, yj[:, None])[:, 0].abs()
                                                  + eps / C_ * v.abs().sum(1))
                                   + alpha * T * T * ((pt * (u - v).abs()).sum(1) / T + 2))
                    err = (rowstat[:, 0].double() - rows).abs()
                    assert bool((err <= tol).all()), (what, float((err / tol).max()))
                    assert abs(float(out3[0]) - float(loss)) <= float(tol.mean()) + 1e-6 * abs(float(loss)), what
                    # per-element dlogits: δ on each term of (1 − α)·(p + q) + α·T·(softmax(z/T) + p_t), then the output rounding
                    p, ps = torch.softmax(z, 1), torch.softmax(z / T, 1)
                    bound = (DELTA * ((1 - alpha) * (p + q) + alpha * T * (ps + pt)) / B + out_rel * d.abs() + 1e-30)
                    derr = (dl.double() - d).abs()
                    assert bool((derr <= bound).all()), (what, float((derr / bound).max()))
                    # the errors: exact, by the rank rule on the values the kernel read
                    lab = yc if lam >= 0.5 else yc.flip(0)
                    zl = z.gather(1, lab[:, None])
                    cols = torch.arange(C_)[None, :]
                    rank = ((z > zl) | ((z == zl) & (cols < lab[:, None]))).sum(1)
                    assert torch.equal(rowstat[:, 1], (rank >= 1).float()) and torch.equal(rowstat[:, 2], (rank >= 5).float()), what


def test_self_distillation_at_alpha_one():
    """α = 1 and t = z: the loss and gradient are 0 up to the kernel's error on the KL term (the bounds of the test above at KL = 0)."""
    z0, _ = _logits(64, 1000, 3)
    z = z0.to(torch.bfloat16).cuda()
    y = torch.randint(0, 1000, (64,)).cuda()
    zc = z.double().cpu()
    for T in (1.0, 2.0, 4.0):
        rowstat, out3, dl = _launch(z, z.clone(), y, None, 1.0, T, 0.1)
        assert float(rowstat[:, 0].abs().max()) <= DELTA * 2 * T * T, T
        ps = torch.softmax(zc / T, 1)
        assert bool((dl.double().abs() <= DELTA * T * 2 * ps / 64 + 1e-30).all()), T


# --------------------------------------------------------------------------- models (subprocesses, deterministic mode)
IMNET = dict(n_class=16, no_paraload=True, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
MODELS = {
    "alexnet_bf16": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, **IMNET)),
    "alexnet_tf32": ("theanompi_b200.models.alex_net", "AlexNet", dict(batch_size=128, file_batch_size=128, dtype="tf32", **IMNET)),
    "resnet50": ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50", dict(batch_size=64, file_batch_size=64, **IMNET)),
}


def _clear():
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import cuda_impl
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    cuda_impl._STEP.clear()


def _model(which, compile=True, **kw):
    import importlib
    mod, cls, cfg = MODELS[which]
    _clear()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", **dict(cfg, **kw)))
    m.rand_crop = False
    if compile:
        m.compile_iter_fns("avg")
    return m


def _rec():
    from theanompi_b200.utils.recorder import Recorder
    return Recorder(None, 10 ** 6, "t", False, device="cuda:0")


def teacher_checkpoint(which, path):
    """A checkpoint of a trained teacher: two steps of the model (eager), so that its momentum and statistics are not the initial ones."""
    from theanompi_b200.utils.helper_funcs import save_checkpoint
    m = _model(which, cuda_graph=False, learning_rate=0.005)
    rec = _rec()
    for i in range(2):
        m.train_iter(i, rec)
    torch.cuda.synchronize()
    save_checkpoint(m, path)
    m.cleanup()
    del m
    torch.cuda.empty_cache()
    return path


def _state(m):
    out = [m.arena.W.clone(), m.arena.U.clone(), m.arena.G.clone()] + ([m.arena.H.clone()] if m.arena.H is not None else [])
    return out + [t.clone() for l in m._bn_layers() for t in (l.running_mean, l.running_var)]


def _same(a, b):
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _load_teacher(which, path, batch_size):
    """The teacher built and loaded by hand, after the student, its layers out of the class lists, in eval mode."""
    import importlib
    from theanompi_b200.models import layers2
    from theanompi_b200.utils.helper_funcs import load_checkpoint
    mod, cls, cfg = MODELS[which]
    n_d, n_b = len(layers2.Dropout.layers), len(layers2.BatchNormal.layers)
    rng = layers2.rng
    t = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", cuda_graph=False,
                                                        **dict(cfg, batch_size=batch_size, file_batch_size=batch_size)))
    layers2.rng = rng
    del layers2.Dropout.layers[n_d:], layers2.BatchNormal.layers[n_b:]
    load_checkpoint(t, path)
    for l in t.layers:
        if isinstance(l, layers2.Dropout):
            l.flag_on = False
        if isinstance(l, layers2.BatchNormal):
            l.training = False
    return t


def _manual(m, teacher, alpha, T):
    """A train_iter_fn for a student built without the key: the teacher's eval forward on x_in, the student's forward, one
    cuda_impl.softmax_xent_kd launch, the backward of its dlogits and the step tail, as separate pieces."""
    from theanompi_b200.ops import cuda_impl

    def step(subb=0):
        B = m.batch_size
        m.x_in.copy_(m.shared_x[subb * B:(subb + 1) * B])
        m.y_in.copy_(m.shared_y[subb * B:(subb + 1) * B])
        m.n_updates += 1
        with torch.no_grad():
            t = teacher.forward(m.x_in)
        z = m.forward(m.x_in)
        loss, err, _, d = cuda_impl.softmax_xent_kd(z, m.y_in, t, alpha, T, label_smoothing=m.label_smoothing)
        z.backward(d)
        with torch.no_grad():
            m._tail()
        m._after_step()
        return loss, err
    return step


def _run(which, n, dist, manual=False, **kw):
    rec = _rec()
    if manual:
        m = _model(which, **kw)
        t = _load_teacher(dist["teacher_model"], dist["checkpoint"], m.batch_size)
        m.train_iter_fn = _manual(m, t, dist["alpha"], dist["temperature"])
    else:
        key = {k: v for k, v in dist.items() if k != "teacher_model"}
        m = _model(which, distill=key, **kw)
    states = []
    for i in range(n):
        m.train_iter(i, rec)
        torch.cuda.synchronize()
        states.append(_state(m))
    return states, m


def model_check(which, teacher, path, n=4):
    """The captured distillation step replays bit for bit like the eager one and like the manual composition; the teacher is unchanged;
    the launches per step are the key-off step's plus the teacher's eval forward."""
    from theanompi_b200.ops import native
    mod, cls, _ = MODELS[teacher]
    dist = dict(teacher="%s:%s" % (mod, cls), checkpoint=path, alpha=0.5, temperature=2.0, teacher_model=teacher)
    graph, m = _run(which, n, dist)
    assert m.captured_steps() == {"step"}
    t = m.distiller.teacher
    sd = torch.load(path, map_location="cpu", weights_only=False)
    assert torch.equal(t.arena.W.cpu(), sd["arena"]["W"]) and torch.equal(t.arena.U.cpu(), sd["arena"]["U"])
    if t.arena.H is not None:
        assert torch.equal(t.arena.H, t.arena.W.to(torch.bfloat16))
    for l, (mu, var) in zip(t._bn_layers(), sd["extra_state"]["bn"]):
        assert torch.equal(l.running_mean.cpu(), mu) and torch.equal(l.running_var.cpu(), var)
    del m, t
    eager, _ = _run(which, n, dist, cuda_graph=False)
    man, _ = _run(which, n, dist, manual=True, cuda_graph=False)
    for i in range(n):
        assert _same(graph[i], eager[i]), ("graph replay != eager", i)
        assert _same(graph[i], man[i]), ("step != manual composition", i)
    counts = {}
    rec = _rec()
    for key, kw in (("off", {}), ("on", dict(distill={k: v for k, v in dist.items() if k != "teacher_model"}))):
        m = _model(which, cuda_graph=False, **kw)
        m.train_iter(0, rec)
        torch.cuda.synchronize()
        native.reset_launch_count()
        m.train_iter(1, rec)
        torch.cuda.synchronize()
        counts[key] = native.launch_count()
        if key == "on":
            native.reset_launch_count()
            m.distiller.target(m.x_in)
            torch.cuda.synchronize()
            counts["teacher"] = native.launch_count()
        del m
    assert counts["on"] == counts["off"] + counts["teacher"], counts
    return counts


def sam_check(path):
    """ResNet50 with mixup and SAM: one teacher forward per step, on the mixed batch, its logits used by both passes."""
    mod, cls, _ = MODELS["resnet50"]
    dist = dict(teacher="%s:%s" % (mod, cls), checkpoint=path, alpha=0.5, temperature=2.0)
    m = _model("resnet50", distill=dist, mixup=dict(alpha=1.0), sam=dict(rho=0.05), cuda_graph=False)
    seen, kds = [], []
    fwd = m.distiller.teacher.forward
    m.distiller.teacher.forward = lambda x: (seen.append(x.clone()), fwd(x))[1]
    tp = m._train_pass
    m._train_pass = lambda rec, kd=None: (kds.append(kd), tp(rec, kd))[1]
    rec = _rec()
    for i in range(3):
        del seen[:], kds[:]
        m.train_iter(i, rec)
        torch.cuda.synchronize()
        assert len(seen) == 1 and len(kds) == 2 and kds[0] is kds[1], (i, len(seen), len(kds))
        assert torch.equal(seen[0], m.x_in)


def _subprocess(code, timeout=2400):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


@pytest.mark.parametrize("which,teacher", [("alexnet_bf16", "alexnet_bf16"), ("alexnet_tf32", "alexnet_tf32"), ("resnet50", "resnet50")])
def test_graph_step_equals_eager_and_manual_composition(which, teacher, tmp_path):
    _subprocess("""
import test_gpu_distill as t
p = t.teacher_checkpoint(%r, %r)
print('launches', t.model_check(%r, %r, p))
print('OK')
""" % (teacher, str(tmp_path / "ckpt_1.pt"), which, teacher))


def test_resnet50_mixup_sam_one_teacher_forward(tmp_path):
    _subprocess("""
import test_gpu_distill as t
p = t.teacher_checkpoint('resnet50', %r)
t.sam_check(p)
print('OK')
""" % str(tmp_path / "ckpt_1.pt"))
