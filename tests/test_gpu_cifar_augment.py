"""CIFAR augmentation on the H100: ``cifar_augment_draw_kernel`` against ``reference.cifar_augment_draw`` bit for bit, the zero-filled
``crop_mirror_norm_kernel`` and Cutout through ``erase_boxes_kernel`` against the reference with torch.equal, and Wide_ResNet under
its CUDA graph: the buffers and the stem input of every replay against the reference, the mix point with mixup, launch counts,
validation and inference that never augment, and bit-reproducible deterministic runs with grad_accum, drop-path and tf32."""
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

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.ops import cifar_augment as ca  # noqa: E402
from theanompi_b200.ops import mixup  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

DEV = "cuda:0"


# --------------------------------------------------------------------------- the draw
@pytest.mark.parametrize("cfg", [dict(), dict(pad=0, cutout=32), dict(pad=31, cutout=17), dict(pad=1, cutout=1)])
def test_draw_kernel_matches_reference(cfg):
    from theanompi_b200.ops import cuda_impl
    for seed in (0, 0xDEADBEEF12345678, 2 ** 64 - 1):
        cfg_s = ca.check_config(dict(cfg, seed=seed))
        for B in (1, 7, 128, 256):
            for rank in range(4):
                aug = ca.CifarAugment(cfg_s, rank, B, DEV)
                for step in (0, 1, 2 ** 32 + 5):
                    st = torch.full((1,), step, dtype=torch.int64, device=DEV)
                    cuda_impl.cifar_augment_draw(aug.cfg, rank, st, aug.offs, aug.flips, aug.boxes)
                    want = ref.cifar_augment_draw(cfg_s, seed, rank, step, B)
                    for got, w in zip((aug.offs, aug.flips, aug.boxes), want):
                        assert torch.equal(got.cpu(), w), (cfg, seed, B, rank, step)


# --------------------------------------------------------------------------- the zero-filled crop and Cutout
def _records(N, pad):
    offs = torch.randint(-pad, pad + 1, (N, 2), dtype=torch.int32)
    offs[0] = torch.tensor([-pad, -pad]); offs[1] = torch.tensor([pad, pad]); offs[2] = torch.tensor([-pad, pad])
    offs[3] = torch.tensor([40, 0]); offs[4] = torch.tensor([0, -33]); offs[5] = torch.tensor([-32, 32])   # wholly outside
    flips = (torch.arange(N) % 2).to(torch.uint8)
    return offs, flips


@pytest.mark.parametrize("tin", [torch.bfloat16, torch.float32, torch.uint8])
@pytest.mark.parametrize("tout", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("pad", [1, 4, 31])
def test_zero_fill_crop_matches_reference(tin, tout, pad):
    from theanompi_b200.ops import cuda_impl
    torch.manual_seed(pad)
    N = 37
    x = torch.randint(0, 256, (N, 32, 32, 3)).to(tin)
    mean = torch.rand(32, 32, 3) * 255
    offs, flips = _records(N, pad)
    got = cuda_impl.crop_mirror_normalize(x.to(DEV), mean.to(DEV), 1.0 / 64.0, (32, 32), offs.to(DEV), flips.to(DEV), tout,
                                          zero_fill=True).cpu()
    want = ref.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), offs, flips, tout, zero_fill=True)
    assert torch.equal(got, want)
    assert (got[3:6] == 0).all()
    zo, zf = torch.zeros((N, 2), dtype=torch.int32), torch.zeros(N, dtype=torch.uint8)
    plain = cuda_impl.crop_mirror_normalize(x.to(DEV), mean.to(DEV), 1.0 / 64.0, (32, 32), zo.to(DEV), zf.to(DEV), tout).cpu()
    assert torch.equal(plain, ref.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), zo, zf, tout))


@pytest.mark.parametrize("dt", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("L", [1, 16, 17, 32])
def test_cutout_through_erase_boxes_matches_reference(dt, L):
    from theanompi_b200.ops import cuda_impl
    torch.manual_seed(L)
    N = 64
    cy, cx = np.random.RandomState(L).randint(0, 32, (2, N))
    cy[:4], cx[:4] = [0, 31, 0, 31], [0, 31, 31, 0]
    boxes = torch.from_numpy(ca.cutout_boxes(cy, cx, L))
    x = torch.randn(N, 32, 32, 3).to(dt)
    got = cuda_impl.random_erase(x.to(DEV), boxes.to(DEV)).cpu()
    want = ref.random_erase(x, boxes)
    assert torch.equal(got, want)
    if L == 1:
        assert torch.equal(got, x)                                  # L = 1 cuts an empty hole


# --------------------------------------------------------------------------- Wide_ResNet
WRN = dict(batch_size=16, file_batch_size=32, depth=10, widen=2, data_kwargs=dict(n_synthetic=256, synthetic=True))


def _model(dev=DEV, **cfg):
    from theanompi_b200.models import layers2
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)
    m = Wide_ResNet(dict(verbose=False, rank=0, size=1, device=dev, **dict(WRN, **cfg)))
    m.compile_iter_fns("avg")
    return m


def _recorder():
    from theanompi_b200.utils.recorder import Recorder
    return Recorder(None, 10 ** 6, "t", False, device=DEV)


def _ref_stem_input(m):
    """The reference augmentation of this step's x_in with the drawn buffers, mixed with the drawn record when mixup is on."""
    aug = m.cifar_aug
    x = ref.crop_mirror_normalize(m.x_in.cpu(), m._mean.cpu(), 1.0 / 64.0, (32, 32), aug.offs.cpu(), aug.flips.cpu(), m.act_dtype,
                                  zero_fill=True)
    if aug.cutout:
        x = ref.random_erase(x, aug.boxes.cpu())
    return x if m.mixer is None else ref.mix_batch(x, m.mixer.rec.cpu())


@pytest.mark.parametrize("extra", [dict(cifar_augment=dict(seed=11)), dict(cifar_augment=dict(cutout=16, pad=4, seed=12)),
                                   dict(cifar_augment=dict(cutout=16), mixup=dict(alpha=1.0, cutmix_alpha=1.0, seed=5))])
def test_graph_replays_draw_anew_and_feed_the_stem_the_reference_batch(extra):
    from theanompi_b200.ops import cuda_impl
    m = _model(cuda_graph=True, **extra)
    keep = torch.empty((16, 32, 32, 3), dtype=m.act_dtype, device=DEV)
    fwd = m.stem.forward
    m.stem.forward = lambda x: (keep.copy_(x), fwd(x))[1]
    rec, prev, modes = _recorder(), None, set()
    cfg = m.cifar_aug.cfg
    for i in range(6):
        step = int(cuda_impl.step_counter(DEV).item())
        m.train_iter(i, rec)
        torch.cuda.synchronize()
        bufs = tuple(t.cpu().clone() for t in (m.cifar_aug.offs, m.cifar_aug.flips, m.cifar_aug.boxes))
        for got, w in zip(bufs, ref.cifar_augment_draw(cfg, cfg["seed"], 0, step, 16)):
            assert torch.equal(got, w), i
        if prev is not None:
            assert not torch.equal(bufs[0], prev[0])
        prev = bufs
        want, got = _ref_stem_input(m), keep.cpu()
        mode = int(mixup.decode(m.mixer.rec)["mode"]) if m.mixer is not None else mixup.MIX_NONE
        modes.add(mode)
        if mode == mixup.MIX_MIXUP:                                 # the mix kernel is within one ulp of the reference
            assert float((got.float() - want.float()).abs().max()) <= 2.0 ** -7 * float(want.float().abs().max()), i
        else:
            assert torch.equal(got, want), i
    assert m.captured_steps() == {"step"}
    assert all(np.isfinite([float(c) for c in rec.train_info["cost"]]))
    m.cleanup()


def test_launch_counts():
    """One native launch more per step with the key (the draw; the crop launch is already in the step), two with Cutout."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    for name, extra in (("absent", {}), ("none", dict(cifar_augment=None)), ("crop", dict(cifar_augment={})),
                        ("cutout", dict(cifar_augment=dict(cutout=16)))):
        m = _model(cuda_graph=False, **extra)
        for _ in range(2):
            torch.cuda.synchronize()
            native.reset_launch_count()
            m.forward_backward(0)
            torch.cuda.synchronize()
            counts[name] = native.launch_count()
        m.cleanup()
    layers2.Dropout.SetDropoutOn(); layers2.Crop.SetRandCropOn()
    print(counts)
    assert counts["none"] == counts["absent"]
    assert counts["crop"] == counts["absent"] + 1 and counts["cutout"] == counts["absent"] + 2, counts


def runs(extra, steps=4, graph=True):
    """A fresh Wide_ResNet with ``extra`` trained ``steps`` steps from a reset device counter: (W, U, losses, graph used)."""
    from theanompi_b200.ops import cuda_impl
    cuda_impl._STEP.clear()
    ops.seed_dropout(0x5EED)
    m = _model(cuda_graph=graph, **extra)
    rec = _recorder()
    for i in range(steps):
        m.train_iter(i, rec)
    torch.cuda.synchronize()
    out = (m.arena.W.clone(), m.arena.U.clone(), [float(c) for c in rec.train_info["cost"]], bool(m.captured_steps()))
    m.cleanup()
    return out


def val_inf_same():
    """Train with cutout, then validate and infer from the same weights and statistics with the key and with it switched off."""
    m = _model(cifar_augment=dict(cutout=16), mixup=dict(cutmix_alpha=1.0))
    rec = _recorder()
    for i in range(3):
        m.train_iter(i, rec)
    m.compile_inference()
    x = m.shared_x[:m.batch_size].clone()
    stats = [(b.running_mean.clone(), b.running_var.clone()) for b in m._bn_layers()]

    def outputs():
        for b, (rm, rv) in zip(m._bn_layers(), stats):
            b.running_mean.copy_(rm); b.running_var.copy_(rv)
        c = [float(v) for v in m.val_fn(0)]
        p = m.inf_fn(x).clone()
        torch.cuda.synchronize()
        return c, p
    c1, p1 = outputs()
    m.cifar_augment = None
    m.check_cifar_augment()
    c0, p0 = outputs()
    print(c1, c0)
    m.cleanup()
    return c1 == c0 and torch.equal(p1, p0)


def _subprocess(code, timeout=900):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-1500:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


def test_validation_and_inference_never_augment():
    _subprocess("""
import test_gpu_cifar_augment as t
assert t.val_inf_same()
print('OK')
""")


@pytest.mark.parametrize("dtype", ["bf16", "tf32"])
def test_deterministic_runs_with_grad_accum_and_drop_path_are_bit_identical(dtype):
    _subprocess("""
import test_gpu_cifar_augment as t
extra = dict(dtype=%r, cifar_augment=dict(cutout=16, seed=4), grad_accum=2, drop_path_rate=0.3, label_smoothing=0.1)
a, b = t.runs(extra, steps=6), t.runs(extra, steps=6)
plain = t.runs(dict(dtype=%r, grad_accum=2, drop_path_rate=0.3, label_smoothing=0.1), steps=6)
print(a[2], b[2], plain[2])
assert a[3] and b[3] and a[2] == b[2] and t.torch.equal(a[0], b[0]) and t.torch.equal(a[1], b[1])
assert all(t.np.isfinite(a[2])) and not t.torch.equal(a[0], plain[0])
print('OK')
""" % (dtype, dtype))


@pytest.mark.parametrize("opt", ["adam", "sgd", "lars", "lamb"])
def test_every_optimizer_trains_with_it(opt):
    extra = dict(optimizer=opt, cifar_augment=dict(cutout=16), lr_schedule=dict(warmup_steps=2, decay="cosine"))
    if opt in ("adam", "sgd"):
        extra["grad_clip"] = 5.0
    w, _, losses, used = runs(extra, steps=4)
    assert used and all(np.isfinite(losses)), losses
