"""Colour jitter and PCA lighting on the H100: ``crop_mean_kernel`` against float64 sums, the jitter path of
``resized_crop_mirror_norm_kernel`` against the float64 sequential oracle (tests/color_oracle.py) over fixed and resized boxes, mean
modes, per-channel scales, output sizes and both output dtypes; the identity record against the existing crop kernels; the CUDA
ParaLoader in thread and process mode against the oracle of what it drew, and bit-identical validation batches; native models training
with the key under the CUDA graph; and the launch counts of the loader and of the step.

Bounds, with ε = 2^-24 (one fp32 rounding) and P = ch·cw output pixels:

* crop mean.  Each bilinear value v̂ carries at most 4 roundings of non-negative terms; each thread adds its
  ⌈ch/16⌉·⌈cw/32⌉ values in order, then 5 shuffle and 4 cross-warp levels add the partial sums; the division rounds once.  So
  |μ − μ₆₄| ≤ u_μ·μ₆₄ with u_μ = (⌈ch/16⌉·⌈cw/32⌉ + 9 + 4 + 1)·ε.  A box of the output's size sums integers below 2^24 exactly:
  μ equals the exact sum divided once in fp32, bit for bit.
* jitter path.  out = (M·v̂ + t − m̂)·s_c with t = K·μ + ℓ.  The record rounds M, K, ℓ once (ε each); t takes three fused
  multiply-adds on top of μ's u_μ; M·v̂ + t three more on top of v̂'s 4ε; m̂ (per-pixel mean) 4ε; the subtraction, the product by s_c and
  s_c = scale·cscale one each.  Every one of these is below (u_μ + 12)·ε relative to a term of
  S = (|M|·v̂ + |K|·μ + |ℓ| + |m̂|)·s_c or to |want|, so |got − want| ≤ u·|want| + u·S with u = u_μ + 12ε.  bf16 adds one
  rounding of the output, 2^-8·|want|.
"""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import color_oracle as co  # noqa: E402
from test_gpu_resized_crop import _boxes  # noqa: E402
from theanompi_b200.models.data.utils import (check_color_jitter, check_resized_crop, color_jitter_records,  # noqa: E402
                                              color_jitter_rng)

H = W = 256
STD = np.array([0.229, 0.224, 0.225], np.float32)
ALL4 = {"brightness": 0.4, "contrast": 0.4, "saturation": 0.4, "lighting": 0.1}
EPS = 2.0 ** -24


def u_mu(out_hw):
    return (-(-out_hw[0] // 16) * -(-out_hw[1] // 32) + 14) * EPS


def u_out(out_hw):
    return u_mu(out_hw) + 12 * EPS


def _inputs(N, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)
    means = {0: torch.tensor([127.5]), 1: torch.tensor([123.7, 116.3, 103.5]), 2: torch.rand(H, W, 3, generator=g) * 255}
    return x, means


def _fixed_boxes(out_hw, N, seed):
    rs = np.random.RandomState(seed)
    oy, ox = rs.randint(0, H - out_hw[0] + 1, N), rs.randint(0, W - out_hw[1] + 1, N)
    oy[:2], ox[:2] = [0, H - out_hw[0]], [0, W - out_hw[1]]
    return torch.tensor(np.stack([oy, ox, np.full(N, out_hw[0]), np.full(N, out_hw[1])], 1), dtype=torch.int32)


def _draw(N, seed, cfg=ALL4, rank=0):
    cfg = check_color_jitter(dict(cfg, seed=seed))
    return color_jitter_records(N, cfg, color_jitter_rng(cfg, rank))


# --------------------------------------------------------------------------- crop mean
@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227), (160, 288)])
def test_crop_mean(out_hw):
    from theanompi_b200.ops import cuda_impl
    boxes = _boxes(out_hw, seed=1)
    x, _ = _inputs(boxes.shape[0], 5)
    xd = x.cuda()
    mu = cuda_impl.crop_mean(xd, boxes.cuda(), out_hw).cpu()
    assert torch.equal(mu, cuda_impl.crop_mean(xd, boxes.cuda(), out_hw).cpu()), "not bit-identical from run to run"
    assert (mu[:, 3] == 0).all()
    want = co.crop_sums(x.numpy(), boxes.numpy(), out_hw) / (out_hw[0] * out_hw[1])
    assert (np.abs(mu[:, :3].double().numpy() - want) <= u_mu(out_hw) * want).all(), np.abs(mu[:, :3].numpy() - want).max()
    if out_hw[1] <= W:                                     # boxes of the output's size: exact integer sums, one division
        fb = _fixed_boxes(out_hw, 8, 2)
        x8 = x[:8]
        mu = cuda_impl.crop_mean(x8.cuda(), fb.cuda(), out_hw).cpu()
        sums = co.crop_sums(x8.numpy(), fb.numpy(), out_hw)
        assert (sums == np.rint(sums)).all()
        exact = torch.tensor(sums, dtype=torch.float32) / torch.tensor(float(out_hw[0] * out_hw[1]))
        assert torch.equal(mu[:, :3], exact)


# --------------------------------------------------------------------------- the jitter path
@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227), (160, 288)])
@pytest.mark.parametrize("kind", ["fixed", "resized"])
@pytest.mark.parametrize("mean_mode", [0, 1, 2])
@pytest.mark.parametrize("cscale", [False, True])
def test_jitter_path_matches_the_oracle(out_hw, kind, mean_mode, cscale):
    """fp32 within u·|want| + u·S, bf16 within that plus 2^-8·|want| (module docstring).  cw = 224, 227 and 288 > 128 use the second
    (and third) blockIdx.y."""
    from theanompi_b200.ops import cuda_impl
    if kind == "fixed" and out_hw[1] > W:
        pytest.skip("a fixed crop must fit the image")
    boxes = _boxes(out_hw, seed=mean_mode) if kind == "resized" else _fixed_boxes(out_hw, 12, mean_mode)
    N = boxes.shape[0]
    x, means = _inputs(N, 11 + mean_mode)
    mean = means[mean_mode]
    scale = torch.from_numpy(1.0 / 255.0 / STD) if cscale else 1.0 / 255.0
    flips = torch.tensor([(i // 2) % 2 for i in range(N)], dtype=torch.uint8)
    rec, fac, order, alpha = _draw(N, 3 + mean_mode)
    sc64 = scale.double().numpy() if cscale else scale
    want, S = co.oracle(x.numpy(), mean.double().numpy(), sc64, out_hw, boxes.numpy(), flips.numpy(), fac, order, alpha, rec)
    xd, bd, fd, rd = x.cuda(), boxes.cuda(), flips.cuda(), torch.from_numpy(rec).cuda()
    mu = cuda_impl.crop_mean(xd, bd, out_hw)
    u = u_out(out_hw)
    got = cuda_impl.color_crop_mirror_normalize(xd, mean.cuda(), scale, out_hw, bd, fd, rd, mu, torch.float32).cpu().numpy()
    co.assert_bounded(got, want, S, u, "fp32")
    got16 = cuda_impl.color_crop_mirror_normalize(xd, mean.cuda(), scale, out_hw, bd, fd, rd, mu, torch.bfloat16).float().cpu().numpy()
    co.assert_bounded(got16, want, S, u + 2.0 ** -8, "bf16")


def test_without_contrast_the_kernel_takes_no_mean():
    """K ≡ 0 when the contrast strength is 0: the loader passes no μ and the output is the oracle's."""
    from theanompi_b200.ops import cuda_impl
    out_hw = (227, 227)
    boxes = _boxes(out_hw, seed=4)
    N = boxes.shape[0]
    x, means = _inputs(N, 4)
    flips = torch.tensor([i % 2 for i in range(N)], dtype=torch.uint8)
    rec, fac, order, alpha = _draw(N, 8, {"brightness": 0.4, "saturation": 0.4, "lighting": 0.1})
    assert (rec[:, 9:18] == 0).all()
    cs = torch.from_numpy(1.0 / 255.0 / STD)
    want, S = co.oracle(x.numpy(), means[2].double().numpy(), cs.double().numpy(), out_hw, boxes.numpy(), flips.numpy(), fac, order,
                        alpha, rec)
    got = cuda_impl.color_crop_mirror_normalize(x.cuda(), means[2].cuda(), cs, out_hw, boxes.cuda(), flips.cuda(),
                                                torch.from_numpy(rec).cuda(), None, torch.float32).cpu().numpy()
    co.assert_bounded(got, want, S, u_out(out_hw), "no mu")


def test_identity_record_equals_the_crop_kernels():
    """M = I, K = 0, ℓ = 0: on boxes of the output's size, crop_mirror_norm bit for bit in both dtypes; on resized boxes,
    resized_crop_mirror_norm within the fp32 bound."""
    from theanompi_b200.ops import cuda_impl
    x, means = _inputs(12, 3)
    ident = torch.zeros(12, 24)
    ident[:, [0, 4, 8]] = 1.0
    ident = ident.cuda()
    cs = torch.from_numpy(1.0 / 255.0 / STD)
    flips = torch.tensor([0, 1] * 6, dtype=torch.uint8).cuda()
    xd = x.cuda()
    for out_hw in ((224, 227), (227, 227)):
        fb = _fixed_boxes(out_hw, 12, 6).cuda()
        for m in means.values():
            for dt in (torch.float32, torch.bfloat16):
                a = cuda_impl.color_crop_mirror_normalize(xd, m.cuda(), cs, out_hw, fb, flips, ident, None, dt)
                b = cuda_impl.crop_mirror_normalize(xd, m.cuda(), cs, out_hw, fb[:, :2].contiguous(), flips, dt)
                assert torch.equal(a, b), (out_hw, dt)
    out_hw = (227, 227)
    boxes = _boxes(out_hw, n_random=3, seed=5).cuda()
    xr = xd[:boxes.shape[0]]
    for m in means.values():
        a = cuda_impl.color_crop_mirror_normalize(xr, m.cuda(), cs, out_hw, boxes, flips[:boxes.shape[0]], ident[:boxes.shape[0]],
                                                  None, torch.float32).cpu().double()
        b = cuda_impl.resized_crop_mirror_normalize(xr, m.cuda(), cs, out_hw, boxes, flips[:boxes.shape[0]], torch.float32).cpu().double()
        mag = (xr.cpu().double().amax() + m.double().abs().max()) * cs.double().max()
        assert ((a - b).abs() <= 2 * u_out(out_hw) * (b.abs() + mag)).all()


def test_wrappers_refuse_bad_inputs():
    from theanompi_b200.ops import cuda_impl
    boxes = torch.tensor([[0, 0, 8, 8]], dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="uint8"):
        cuda_impl.crop_mean(torch.zeros(1, 8, 8, 3, device="cuda"), boxes, (4, 4))
    with pytest.raises(ValueError, match="C = 3"):
        cuda_impl.crop_mean(torch.zeros(1, 8, 8, 4, dtype=torch.uint8, device="cuda"), boxes, (4, 4))
    rec = torch.zeros(1, 25, device="cuda")[:, 1:]                # 4-byte aligned only
    with pytest.raises(AssertionError):
        cuda_impl.color_crop_mirror_normalize(torch.zeros(1, 8, 8, 3, dtype=torch.uint8, device="cuda"), torch.zeros(1, device="cuda"),
                                              1.0, (4, 4), boxes, torch.zeros(1, dtype=torch.uint8, device="cuda"), rec)


# --------------------------------------------------------------------------- the CUDA loader
CJ = check_color_jitter(dict(ALL4, seed=6))
RRC = check_resized_crop({"seed": 4})


def _raw(d, item):
    raw = np.empty((16, H, W, 3), np.uint8)
    src = d.read(item, raw)
    return src.numpy().copy() if src is not None else raw


def _check_train_batches(ld, raw_of, items, mean, sc, rank, n=3):
    rng = color_jitter_rng(CJ, rank)
    ld.request(items[0], "train")
    for k in range(1, n + 1):
        ld.request(items[k % len(items)], "train")
        b = ld.get()
        torch.cuda.synchronize()
        rec, fac, order, alpha = color_jitter_records(16, CJ, rng)
        assert np.array_equal(b.records, rec)
        want, S = co.oracle(raw_of(b.item), mean, sc, (224, 224), b.boxes, b.flips, fac, order, alpha, rec)
        assert b.x.dtype == torch.bfloat16 and tuple(b.x.shape) == (16, 224, 224, 3)
        co.assert_bounded(b.x.float().cpu().numpy(), want, S, u_out((224, 224)) + 2.0 ** -8, "loader batch %d" % k)
        assert b.h2d_bytes == 16 * H * W * 3 + 16 * 17 + 16 * 96
    ld.drain()


@pytest.mark.parametrize("rrc", [None, RRC])
def test_thread_loader_reproduces_the_oracle_of_its_draw(rrc):
    from theanompi_b200.models.data.imagenet import ImageNet_data
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    ld = d.para_load_init("cuda:0", 224, 224, True, False, out_dtype=torch.bfloat16, resized_crop=rrc, rank=1, color_jitter=CJ)
    try:
        _check_train_batches(ld, lambda item: _raw(d, item), d.train_img, d.rawdata[4].astype(np.float64),
                             (1.0 / 255.0 / d.rawdata[5]).astype(np.float64), 1)
    finally:
        d.para_load_close()


@pytest.mark.parametrize("rrc", [None, RRC])
def test_process_loader_reproduces_the_oracle_of_its_draw(tmp_path, rrc):
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.models.data.proc_loader import ProcReader
    files = {}
    for i in range(3):
        a = np.random.RandomState(i).randint(0, 256, (16, H, W, 3), dtype=np.uint8)
        files[str(tmp_path / ("b%d.npy" % i))] = a
        np.save(str(tmp_path / ("b%d.npy" % i)), a)
    mean = np.random.RandomState(9).uniform(0, 255, (H, W, 3)).astype(np.float32)
    pr = ProcReader((16, H, W, 3), depth=2)
    ld = ParaLoader(pr.read, "cuda:0", (16, H, W, 3), (224, 224), mean=mean, std_scale=1.0 / 255.0 / STD, out_dtype=torch.bfloat16,
                    host_buffers=pr.tensors, on_close=pr.close, resized_crop=rrc, rank=0, color_jitter=CJ)
    try:
        _check_train_batches(ld, lambda item: files[item], sorted(files), mean.astype(np.float64),
                             (1.0 / 255.0 / STD).astype(np.float64), 0)
    finally:
        ld.close()


def test_val_batches_are_bit_identical_to_a_loader_without_the_key():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    outs = []
    for cfg in (None, CJ):
        d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=2, file_batch_size=16)
        d.batch_data(16)
        ld = d.para_load_init("cuda:0", 227, 227, True, False, out_dtype=torch.bfloat16, color_jitter=cfg)
        try:
            if cfg is not None:                             # a train batch first: val must not depend on it
                ld.request(d.train_img[0], "train"); ld.request(d.train_img[1], "train"); ld.get(); ld.drain()
            ld.request(d.val_img[0], "val"); ld.request(d.val_img[1], "val")
            outs.append([ld.get().x.clone(), ld.get().x.clone()])
            ld.drain()
        finally:
            d.para_load_close()
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_loader_launches_per_train_batch():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.ops import native
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    counts = {}
    for name, cfg in (("off", None), ("contrast", CJ), ("no contrast", check_color_jitter({"lighting": 0.1}))):
        ld = ParaLoader(d.read, "cuda:0", (16, H, W, 3), (224, 224), mean=d.rawdata[4], threaded=False, color_jitter=cfg)
        torch.cuda.synchronize()
        native.reset_launch_count()
        ld.request(d.train_img[0], "train")
        ld.get()
        torch.cuda.synchronize()
        counts[name] = native.launch_count()
        ld.close()
    assert counts == {"off": 1, "contrast": 2, "no contrast": 1}, counts


# --------------------------------------------------------------------------- models
def _model(cls_path, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    mod, cls = cls_path.rsplit(".", 1)
    return getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", n_class=100,
                                                            data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True), **cfg))


def _train_val(m, steps):
    from theanompi_b200.utils.recorder import Recorder
    rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
    m.compile_iter_fns("avg")
    m.reset_iter("train")
    costs = []
    for i in range(steps):
        m.train_iter(i, rec)
        torch.cuda.synchronize()
        costs.append(float(rec.train_info["cost"][-1]))
    m.reset_iter("train")
    m.reset_iter("val")
    m.val_iter(0, rec)
    torch.cuda.synchronize()
    return costs, float(rec.val_info["cost"][-1])


@pytest.mark.parametrize("name,cls,extra", [
    ("alexnet", "theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64, color_jitter={"lighting": 0.1})),
    ("resnet50", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50",
     dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 1, 1), random_resized_crop={"seed": 1}, color_jitter=ALL4)),
    ("resnet50_mix_drop", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50",
     dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 2, 1), random_resized_crop={"seed": 1}, color_jitter=ALL4,
          mixup=dict(alpha=0.2, cutmix_alpha=1.0), drop_path_rate=0.1))])
def test_models_train_with_the_key_under_the_cuda_graph(name, cls, extra):
    m = _model(cls, cuda_graph=True, **extra)
    try:
        assert m.data.loader is not None and m.data.loader.color_jitter is not None
        costs, val = _train_val(m, 4)
        assert "step" in m.captured_steps(), "the step was not captured"
        assert all(np.isfinite(costs)) and np.isfinite(val), (costs, val)
    finally:
        m.cleanup()


def test_the_key_does_not_change_the_step_launches():
    """The loader kernels run on the copy stream, outside the step: AlexNet's training step launches what it launches without the key."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    for name, extra in (("off", {}), ("on", dict(color_jitter=ALL4))):
        m = _model("theanompi_b200.models.alex_net.AlexNet", cuda_graph=False, batch_size=64, file_batch_size=64, no_paraload=True, **extra)
        m.compile_iter_fns("avg")
        layers2.Dropout.SetDropoutOn()
        for _ in range(2):
            torch.cuda.synchronize()
            native.reset_launch_count()
            m.forward_backward(0)
            torch.cuda.synchronize()
            counts[name] = native.launch_count()
        m.cleanup()
    assert counts["off"] == counts["on"], counts
