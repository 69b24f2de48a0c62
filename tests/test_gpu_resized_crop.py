"""Random-resized crop on the H100: ``resized_crop_mirror_norm_kernel`` against ``reference.resized_crop_mirror_normalize`` over edge
boxes, mirrors, mean modes, per-channel scales and output sizes; the CUDA ParaLoader in thread and process mode against the reference
of the boxes it drew, and bit-identical validation batches; native models training with the key under the CUDA graph; and the
launch counts of the step and of the loader."""
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from theanompi_b200.models.data.utils import check_resized_crop, draw_resized_crops  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402

H = W = 256
STD = np.array([0.229, 0.224, 0.225], np.float32)


def _boxes(out_hw, n_random=6, seed=0):
    """Full image, 1 pixel, tiny (heavy upsampling), touching the bottom / right edges, the output's size at the corner, larger
    than the output (downscaling), plus random draws."""
    oh, ow = min(out_hw[0], H), min(out_hw[1], W)           # the output's size where it fits the image
    fixed = [[0, 0, H, W], [100, 37, 1, 1], [255, 255, 1, 1], [17, 250, 3, 2], [W - 60, H - 45, 60, 45], [0, W - 9, 200, 9],
             [H - oh, W - ow, oh, ow], [5, 3, 250, 240], [0, 0, H, 1]]
    rnd, _ = draw_resized_crops(n_random, (H, W), (0.08, 1.0), (0.75, 4 / 3), np.random.default_rng(seed))
    return torch.tensor(np.concatenate([np.int32(fixed), rnd]), dtype=torch.int32)


def _inputs(N, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)
    means = {0: torch.tensor([127.5]), 1: torch.tensor([123.7, 116.3, 103.5]), 2: torch.rand(H, W, 3, generator=g) * 255}
    return x, means


@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227), (160, 288)])
@pytest.mark.parametrize("mean_mode", [0, 1, 2])
@pytest.mark.parametrize("cscale", [False, True])
def test_kernel_matches_reference(out_hw, mean_mode, cscale):
    """fp32 within 1e-6 + 5e-7·|ref| (about 4 ulp at the normalised range); bf16 within one bf16 rounding (2^-8 relative) of the
    fp32 reference.  cw = 224, 227 and 288 > 128 use the second (and third) blockIdx.y."""
    from theanompi_b200.ops import cuda_impl
    boxes = _boxes(out_hw, seed=mean_mode)
    N = boxes.shape[0]
    x, means = _inputs(N, 7 + mean_mode)
    mean = means[mean_mode]
    scale = torch.from_numpy(1.0 / 255.0 / STD) if cscale else 1.0 / 255.0
    flips = torch.tensor([i % 2 for i in range(N)], dtype=torch.uint8)
    want = ref.resized_crop_mirror_normalize(x, mean, scale, out_hw, boxes, flips)
    xd, bd, fd = x.cuda(), boxes.cuda(), flips.cuda()
    got = cuda_impl.resized_crop_mirror_normalize(xd, mean.cuda(), scale, out_hw, bd, fd, torch.float32).cpu()
    torch.testing.assert_close(got, want, rtol=5e-7, atol=1e-6)
    got16 = cuda_impl.resized_crop_mirror_normalize(xd, mean.cuda(), scale, out_hw, bd, fd, torch.bfloat16).float().cpu()
    assert ((got16 - want).abs() <= want.abs() * 2.0 ** -8 + 1e-6).all()


def test_box_of_the_output_size_equals_the_fixed_crop_kernel():
    """A box equal to the output size is the existing crop kernel's output bit for bit, mirrored or not, in both dtypes."""
    from theanompi_b200.ops import cuda_impl
    x, means = _inputs(8, 3)
    offs = torch.tensor([[0, 0], [32, 29], [3, 7], [16, 1], [0, 29], [32, 0], [10, 10], [5, 20]], dtype=torch.int32)
    flips = torch.tensor([0, 1, 1, 0, 1, 0, 1, 0], dtype=torch.uint8)
    boxes = torch.cat([offs, torch.tensor([[224, 227]] * 8, dtype=torch.int32)], 1)
    cs = torch.from_numpy(1.0 / 255.0 / STD)
    for dt in (torch.float32, torch.bfloat16):
        a = cuda_impl.resized_crop_mirror_normalize(x.cuda(), means[2].cuda(), cs, (224, 227), boxes.cuda(), flips.cuda(), dt)
        b = cuda_impl.crop_mirror_normalize(x.cuda(), means[2].cuda(), cs, (224, 227), offs.cuda(), flips.cuda(), dt)
        assert torch.equal(a, b), dt


def test_kernel_refuses_a_non_uint8_batch():
    from theanompi_b200.ops import cuda_impl
    x = torch.zeros(1, 8, 8, 3, device="cuda")
    with pytest.raises(ValueError, match="uint8"):
        cuda_impl.resized_crop_mirror_normalize(x, torch.zeros(1, device="cuda"), 1.0, (4, 4),
                                                torch.tensor([[0, 0, 8, 8]], dtype=torch.int32, device="cuda"),
                                                torch.zeros(1, dtype=torch.uint8, device="cuda"))


# --------------------------------------------------------------------------- the CUDA loader
CFG = check_resized_crop({"scale": [0.08, 1.0], "seed": 4})


def _raw(d, item):
    raw = np.empty((16, H, W, 3), np.uint8)
    src = d.read(item, raw)
    return torch.from_numpy(src.numpy().copy() if src is not None else raw)


def _check_train_batches(ld, raw_of, items, mean, cs, n=3):
    ld.request(items[0], "train")
    for k in range(1, n + 1):
        ld.request(items[k % len(items)], "train")
        b = ld.get()
        torch.cuda.synchronize()
        assert b.boxes is not None and b.boxes.shape == (16, 4)
        want = ref.resized_crop_mirror_normalize(raw_of(b.item), mean, cs, (224, 224), b.boxes, b.flips)
        got = b.x.float().cpu()
        assert b.x.dtype == torch.bfloat16 and tuple(got.shape) == (16, 224, 224, 3)
        assert ((got - want).abs() <= want.abs() * 2.0 ** -8 + 1e-6).all()
        assert b.h2d_bytes == 16 * H * W * 3 + 16 * 17
    ld.drain()


def test_thread_loader_reproduces_the_reference_of_its_boxes():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    ld = d.para_load_init("cuda:0", 224, 224, True, False, out_dtype=torch.bfloat16, resized_crop=CFG, rank=1)
    try:
        _check_train_batches(ld, lambda item: _raw(d, item), d.train_img, torch.from_numpy(d.rawdata[4]),
                             torch.from_numpy(1.0 / 255.0 / d.rawdata[5]))
    finally:
        d.para_load_close()


def test_process_loader_reproduces_the_reference_of_its_boxes(tmp_path):
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
                    host_buffers=pr.tensors, on_close=pr.close, resized_crop=CFG, rank=0)
    try:
        _check_train_batches(ld, lambda item: torch.from_numpy(files[item]), sorted(files), torch.from_numpy(mean),
                             torch.from_numpy(1.0 / 255.0 / STD))
    finally:
        ld.close()


def test_val_batches_are_bit_identical_to_a_loader_without_the_key():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    outs = []
    for cfg in (None, CFG):
        d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=2, file_batch_size=16)
        d.batch_data(16)
        ld = d.para_load_init("cuda:0", 227, 227, True, False, out_dtype=torch.bfloat16, resized_crop=cfg)
        try:
            if cfg is not None:                             # a train batch first: val must not depend on it
                ld.request(d.train_img[0], "train"); ld.request(d.train_img[1], "train"); ld.get(); ld.drain()
            ld.request(d.val_img[0], "val"); ld.request(d.val_img[1], "val")
            outs.append([ld.get().x.clone(), ld.get().x.clone()])
            ld.drain()
        finally:
            d.para_load_close()
    assert all(torch.equal(a, b) for a, b in zip(*outs))


def test_loader_launches_one_native_kernel_per_batch():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.ops import native
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    counts = {}
    for name, cfg in (("off", None), ("on", CFG)):
        ld = ParaLoader(d.read, "cuda:0", (16, H, W, 3), (224, 224), mean=d.rawdata[4], threaded=False, resized_crop=cfg)
        torch.cuda.synchronize()
        native.reset_launch_count()
        ld.request(d.train_img[0], "train")
        ld.get()
        torch.cuda.synchronize()
        counts[name] = native.launch_count()
        ld.close()
    assert counts == {"off": 1, "on": 1}, counts


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
    ("alexnet", "theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64)),
    ("resnet50", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50", dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 1, 1))),
    ("resnet50_mix_drop", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50",
     dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 2, 1), mixup=dict(alpha=0.2, cutmix_alpha=1.0), drop_path_rate=0.1))])
def test_models_train_with_the_key_under_the_cuda_graph(name, cls, extra):
    m = _model(cls, cuda_graph=True, random_resized_crop={"seed": 1}, **extra)
    try:
        assert m.data.loader is not None and m.data.loader.resized_crop is not None
        costs, val = _train_val(m, 4)
        assert "step" in m.captured_steps(), "the step was not captured"
        assert all(np.isfinite(costs)) and np.isfinite(val), (costs, val)
    finally:
        m.cleanup()


def test_the_key_does_not_change_the_step_launches():
    """The loader kernel runs on the copy stream, outside the step: AlexNet's training step launches what it launches without the key."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    for name, extra in (("off", {}), ("on", dict(random_resized_crop={}))):
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
