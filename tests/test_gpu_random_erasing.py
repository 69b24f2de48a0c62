"""Random erasing on the H100: ``erase_boxes_kernel`` against the torch reference (it must zero exactly its boxes and leave every other
element bit-identical, in bf16 and fp32, at the models' output sizes and at the edges of the output); the CUDA ParaLoader in thread and
process mode, over the fixed, resized and colour-jittered crop paths, against the reference of its own draw; validation batches left
bit-identical; the launch counts of the loader and of the step; and native models training with the key under the CUDA graph.

Erasing is a store of zeros, so every comparison here is exact: the loader's batch with the key must equal, bit for bit, the batch of a
loader without it (same crop and colour draws, same kernels) with the drawn boxes set to 0.
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

from theanompi_b200.models.data.utils import (check_color_jitter, check_random_erasing, check_resized_crop,  # noqa: E402
                                              draw_erase_boxes, random_erasing_rng)
from theanompi_b200.ops import reference as ref  # noqa: E402

H = W = 256
STD = np.array([0.229, 0.224, 0.225], np.float32)
ALL4 = {"brightness": 0.4, "contrast": 0.4, "saturation": 0.4, "lighting": 0.1}
RE = check_random_erasing({"p": 0.7, "seed": 12})


# --------------------------------------------------------------------------- the kernel
def _edge_boxes(out_hw):
    h, w = out_hw
    return np.int32([[0, 0, 0, 0], [0, 0, h - 1, w - 1], [1, 1, h - 1, w - 1], [h - 1, w - 1, 1, 1], [0, 0, h, w], [5, 0, 3, w],
                     [0, w - 7, h, 7], [h // 2, 3, 0, 10]])


@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227), (160, 288)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_erase_kernel_zeroes_exactly_its_boxes(out_hw, dtype):
    from theanompi_b200.ops import cuda_impl, functional
    N = 136
    g = torch.Generator().manual_seed(1)
    x = (torch.rand((N,) + out_hw + (3,), generator=g) + 0.5).to(dtype)       # no zero outside the boxes
    cfg = check_random_erasing({"p": 0.9, "scale": [0.02, 0.6], "seed": out_hw[1]})
    boxes = draw_erase_boxes(N, out_hw, cfg, random_erasing_rng(cfg, 0))
    boxes[:8] = _edge_boxes(out_hw)
    want = ref.random_erase(x, boxes)
    xd = x.cuda()
    db = torch.from_numpy(boxes).cuda()
    got = cuda_impl.random_erase(xd, db)
    assert got is xd
    torch.cuda.synchronize()
    assert torch.equal(got.cpu(), want)
    erased = (want == 0).all(-1)
    assert int(erased.sum()) == int((boxes[:, 2].astype(np.int64) * boxes[:, 3]).sum())
    # the dispatch entry takes the same path; erasing twice changes nothing
    assert torch.equal(functional.random_erase(xd, db).cpu(), want)


def test_erase_wrapper_refuses_bad_inputs():
    from theanompi_b200.ops import cuda_impl
    boxes = torch.zeros((2, 4), dtype=torch.int32, device="cuda")
    with pytest.raises(ValueError, match="random_erase"):
        cuda_impl.random_erase(torch.zeros((2, 8, 8, 3)), boxes)
    with pytest.raises(ValueError, match="random_erase"):
        cuda_impl.random_erase(torch.zeros((2, 8, 8, 3), dtype=torch.uint8, device="cuda"), boxes)
    with pytest.raises(ValueError, match="random_erase"):
        cuda_impl.random_erase(torch.zeros((2, 8, 8, 3), device="cuda").transpose(1, 2), boxes)


# --------------------------------------------------------------------------- the CUDA loader
def _pair(make):
    """Two loaders built by make(random_erasing): with the key and without it."""
    return make(RE), make(None)


def _check_train_batches(ld, ld0, items, rank, n=4):
    rng = random_erasing_rng(RE, rank)
    for L in (ld, ld0):
        L.request(items[0], "train")
    erased = 0
    for k in range(1, n + 1):
        for L in (ld, ld0):
            L.request(items[k % len(items)], "train")
        b, b0 = ld.get(), ld0.get()
        torch.cuda.synchronize()
        boxes = draw_erase_boxes(16, (224, 224), RE, rng)
        assert np.array_equal(b.erase, boxes) and b0.erase is None
        for a in ("boxes", "flips", "records"):
            assert (getattr(b, a) is None and getattr(b0, a) is None) or np.array_equal(getattr(b, a), getattr(b0, a)), a
        assert b.x.dtype == torch.bfloat16 and tuple(b.x.shape) == (16, 224, 224, 3)
        assert torch.equal(b.x.cpu(), ref.random_erase(b0.x.cpu(), boxes)), "loader batch %d" % k
        assert b.h2d_bytes == b0.h2d_bytes + 16 * 16
        erased += int((boxes[:, 2] > 0).sum())
    assert erased > 0
    ld.drain(); ld0.drain()


@pytest.mark.parametrize("crop", ["fixed", "resized", "resized+color"])
def test_thread_loader_reproduces_the_reference_of_its_draw(crop):
    from theanompi_b200.models.data.imagenet import ImageNet_data
    rrc = check_resized_crop({"seed": 4}) if "resized" in crop else None
    cj = check_color_jitter(dict(ALL4, seed=6)) if "color" in crop else None
    ds = []

    def make(re):
        d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
        d.batch_data(16)
        ds.append(d)
        return d.para_load_init("cuda:0", 224, 224, True, False, out_dtype=torch.bfloat16, resized_crop=rrc, rank=1, color_jitter=cj,
                                random_erasing=re)
    try:
        ld, ld0 = _pair(make)
        _check_train_batches(ld, ld0, ds[0].train_img, 1)
    finally:
        for d in ds:
            d.para_load_close()


def test_process_loader_reproduces_the_reference_of_its_draw(tmp_path):
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.models.data.proc_loader import ProcReader
    files = {}
    for i in range(3):
        a = np.random.RandomState(i).randint(0, 256, (16, H, W, 3), dtype=np.uint8)
        files[str(tmp_path / ("b%d.npy" % i))] = a
        np.save(str(tmp_path / ("b%d.npy" % i)), a)
    mean = np.random.RandomState(9).uniform(0, 255, (H, W, 3)).astype(np.float32)
    lds = []

    def make(re):
        pr = ProcReader((16, H, W, 3), depth=2)
        lds.append(ParaLoader(pr.read, "cuda:0", (16, H, W, 3), (224, 224), mean=mean, std_scale=1.0 / 255.0 / STD,
                              out_dtype=torch.bfloat16, host_buffers=pr.tensors, on_close=pr.close, rank=0, random_erasing=re))
        return lds[-1]
    try:
        ld, ld0 = _pair(make)
        _check_train_batches(ld, ld0, sorted(files), 0)
    finally:
        for ld in lds:
            ld.close()


def test_val_batches_are_bit_identical_to_a_loader_without_the_key():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    outs = []
    for cfg in (None, check_random_erasing({"p": 1.0})):
        d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=2, file_batch_size=16)
        d.batch_data(16)
        ld = d.para_load_init("cuda:0", 227, 227, True, False, out_dtype=torch.bfloat16, random_erasing=cfg)
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
    """One launch for the crop path (two with colour jitter's crop mean), plus one erase launch with the key; none on val batches."""
    from theanompi_b200.models.data.imagenet import ImageNet_data
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.ops import native
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    counts = {}
    cj = check_color_jitter(ALL4)
    for name, kw in (("off", {}), ("on", dict(random_erasing=RE)), ("rrc", dict(resized_crop=check_resized_crop({}), random_erasing=RE)),
                     ("color", dict(color_jitter=cj, random_erasing=RE))):
        ld = ParaLoader(d.read, "cuda:0", (16, H, W, 3), (224, 224), mean=d.rawdata[4], threaded=False, **kw)
        for mode in ("train", "val"):
            torch.cuda.synchronize()
            native.reset_launch_count()
            ld.request(d.train_img[0], mode)
            ld.get()
            torch.cuda.synchronize()
            counts[name, mode] = native.launch_count()
        ld.close()
    assert counts == {("off", "train"): 1, ("off", "val"): 1, ("on", "train"): 2, ("on", "val"): 1, ("rrc", "train"): 2,
                      ("rrc", "val"): 1, ("color", "train"): 3, ("color", "val"): 1}, counts


# --------------------------------------------------------------------------- models
def _model(cls_path, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    mod, cls = cls_path.rsplit(".", 1)
    return getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", n_class=100,
                                                            data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True), **cfg))


@pytest.mark.parametrize("name,cls,extra", [
    ("alexnet", "theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64, random_erasing={"p": 0.5})),
    ("resnet50", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50",
     dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 1, 1), random_resized_crop={"seed": 1}, color_jitter=ALL4,
          random_erasing={"p": 0.25}))])
def test_models_train_with_the_key_under_the_cuda_graph(name, cls, extra):
    from theanompi_b200.utils.recorder import Recorder
    m = _model(cls, cuda_graph=True, **extra)
    try:
        assert m.data.loader is not None and m.data.loader.random_erasing is not None
        rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
        m.compile_iter_fns("avg")
        m.reset_iter("train")
        costs = []
        for i in range(4):
            m.train_iter(i, rec)
            torch.cuda.synchronize()
            costs.append(float(rec.train_info["cost"][-1]))
        m.reset_iter("train")
        m.reset_iter("val")
        m.val_iter(0, rec)
        torch.cuda.synchronize()
        assert "step" in m.captured_steps(), "the step was not captured"
        assert all(np.isfinite(costs)) and np.isfinite(float(rec.val_info["cost"][-1])), costs
    finally:
        m.cleanup()


def test_the_key_does_not_change_the_step_launches():
    """The erase kernel runs on the loader's copy stream, outside the step: AlexNet's training step launches what it launches
    without the key."""
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    for name, extra in (("off", {}), ("on", dict(random_erasing={"p": 1.0}))):
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
