"""TrivialAugmentWide / RandAugment on the H100, against the in-repo torch reference (``reference.aa_crop_u8``, ``aa_apply_op``,
``auto_augment_crop_normalize``) under the tie rule of tests/auto_augment_oracle.py: the uint8 crop, each op's LUT + apply kernels, the
full pipeline, the loaders, the launch counts and native models training under the CUDA graph.

Full-pipeline bound.  out = (u' − m̂)·s_c.  u' is an integer, equal to the reference's except at tie-rule elements; m̂ is the same
bilinear resample with the same taps, so it differs from the reference's F.interpolate by at most 4 roundings of a value ≤ 255
(4·2⁻²⁴·255); the subtraction and the product round once each.  So at an element where u' agrees |got − want| ≤ (|u'| + |m̂|)·s_c·6·2⁻²⁴
(+ 2⁻⁸·|want| for bf16); elsewhere the tie rule counts the element.
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

from auto_augment_oracle import assert_tie_rule  # noqa: E402
from theanompi_b200.models.data.utils import (AA_OPS, auto_augment_records, auto_augment_rng, check_auto_augment,  # noqa: E402
                                              check_random_erasing, check_resized_crop)
from theanompi_b200.ops import reference as ref  # noqa: E402

H = W = 256
STD = np.array([0.229, 0.224, 0.225], np.float32)


def _fixed(out_hw, N, seed):
    rs = np.random.RandomState(seed)
    oy, ox = rs.randint(0, H - out_hw[0] + 1, N), rs.randint(0, W - out_hw[1] + 1, N)
    return np.stack([oy, ox, np.full(N, out_hw[0]), np.full(N, out_hw[1])], 1).astype(np.int32)


def _inputs(N, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, generator=g)


@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227)])
def test_uint8_crop_matches_the_reference(out_hw):
    from theanompi_b200.ops import cuda_impl
    N = 32
    x = _inputs(N, 1)
    from theanompi_b200.models.data.utils import draw_resized_crops, resized_crop_rng
    c = check_resized_crop({"seed": 3})
    boxes = np.concatenate([_fixed(out_hw, N // 2, 2), draw_resized_crops(N // 2, (H, W), c["scale"], c["ratio"], resized_crop_rng(c, 0))[0]])
    flips = (np.arange(N) % 2).astype(np.uint8)
    got = cuda_impl.aa_crop_u8(x.cuda(), out_hw, torch.from_numpy(boxes).cuda(), torch.from_numpy(flips).cuda())
    want = ref.aa_crop_u8(x, out_hw, boxes, flips)
    assert torch.equal(got.cpu()[: N // 2], want[: N // 2])                      # fixed crops: an exact copy
    assert_tie_rule(got.cpu().numpy(), want.numpy(), "uint8 crop")


@pytest.mark.parametrize("op", range(14))
@pytest.mark.parametrize("policy", ["trivial_wide", "rand"])
def test_each_op_kernel_matches_the_reference(op, policy):
    from theanompi_b200.ops import cuda_impl
    N, hw = 24, (224, 224)
    cfg = check_auto_augment({"policy": policy, "seed": op} if policy == "trivial_wide" else {"policy": policy, "num_ops": 1, "seed": op})
    rec = np.zeros((0, 1, 12), np.float32)
    rng = auto_augment_rng(cfg, 0)
    while len(rec) < N:                                       # N records of this op, with their drawn magnitudes and signs
        r, o, _ = auto_augment_records(2048, cfg, rng, hw)
        rec = np.concatenate([rec, r[o[:, 0] == op]])
    rec = np.ascontiguousarray(rec[:N])
    g = torch.Generator().manual_seed(op)
    u = torch.randint(0, 256, (N,) + hw + (3,), dtype=torch.uint8, generator=g)
    u[0] = 77                                                 # a constant image (AutoContrast / Equalize's step == 0)
    u[1, ..., 0] = torch.where(torch.rand(hw, generator=g) < 0.999, 10, 200).to(torch.uint8)
    ud, rd = u.cuda(), torch.from_numpy(rec).cuda()
    lut = cuda_impl.aa_lut(ud, rd, 0)
    got = cuda_impl.aa_apply(ud, rd, 0, lut).cpu()
    want = torch.stack([ref.aa_apply_op(u[i].permute(2, 0, 1), rec[i, 0]).permute(1, 2, 0) for i in range(N)])
    if op in (0, 6, 10, 11, 12, 13):                          # Identity and the pure LUT ops: bit for bit
        assert torch.equal(got, want), AA_OPS[op]
    else:
        assert_tie_rule(got.numpy(), want.numpy(), AA_OPS[op], level=None if 1 <= op <= 5 else 1)


def _pipeline_case(policy, out_hw, resized, mean_mode, dtype, N=16, seed=0):
    from theanompi_b200.ops import cuda_impl
    x = _inputs(N, seed)
    g = torch.Generator().manual_seed(seed + 1)
    mean = {0: torch.tensor([127.5]), 1: torch.tensor([123.7, 116.3, 103.5]), 2: torch.rand(H, W, 3, generator=g) * 255}[mean_mode]
    if resized:
        c = check_resized_crop({"seed": seed})
        from theanompi_b200.models.data.utils import draw_resized_crops, resized_crop_rng
        boxes, flips = draw_resized_crops(N, (H, W), c["scale"], c["ratio"], resized_crop_rng(c, 0))
    else:
        boxes, flips = _fixed(out_hw, N, seed), (np.arange(N) % 2).astype(np.uint8)
    cfg = check_auto_augment({"policy": policy, "seed": seed})
    rec, ops, _ = auto_augment_records(N, cfg, auto_augment_rng(cfg, 0), out_hw)
    cs = torch.from_numpy(1.0 / 255.0 / STD)
    got = cuda_impl.auto_augment_crop_normalize(x.cuda(), mean.cuda(), cs.cuda(), out_hw, torch.from_numpy(boxes).cuda(),
                                                torch.from_numpy(flips).cuda(), torch.from_numpy(rec).cuda(), ops, dtype)
    want = ref.auto_augment_crop_normalize(x, mean, cs, out_hw, boxes, flips, rec)
    return got.float().cpu(), want, mean, cs


@pytest.mark.parametrize("policy", ["trivial_wide", "rand"])
@pytest.mark.parametrize("resized", [False, True])
@pytest.mark.parametrize("mean_mode", [0, 2])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_full_pipeline_matches_the_reference(policy, resized, mean_mode, dtype):
    got, want, mean, cs = _pipeline_case(policy, (224, 224), resized, mean_mode, dtype)
    bound = 6 * 2.0 ** -24 * 2 * 255 * float(cs.max()) + (2.0 ** -8 * want.abs() if dtype == torch.bfloat16 else 0)
    off = (got - want).abs() > bound
    assert off.float().mean() < 1e-3, "%d of %d elements outside the bound" % (int(off.sum()), off.numel())


def test_launches_per_training_batch():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.models.data.utils import AA_LUT_OPS
    from theanompi_b200.ops import native
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    for cfg, re in ((check_auto_augment({"seed": 1}), None), (check_auto_augment({"policy": "rand", "num_ops": 3, "seed": 2}),
                                                              check_random_erasing({}))):
        ld = ParaLoader(d.read, "cuda:0", (16, H, W, 3), (224, 224), mean=d.rawdata[4], threaded=False, auto_augment=cfg,
                        random_erasing=re)
        torch.cuda.synchronize()
        native.reset_launch_count()
        ld.request(d.train_img[0], "train")
        b = ld.get()
        torch.cuda.synchronize()
        ops = b.aa_records[..., 0].astype(int)
        want = 1 + sum(int(any(o in AA_LUT_OPS for o in ops[:, s])) + 1 for s in range(ops.shape[1])) + 1 + (re is not None)
        assert native.launch_count() == want
        native.reset_launch_count()
        ld.request(d.train_img[0], "val")
        ld.get()
        torch.cuda.synchronize()
        assert native.launch_count() == 1
        ld.close()


@pytest.mark.parametrize("mode", ["thread", "process"])
def test_loaders_reproduce_the_reference_of_their_draw(tmp_path, mode):
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.models.data.proc_loader import ProcReader
    files = {}
    for i in range(2):
        a = np.random.RandomState(i).randint(0, 256, (16, H, W, 3), dtype=np.uint8)
        files[str(tmp_path / ("b%d.npy" % i))] = a
        np.save(str(tmp_path / ("b%d.npy" % i)), a)
    mean = np.random.RandomState(9).uniform(0, 255, (H, W, 3)).astype(np.float32)
    cfg = check_auto_augment({"policy": "rand", "seed": 3})
    kw = dict(mean=mean, std_scale=1.0 / 255.0 / STD, out_dtype=torch.float32, rank=1, auto_augment=cfg)
    if mode == "process":
        pr = ProcReader((16, H, W, 3), depth=2)
        ld = ParaLoader(pr.read, "cuda:0", (16, H, W, 3), (224, 224), host_buffers=pr.tensors, on_close=pr.close, **kw)
    else:
        ld = ParaLoader(lambda item, out: np.copyto(out, files[item]), "cuda:0", (16, H, W, 3), (224, 224), **kw)
    try:
        items = sorted(files)
        ld.request(items[0], "train")
        for k in range(1, 3):
            ld.request(items[k % 2], "train")
            b = ld.get()
            torch.cuda.synchronize()
            want = ref.auto_augment_crop_normalize(torch.from_numpy(files[b.item]), torch.from_numpy(mean),
                                                   torch.from_numpy(1.0 / 255.0 / STD), (224, 224), b.boxes, b.flips, b.aa_records)
            bound = 6 * 2.0 ** -24 * 2 * 255 / 255 / float(STD.min())
            off = (b.x.cpu() - want).abs() > bound
            assert off.float().mean() < 1e-3, int(off.sum())
        ld.drain()
    finally:
        ld.close()


def _model(cls_path, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    mod, cls = cls_path.rsplit(".", 1)
    return getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", n_class=100,
                                                            data_kwargs=dict(n_train_files=4, n_val_files=1, synthetic=True), **cfg))


@pytest.mark.parametrize("name,cls,extra", [
    ("alexnet", "theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64, auto_augment={},
                                                              random_erasing={"p": 0.1})),
    ("resnet50", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50",
     dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 1, 1), random_resized_crop={"seed": 1}, auto_augment={"policy": "rand"},
          random_erasing={}))])
def test_models_train_with_the_keys_under_the_cuda_graph(name, cls, extra):
    from theanompi_b200.utils.recorder import Recorder
    m = _model(cls, cuda_graph=True, **extra)
    try:
        rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
        m.compile_iter_fns("avg")
        m.reset_iter("train")
        costs = []
        for i in range(4):
            m.train_iter(i, rec)
            torch.cuda.synchronize()
            costs.append(float(rec.train_info["cost"][-1]))
        assert "step" in m.captured_steps()
        assert all(np.isfinite(costs)), costs
    finally:
        m.cleanup()


def test_the_keys_do_not_change_the_step_launches():
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    for name, extra in (("off", {}), ("on", dict(auto_augment={}, random_erasing={}))):
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
