"""AutoAugment, AugMix and bilinear geometry on the H100, against the in-repo torch reference (``reference.aa_apply_op``,
``augmix_mix``, ``auto_augment_crop_normalize``; itself checked against torchvision in tests/test_augmix_cpu.py): the Invert LUT, the
bilinear apply, the mix kernel, whole batches of every policy, the loaders, the launch counts, native models training under the CUDA
graph, unchanged validation and determinism.

Bilinear bound.  ``aa_apply_kernel<true>`` evaluates the fp32 expressions of torchvision's CPU path in the same order: the rescaled
matrix (one division each), the grid as the CPU bmm rounds it (bx·t0 rounded, fused into by·t1, then + t2), grid_sample's
unnormalize (g + 1)·(size/2) − ½, the tap weights and the left-to-right sum of the four products.  The only freedom left is the bmm's
rounding on another CPU, which moves a coordinate by an ulp and the interpolated value by less than 255·4·2⁻¹⁵ ≈ 0.03; after the round
half to even that is at most one level, at elements within 0.03 of a half, so the tie rule (one level, fewer than 1e-3 of the
elements) is the bound.  The Invert LUT, the mix (the same fp32 multiplies and adds, then truncation) and a "trivial_wide" config
without ``interpolation`` are held bit for bit.

Full-pipeline bound: as tests/test_gpu_auto_augment.py, |got − want| ≤ (|u'| + |m̂|)·s_c·6·2⁻²⁴ (+ 2⁻⁸·|want| in bf16) where u'
agrees; AugMix's u' is the truncated mix of chains that agree under the tie rule, so it agrees except at those elements.
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
from test_gpu_auto_augment import STD, H, W, _fixed, _inputs, _model  # noqa: E402
from theanompi_b200.models.data.utils import (AA_INVERT, AA_LUT_OPS, AA_NONE, aa_compose_records, aa_slots, augmix_records,  # noqa: E402
                                              auto_augment_records, auto_augment_rng, check_auto_augment)
from theanompi_b200.ops import reference as ref  # noqa: E402

POLICIES = [{"policy": "trivial_wide"}, {"policy": "rand"}, {"policy": "autoaugment"}, {"policy": "augmix"},
            {"policy": "trivial_wide", "interpolation": "bilinear"}, {"policy": "augmix", "chain_depth": 1, "all_ops": False}]


def _apply_all(u, rec, bilinear):
    from theanompi_b200.ops import cuda_impl
    ud, rd = u.cuda(), torch.from_numpy(np.ascontiguousarray(rec)).cuda()
    return cuda_impl.aa_apply(ud, rd, 0, cuda_impl.aa_lut(ud, rd, 0), bilinear=bilinear).cpu()


def _ref_all(u, rec):
    return torch.stack([ref.aa_apply_op(u[i].permute(2, 0, 1), rec[i, 0]).permute(1, 2, 0) for i in range(len(u))])


def test_invert_lut_is_bit_for_bit():
    N, hw = 16, (227, 227)
    u = torch.randint(0, 256, (N,) + hw + (3,), dtype=torch.uint8, generator=torch.Generator().manual_seed(0))
    rec = aa_compose_records(np.full((N, 1), AA_INVERT), np.zeros((N, 1)), hw)
    got = _apply_all(u, rec, False)
    assert torch.equal(got, 255 - u) and torch.equal(got, _ref_all(u, rec))


@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227)])
@pytest.mark.parametrize("op", [1, 2, 3, 4, 5])
def test_bilinear_geometry_matches_the_reference(op, out_hw):
    N = 24
    g = torch.Generator().manual_seed(op)
    u = torch.randint(0, 256, (N,) + out_hw + (3,), dtype=torch.uint8, generator=g)
    cfg = check_auto_augment({"policy": "augmix", "severity": 10})
    rng = np.random.default_rng(op)
    space = {1: 0.3, 2: 0.3, 3: out_hw[1] / 3.0, 4: out_hw[0] / 3.0, 5: 30.0}[op]
    mag = rng.uniform(-space, space, (N, 1))
    rec = aa_compose_records(np.full((N, 1), op), mag, out_hw, bilinear=True)
    assert cfg["interpolation"] == "bilinear" and np.all(rec[..., 3] == 1)
    got, want = _apply_all(u, rec, True), _ref_all(u, rec)
    assert_tie_rule(got.numpy(), want.numpy(), "bilinear op %d" % op, level=1)
    # the nearest path of the same records is untouched by the flag in field 3
    rec[..., 3] = 0
    assert_tie_rule(_apply_all(u, rec, False).numpy(), _ref_all(u, rec).numpy(), "nearest op %d" % op, level=None)


def test_augmix_mix_is_bit_for_bit():
    from theanompi_b200.ops import cuda_impl
    N, hw, width = 32, (224, 224), 3
    cfg = check_auto_augment({"policy": "augmix", "seed": 1})
    rec, wts, op, _ = augmix_records(N, cfg, auto_augment_rng(cfg, 0), hw)
    g = torch.Generator().manual_seed(5)
    u = torch.randint(0, 256, (N,) + hw + (3,), dtype=torch.uint8, generator=g)
    chains = torch.randint(0, 256, (width, 2, N) + hw + (3,), dtype=torch.uint8, generator=g)
    got = cuda_impl.aa_mix(u.cuda(), chains.cuda(), torch.from_numpy(rec).cuda(), torch.from_numpy(wts).cuda()).cpu()
    depth = (op.reshape(N, width, 3) != AA_NONE).sum(2)
    for n in range(N):
        want = ref.augmix_mix(u[n], [chains[i, (depth[n, i] - 1) % 2, n] for i in range(width)], wts[n])
        assert torch.equal(got[n], want), n


def _case(cfg, out_hw, dtype, N=16, seed=0):
    from theanompi_b200.models.data.utils import draw_resized_crops, resized_crop_rng, check_resized_crop
    from theanompi_b200.ops import cuda_impl
    x = _inputs(N, seed)
    mean = torch.rand(H, W, 3, generator=torch.Generator().manual_seed(seed + 1)) * 255
    c = check_resized_crop({"seed": seed})
    boxes, flips = draw_resized_crops(N, (H, W), c["scale"], c["ratio"], resized_crop_rng(c, 0))
    boxes[: N // 2] = _fixed(out_hw, N // 2, seed)
    cfg = check_auto_augment(dict(cfg, seed=seed))
    wts = None
    if cfg["policy"] == "augmix":
        rec, wts, ops, _ = augmix_records(N, cfg, auto_augment_rng(cfg, 0), out_hw)
    else:
        rec, ops, _ = auto_augment_records(N, cfg, auto_augment_rng(cfg, 0), out_hw)
    cs = torch.from_numpy(1.0 / 255.0 / STD)
    got = cuda_impl.auto_augment_crop_normalize(x.cuda(), mean.cuda(), cs.cuda(), out_hw, torch.from_numpy(boxes).cuda(),
                                                torch.from_numpy(flips).cuda(), torch.from_numpy(rec).cuda(), ops, dtype,
                                                weights=None if wts is None else torch.from_numpy(wts).cuda())
    want = ref.auto_augment_crop_normalize(x, mean, cs, out_hw, boxes, flips, rec, weights=wts)
    return got.float().cpu(), want, cs


@pytest.mark.parametrize("cfg", POLICIES, ids=lambda c: "-".join(str(v) for v in c.values()))
@pytest.mark.parametrize("out_hw", [(224, 224), (227, 227)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_whole_batches_match_the_reference(cfg, out_hw, dtype):
    got, want, cs = _case(cfg, out_hw, dtype)
    bound = 6 * 2.0 ** -24 * 2 * 255 * float(cs.max()) + (2.0 ** -8 * want.abs() if dtype == torch.bfloat16 else 0)
    off = (got - want).abs() > bound
    assert off.float().mean() < 1e-3, "%d of %d elements outside the bound" % (int(off.sum()), off.numel())


def test_trivial_wide_without_interpolation_is_bit_for_bit_the_nearest_config():
    a, _, _ = _case({"policy": "trivial_wide"}, (224, 224), torch.float32, seed=3)
    b, _, _ = _case({"policy": "trivial_wide", "interpolation": "nearest"}, (224, 224), torch.float32, seed=3)
    assert torch.equal(a, b)


def _launches(cfg, ops):
    """The documented launches of one training batch: 1 crop + Σ over slots (a LUT when a point op is drawn, an apply when any image's
    op is not AA_NONE) + 1 mix ("augmix") + 1 normalisation."""
    per = sum(int(any(o in AA_LUT_OPS for o in ops[:, s])) + int(any(o != AA_NONE for o in ops[:, s])) for s in range(ops.shape[1]))
    return 1 + per + (cfg["policy"] == "augmix") + 1


def test_launches_per_training_batch():
    from theanompi_b200.models.data.imagenet import ImageNet_data
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.ops import native
    d = ImageNet_data(synthetic=True, n_train_files=3, n_val_files=1, file_batch_size=16)
    d.batch_data(16)
    for c in ({"policy": "autoaugment"}, {"policy": "augmix"}, {"policy": "augmix", "chain_depth": 1, "mixture_width": 2}):
        cfg = check_auto_augment(dict(c, seed=1))
        ld = ParaLoader(d.read, "cuda:0", (16, H, W, 3), (224, 224), mean=d.rawdata[4], threaded=False, auto_augment=cfg)
        torch.cuda.synchronize()
        native.reset_launch_count()
        ld.request(d.train_img[0], "train")
        b = ld.get()
        torch.cuda.synchronize()
        ops = b.aa_records[..., 0].astype(int)
        assert ops.shape[1] == aa_slots(cfg)
        assert native.launch_count() == _launches(cfg, ops)
        if c.get("chain_depth") == 1:
            assert native.launch_count() <= 1 + 2 * 2 + 1 + 1            # the empty steps 2 and 3 of each chain launch nothing
        native.reset_launch_count()
        ld.request(d.train_img[0], "val")
        ld.get()
        torch.cuda.synchronize()
        assert native.launch_count() == 1
        ld.close()


def _loader(mode, files, cfg, **kw):
    from theanompi_b200.models.data.loader import ParaLoader
    from theanompi_b200.models.data.proc_loader import ProcReader
    if mode == "process":
        pr = ProcReader((16, H, W, 3), depth=2)
        return ParaLoader(pr.read, "cuda:0", (16, H, W, 3), (224, 224), host_buffers=pr.tensors, on_close=pr.close, auto_augment=cfg, **kw)
    return ParaLoader(lambda item, out: np.copyto(out, files[item]), "cuda:0", (16, H, W, 3), (224, 224), auto_augment=cfg, **kw)


def _files(tmp_path):
    files = {}
    for i in range(2):
        a = np.random.RandomState(i).randint(0, 256, (16, H, W, 3), dtype=np.uint8)
        files[str(tmp_path / ("b%d.npy" % i))] = a
        np.save(str(tmp_path / ("b%d.npy" % i)), a)
    return files


@pytest.mark.parametrize("policy", ["autoaugment", "augmix"])
@pytest.mark.parametrize("mode", ["thread", "process"])
def test_loaders_reproduce_the_reference_of_their_draw(tmp_path, mode, policy):
    files = _files(tmp_path)
    mean = np.random.RandomState(9).uniform(0, 255, (H, W, 3)).astype(np.float32)
    cfg = check_auto_augment({"policy": policy, "seed": 3})
    ld = _loader(mode, files, cfg, mean=mean, std_scale=1.0 / 255.0 / STD, out_dtype=torch.float32, rank=1)
    try:
        items = sorted(files)
        ld.request(items[0], "train")
        for k in range(1, 3):
            ld.request(items[k % 2], "train")
            b = ld.get()
            torch.cuda.synchronize()
            assert (b.aa_weights is not None) == (policy == "augmix")
            want = ref.auto_augment_crop_normalize(torch.from_numpy(files[b.item]), torch.from_numpy(mean),
                                                   torch.from_numpy(1.0 / 255.0 / STD), (224, 224), b.boxes, b.flips, b.aa_records,
                                                   weights=b.aa_weights)
            bound = 6 * 2.0 ** -24 * 2 * 255 / 255 / float(STD.min())
            off = (b.x.cpu() - want).abs() > bound
            assert off.float().mean() < 1e-3, int(off.sum())
        ld.drain()
    finally:
        ld.close()


def test_same_seed_same_batches_and_validation_is_unchanged(tmp_path):
    files = _files(tmp_path)
    items = sorted(files)
    outs = {}
    for name, cfg in (("a", check_auto_augment({"policy": "augmix", "seed": 8})), ("b", check_auto_augment({"policy": "augmix", "seed": 8})),
                      ("off", None)):
        ld = _loader("thread", files, cfg, mean=np.float32([120.0, 115.0, 100.0]), out_dtype=torch.bfloat16)
        try:
            got = []
            for mode in ("train", "val", "train"):
                ld.request(items[0], mode)
                got.append(ld.get().x.clone())
                torch.cuda.synchronize()
            ld.drain()
        finally:
            ld.close()
        outs[name] = got
    assert all(torch.equal(x, y) for x, y in zip(outs["a"], outs["b"]))
    assert torch.equal(outs["a"][1], outs["off"][1]) and not torch.equal(outs["a"][0], outs["off"][0])


@pytest.mark.parametrize("name,cls,extra", [
    ("alexnet", "theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64, auto_augment={"policy": "augmix"})),
    ("alexnet-serial", "theanompi_b200.models.alex_net.AlexNet",
     dict(batch_size=32, file_batch_size=32, no_paraload=True, auto_augment={"policy": "autoaugment"})),
    ("resnet50", "theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50",
     dict(batch_size=32, file_batch_size=32, blocks=(1, 1, 1, 1), random_resized_crop={"seed": 1}, auto_augment={"policy": "augmix"},
          random_erasing={}))])
def test_models_train_with_the_policies_under_the_cuda_graph(name, cls, extra):
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


def test_augmix_does_not_change_the_step_launches():
    from theanompi_b200.models import layers2
    from theanompi_b200.ops import native
    counts = {}
    for name, extra in (("off", {}), ("on", dict(auto_augment={"policy": "augmix"}))):
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
