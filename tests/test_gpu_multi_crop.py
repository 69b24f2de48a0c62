"""Ten-crop and mirrored validation (config['val_crops']) on the H100 (run with ``pytest -m gpu``): ``multi_crop_norm`` bit for bit
against the reference and against ``crop_mirror_norm`` with each view's offsets broadcast; the view-accumulate and metrics launches
against float64 with the per-element bounds of tests/layer_oracle.py; the thread, process and serial loaders; the models' multi-view
validation against the host average of single-view forwards; the training step's launches; and determinism.

Bounds of p̄ = (1/V)·Σ_v softmax(z_v) (fp32 accumulator, ``--use_fast_math``).  Per element and view, ``__expf(x)`` is within
(2 + 1.16·|x|) ulp of eˣ for x = z − max; the row sum se is an fp32 sum of C such terms (``red_rel(C)`` relative); the reciprocal, the
product, the V − 1 additions and the IEEE division by V add a few more roundings (``u`` = 2⁻²² with slack 8).  Results below FLT_MIN
flush to zero, hence an absolute 2⁻¹²⁶.  The cost of a row is −log max(p̄_y, FLT_MIN): its error is the relative error of p̄_y plus
that of ``__logf``.  A row's top-1 / top-5 flags are exact whenever p̄_y lies farther than the two elements' bounds from its first and
fifth competitors; the tests count the rows inside that band and require exact flags on tied rows (tied logits give bit-equal
probabilities in every view, so the rank rule decides them exactly)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import layer_oracle as lo
from theanompi_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
FLT_MIN = float(np.finfo(np.float32).tiny)


def _ci():
    from theanompi_b200.ops import cuda_impl
    return cuda_impl


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


# --------------------------------------------------------------------------- multi_crop_norm
@pytest.mark.parametrize("N", [1, 3, 128])
@pytest.mark.parametrize("V", [2, 10])
@pytest.mark.parametrize("out_dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("mean_mode", ["scalar", "pixel"])
@pytest.mark.parametrize("scale", ["scalar", "channel"])
def test_multi_crop_norm_is_bit_exact(N, V, out_dtype, mean_mode, scale):
    ci = _ci()
    g = _gen(N * 31 + V)
    H = W = 256
    ch = 227 if N != 3 else 224
    x = torch.randint(0, 256, (N, H, W, 3), device=DEV, generator=g, dtype=torch.uint8)
    mean = torch.full((1,), 127.5, device=DEV) if mean_mode == "scalar" else torch.rand((H, W, 3), device=DEV, generator=g) * 255
    sc = 1.0 / 255.0 if scale == "scalar" else torch.tensor([1 / 255 / 0.229, 1 / 255 / 0.224, 1 / 255 / 0.225], device=DEV)
    got = ci.multi_crop_normalize(x, mean, sc, (ch, ch), V, out_dtype)
    want = ref.multi_crop_normalize(x, mean, sc, (ch, ch), V, out_dtype)
    torch.cuda.synchronize()
    assert got.shape == (V, N, ch, ch, 3) and got.dtype == out_dtype
    assert torch.equal(got, want)
    for v, (y0, x0, m) in enumerate(ref.multi_crop_views((H, W), (ch, ch), V).tolist()):
        offs = torch.tensor([[y0, x0]], dtype=torch.int32, device=DEV).expand(N, 2)
        one = ci.crop_mirror_normalize(x, mean, sc, (ch, ch), offs, torch.full((N,), m, dtype=torch.uint8, device=DEV), out_dtype)
        assert torch.equal(got[v], one), v


def test_multi_crop_norm_refuses_bad_input():
    ci = _ci()
    x = torch.zeros((2, 256, 256, 3), dtype=torch.uint8, device=DEV)
    with pytest.raises(ValueError):
        ci.multi_crop_normalize(x, torch.zeros(1, device=DEV), 1.0, (227, 227), 3)
    with pytest.raises(ValueError):
        ci.multi_crop_normalize(x.float(), torch.zeros(1, device=DEV), 1.0, (227, 227), 2)
    with pytest.raises(ValueError):
        ci.multi_crop_normalize(x, torch.zeros(1, device=DEV), 1.0, (257, 227), 2)


# --------------------------------------------------------------------------- view_softmax_accum + metrics
def _view_logits(kind, V, B, C, g, dtype):
    """V views of [B, C] logits and labels (row 0 labelled 0, the last row C − 1).  ``ties``: every row has min(C, 8) columns at the
    same value in every view, the label among them; ``extreme``: logits spread over ±300, row 0's label at −10⁴ below the rest in
    every view so p̄_y underflows to the clamp."""
    lab = torch.randint(0, C, (B,), device=DEV, generator=g)
    if kind == "ties":
        m = min(C, 8)
        top = torch.rand(B, C, device=DEV, generator=g).argsort(1)[:, :m]
        lab = top.gather(1, torch.randint(0, m, (B, 1), device=DEV, generator=g))[:, 0]
        zs = []
        for _ in range(V):
            z = torch.randint(-8, -3, (B, C), device=DEV, generator=g).float()
            zs.append(z.scatter_(1, top, 3.0))
    else:
        s = 100.0 if kind == "extreme" else 3.0
        zs = [torch.randn((B, C), device=DEV, generator=g) * s for _ in range(V)]
    if kind != "ties":
        lab[0], lab[-1] = 0, C - 1
    if kind == "extreme":
        for z in zs:
            z[0, lab[0]] = z[0].max() - 1e4
    return [z.to(dtype) for z in zs], lab


def _pbar_bound(zs, pbar64):
    """Per-element bound of the kernel's p̄ (module docstring) and the float64 p̄."""
    V = len(zs)
    C = zs[0].shape[1]
    extra = torch.zeros_like(pbar64)
    for z in zs:
        z = z.double()
        x = z - z.max(1, keepdim=True).values
        extra += (2.0 + 1.16 * x.abs()) * 2.0 ** -23 * torch.softmax(z, 1) / V
    return extra + lo.red_rel(C) * pbar64 + 2.0 ** -126


def _assert_cost(cost, c64, pbar64, bound, lab, what):
    """The mean cost against float64: per row the relative bound of p̄_y (none where both sides clamp to FLT_MIN) plus the error of
    ``__logf``, then an fp32 mean of B terms."""
    py = pbar64.gather(1, lab[:, None])[:, 0]
    by = bound.gather(1, lab[:, None])[:, 0]
    nll64 = -py.clamp_min(FLT_MIN).log()
    rel = torch.where(py + by < FLT_MIN, torch.zeros_like(py), by / py.clamp_min(FLT_MIN)) + 8 * 2.0 ** -22
    lo.assert_reduction(torch.as_tensor(cost), c64, (nll64.abs() + 1).mean(), len(lab),
                        extra_abs=(rel + 2.0 ** -20 * (nll64.abs() + 1)).mean(), what=what)


@pytest.mark.parametrize("kind", ["normal", "ties", "extreme"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("V", [2, 10])
@pytest.mark.parametrize("C", [10, 1000, 21841])
@pytest.mark.parametrize("B", [1, 32, 128, 256])
def test_view_softmax_accum(B, C, V, dtype, kind):
    ci = _ci()
    g = _gen(B * 131 + C * 7 + V)
    zs, lab = _view_logits(kind, V, B, C, g, dtype)
    acc = torch.empty((B, C), dtype=torch.float32, device=DEV)
    rowstat = torch.empty((B, 3), dtype=torch.float32, device=DEV)
    outs = [ci.view_softmax_accum(z, lab, acc, v, V, rowstat=rowstat) for v, z in enumerate(zs)]
    torch.cuda.synchronize()
    assert all(o is None for o in outs[:-1])
    cost, e1, e5 = outs[-1]
    c64, _, _, pbar64 = ref.multi_view_xent(zs, lab)
    extra = _pbar_bound(zs, pbar64)
    lo.assert_elementwise(acc, pbar64, torch.float32, extra_abs=extra, slack=8, what="p̄")
    _assert_cost(cost, c64, pbar64, extra, lab, "cost")
    assert abs(float(rowstat[:, 0].double().mean()) - float(cost)) <= lo.red_rel(B) * float((rowstat[:, 0].abs() + 1).double().mean())
    # the flags: exact outside the band, exact on tied rows
    rank = lo.label_rank(pbar64, lab)
    near1, near5 = _near(pbar64, lab, extra + 8 * 2.0 ** -22 * pbar64)
    sure = ~(near1 | near5) if kind != "ties" else torch.ones(B, dtype=torch.bool, device=DEV)
    f1, f5 = rowstat[:, 1].bool(), rowstat[:, 2].bool()
    assert torch.equal(f1[sure], (rank >= 1)[sure]) and torch.equal(f5[sure], (rank >= 5)[sure])
    print("%s B=%d C=%d V=%d: %d of %d rows inside the bound of a competitor" % (kind, B, C, V, int((~sure).sum()), B))
    assert abs(float(e1) - float(f1.float().mean())) <= 2.0 ** -22 and abs(float(e5) - float(f5.float().mean())) <= 2.0 ** -22
    if kind == "extreme":
        assert float(rowstat[0, 0]) == pytest.approx(-np.log(FLT_MIN), rel=1e-6)


# --------------------------------------------------------------------------- loaders
def _data(n=16):
    from theanompi_b200.models.data.imagenet import ImageNet_data
    d = ImageNet_data(file_batch_size=n, n_train_files=3, n_val_files=2, synthetic=True)
    d.batch_data(n)
    return d


@pytest.mark.parametrize("mode", ["thread", "process"])
@pytest.mark.parametrize("V", [2, 10])
def test_loaders_cut_the_reference_views_and_keep_training_batches(mode, V):
    out = {}
    for vc in (1, V):
        d = _data()
        ld = d.para_load_init("cuda:0", 227, 227, True, False, out_dtype=torch.bfloat16, mode=mode, val_crops=vc)
        seq = []
        try:
            for item, m in ((d.train_img[0], "train"), (d.val_img[0], "val"), (d.train_img[1], "train"), (d.val_img[1], "val"),
                            (d.train_img[2], "train")):
                ld.request(item, m)
                b = ld.get()
                # the staged uint8 batch the views were cut from (the process loader's reader has its own synthetic pool)
                seq.append((m, ld.stage[b.slot].clone(), b.x.clone(), b.h2d_bytes))
            torch.cuda.synchronize()
        finally:
            d.para_load_close()
        out[vc] = (seq, d)
    for (m, raw, x, nb), (_, raw1, x1, nb1) in zip(out[V][0], out[1][0]):
        assert nb == nb1 and torch.equal(raw, raw1)
        if m == "train":
            assert torch.equal(x, x1)
            continue
        d = out[V][1]
        want = ref.multi_crop_normalize(raw.cpu(), torch.from_numpy(d.rawdata[4]), torch.from_numpy(1.0 / 255.0 / d.rawdata[5]),
                                        (227, 227), V, torch.bfloat16)
        assert x.shape == (V, 16, 227, 227, 3) and torch.equal(x.cpu(), want)
        assert torch.equal(x[0 if V == 2 else 4], x1), "the centre view is the single-crop validation batch"


# --------------------------------------------------------------------------- models
def _model(cls_path, **cfg):
    import importlib
    from theanompi_b200.models import layers2
    layers2.reseed(); layers2.Dropout.layers.clear(); layers2.Crop.layers.clear(); layers2.BatchNormal.layers.clear()
    np.random.seed(1234); torch.manual_seed(1234)
    mod, cls = cls_path.rsplit(".", 1)
    return getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0",
                                                            data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True), **cfg))


def _eval_flags(on):
    from theanompi_b200.models.layers2 import BatchNormal, Crop, Dropout
    if on:
        Dropout.SetDropoutOn(); Crop.SetRandCropOn(); BatchNormal.SetTrainOn()
    else:
        Dropout.SetDropoutOff(); Crop.SetRandCropOff(); BatchNormal.SetTrainOff()


def _val_against_single_views(m):
    """val_fn of a val_crops = V model on the first validation file, and the float64 average of its V single-view forwards."""
    m.compile_iter_fns("avg")
    m.reset_iter("val")
    m._load_file_batch("val", 0, m.data.val_img_shard, m.data.val_labels_shard, m.data.n_batch_val)
    B, V = m.batch_size, m.val_crops
    y = m.shared_y[:B]
    _eval_flags(False)
    try:
        cost, e1, e5 = (float(t) for t in m.val_fn(0))
        zs = []
        with torch.no_grad():
            for v in range(V):
                m.forward(m.val_x[v, :B])
                zs.append(m.output_layer.logits.clone())
    finally:
        _eval_flags(True)
    torch.cuda.synchronize()
    return cost, e1, e5, zs, y


def _near(pbar64, lab, bound):
    """Rows whose p̄_y lies within the bounds of its first or fifth competitor: the only rows whose flags may differ."""
    py = pbar64.gather(1, lab[:, None])[:, 0]
    by = bound.gather(1, lab[:, None])[:, 0]
    others = pbar64.scatter(1, lab[:, None], -1.0).sort(1, descending=True)
    ob = bound.gather(1, others.indices)
    k = min(5, pbar64.shape[1] - 1)
    near1 = (others.values[:, 0] - py).abs() <= ob[:, 0] + by
    near5 = (others.values[:, k - 1] - py).abs() <= ob[:, k - 1] + by
    return near1, near5


MODELS = {
    "alexnet_bf16": ("theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64, dtype="bf16")),
    "alexnet_tf32": ("theanompi_b200.models.alex_net.AlexNet", dict(batch_size=64, file_batch_size=64, dtype="tf32")),
    "googlenet": ("theanompi_b200.models.googlenet.GoogLeNet", dict(batch_size=32, file_batch_size=32, dtype="bf16")),
    "resnet50": ("theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50", dict(batch_size=32, file_batch_size=32, dtype="bf16"))}


def model_check(name):
    """val_crops = 10 validation of one model against the float64 average of its ten single-view forwards (run under
    TMPI_DETERMINISTIC=1, so the forwards repeat bit for bit)."""
    from theanompi_b200.ops import precision
    cls, extra = MODELS[name]
    old = precision.precision()
    m = _model(cls, val_crops=10, **extra)
    try:
        assert m.data.loader is not None and m.data.loader.val_crops == 10
        cost, e1, e5, zs, y = _val_against_single_views(m)
        c64, e164, e564, pbar64 = ref.multi_view_xent(zs, y)
        B = len(y)
        extra_b = _pbar_bound(zs, pbar64)
        _assert_cost(cost, c64, pbar64, extra_b, y, name + " cost")
        near1, near5 = _near(pbar64, y, extra_b + 8 * 2.0 ** -22 * pbar64)
        print(name, cost, float(c64), e1, float(e164), e5, float(e564), "rows inside the bound:", int(near1.sum()), int(near5.sum()))
        assert round(abs(e1 - float(e164)) * B) <= int(near1.sum()) and round(abs(e5 - float(e564)) * B) <= int(near5.sum())
    finally:
        m.cleanup()
        precision.set_precision(old)


def _subprocess(code, timeout=1500):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    print(r.stdout[-3000:])
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


def test_models_average_ten_single_view_forwards():
    _subprocess("import test_gpu_multi_crop as t\nfor n in t.MODELS:\n    t.model_check(n)\nprint('OK')\n")


def test_serial_path_matches_the_loader():
    cls = "theanompi_b200.models.alex_net.AlexNet"
    outs = []
    for serial in (False, True):
        m = _model(cls, val_crops=10, batch_size=32, file_batch_size=32, no_paraload=serial)
        try:
            m.compile_iter_fns("avg")
            m.reset_iter("val")
            m._load_file_batch("val", 0, m.data.val_img_shard, m.data.val_labels_shard, m.data.n_batch_val)
            torch.cuda.synchronize()
            outs.append(m.val_x[:, :32].clone())
        finally:
            m.cleanup()
    # the loader normalises in the fused kernel, the serial path in the reference: the same fp32 expression, then one bf16 rounding
    assert torch.equal(outs[0], outs[1])


def test_val_crops_1_is_the_model_without_the_key():
    cls = "theanompi_b200.models.alex_net.AlexNet"
    res = []
    for cfg in (dict(), dict(val_crops=1)):
        m = _model(cls, batch_size=32, file_batch_size=32, **cfg)
        try:
            m.compile_iter_fns("avg")
            m.reset_iter("val")
            m._load_file_batch("val", 0, m.data.val_img_shard, m.data.val_labels_shard, m.data.n_batch_val)
            _eval_flags(False)
            try:
                res.append([float(t) for t in m.val_fn(0)])
            finally:
                _eval_flags(True)
        finally:
            m.cleanup()
    assert res[0] == res[1]


def test_training_step_launches_do_not_change():
    from theanompi_b200.ops import native
    from theanompi_b200.utils.recorder import Recorder
    counts = []
    for cfg in (dict(), dict(val_crops=10)):
        m = _model("theanompi_b200.models.alex_net.AlexNet", batch_size=32, file_batch_size=32, **cfg)
        try:
            rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
            m.compile_iter_fns("avg")
            m.reset_iter("train")
            m.train_iter(0, rec)
            torch.cuda.synchronize()
            native.reset_launch_count()
            for i in range(1, 3):
                m.train_iter(i, rec)
            torch.cuda.synchronize()
            counts.append(native.launch_count())
        finally:
            m.cleanup()
    assert counts[0] == counts[1], counts


def test_resnet50_torch_matches_its_torch_reference():
    m = _model("theanompi_b200.models.lasagne_model_zoo.resnet50.ResNet50Torch", val_crops=10, batch_size=16, file_batch_size=16,
               blocks=(1, 1, 1, 1))
    try:
        m.compile_iter_fns("avg")
        m.reset_iter("val")
        m._load_file_batch("val", 0, m.data.val_img_shard, m.data.val_labels_shard, m.data.n_batch_val)
        cost, e1, e5 = (float(t) for t in m.val_fn(0))
        m.module.eval()
        with torch.no_grad():
            zs = [m.forward(m.val_x[v, :16]).float() for v in range(10)]
        m.module.train()
        c64, e164, e564, pbar64 = ref.multi_view_xent(zs, m.shared_y[:16])
        # fp32 softmax and sum against float64; the twin's bf16-autocast library convolutions may pick another algorithm per call
        assert abs(cost - float(c64)) <= 1e-3 * (1 + abs(float(c64)))
        assert abs(e1 - float(e164)) <= 1 / 16 and abs(e5 - float(e564)) <= 1 / 16
    finally:
        m.cleanup()


def validation_run(V):
    """Validation of a fresh val_crops = V AlexNet after two training steps from a reset device counter (used in a
    TMPI_DETERMINISTIC=1 subprocess)."""
    from theanompi_b200 import ops
    from theanompi_b200.utils.recorder import Recorder
    _ci()._STEP.clear()
    ops.seed_dropout(0x5EED)
    m = _model("theanompi_b200.models.alex_net.AlexNet", val_crops=V, batch_size=32, file_batch_size=32)
    try:
        rec = Recorder(None, 10 ** 6, "t", False, device="cuda:0")
        m.compile_iter_fns("avg")
        m.reset_iter("train")
        for i in range(2):
            m.train_iter(i, rec)
        m.reset_iter("train")
        m.reset_iter("val")
        m.val_iter(0, rec)
        torch.cuda.synchronize()
        return [float(rec.val_info[k][-1]) for k in ("cost", "error", "error_top5")]
    finally:
        m.cleanup()


def test_deterministic_runs_are_bit_equal():
    _subprocess("import test_gpu_multi_crop as t\na, b = t.validation_run(10), t.validation_run(10)\nprint(a, b)\n"
                "assert a == b and all(x == x for x in a)\nprint('OK')\n")
