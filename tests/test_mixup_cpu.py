"""Mixup / CutMix (``config['mixup']``) on the CPU reference path: the distribution of ``reference.mix_draw`` over consecutive step
counter values (every check seeded), ``reference.mix_batch`` against explicit torch, the mixed soft-target ``reference.softmax_xent``
against fp64 ``F.cross_entropy`` with probability targets, the validation of the key and the refusals, training steps whose recorded
cost is torch's soft-target loss of the step's logits under the step's record while validation stays plain NLL, ``grad_accum``
micro-steps, and a two-rank gloo BSP run through the Rule API."""
import math
import os
import pickle
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from theanompi_b200 import ops  # noqa: E402
from theanompi_b200.models import layers2  # noqa: E402
from theanompi_b200.models.layers2 import Crop, Dropout  # noqa: E402
from theanompi_b200.ops import mixup  # noqa: E402
from theanompi_b200.ops import reference as ref  # noqa: E402
from theanompi_b200.utils.recorder import Recorder  # noqa: E402

N_STEPS = 20000


def _cfg(**kw):
    return mixup.check_config(kw)


def _draws(cfg, seed=0, rank=0, hw=(32, 32), start=0):
    return ref.mix_draw(cfg, seed, rank, np.arange(start, start + N_STEPS), hw)


# --------------------------------------------------------------------------- reference.mix_draw
@pytest.mark.parametrize("alpha", [0.2, 1.0, 4.0])
@pytest.mark.parametrize("kind", ["mixup", "cutmix"])
def test_lambda_is_beta_distributed(alpha, kind):
    from scipy import stats
    cfg = _cfg(alpha=alpha) if kind == "mixup" else _cfg(cutmix_alpha=alpha)
    r = _draws(cfg, seed=1234)
    assert (r["mode"] == (mixup.MIX_MIXUP if kind == "mixup" else mixup.MIX_CUTMIX)).all()
    p = stats.kstest(r["lam_raw"], stats.beta(alpha, alpha).cdf).pvalue
    assert p > 1e-3, p
    if kind == "mixup":
        assert np.array_equal(r["lam"], r["lam_raw"].astype(np.float32))


@pytest.mark.parametrize("cfg, p_none, p_cut", [
    (dict(alpha=1.0, prob=0.7), 0.3, 0.0),
    (dict(alpha=0.4, cutmix_alpha=1.0), 0.0, 0.5),
    (dict(alpha=0.4, cutmix_alpha=1.0, switch_prob=0.2, prob=0.6), 0.4, 0.6 * 0.2),
    (dict(cutmix_alpha=2.0, prob=0.9), 0.1, 0.9),
    (dict(alpha=1.0, prob=0.0), 1.0, 0.0),
])
def test_mode_frequencies(cfg, p_none, p_cut):
    r = _draws(_cfg(**cfg), seed=99)
    for mode, p in ((mixup.MIX_NONE, p_none), (mixup.MIX_CUTMIX, p_cut), (mixup.MIX_MIXUP, 1.0 - p_none - p_cut)):
        f = float((r["mode"] == mode).mean())
        sigma = math.sqrt(max(p * (1 - p), 1e-12) / N_STEPS)
        assert abs(f - p) <= 5 * sigma + 1e-12, (mode, f, p)
    none = r[r["mode"] == mixup.MIX_NONE]
    assert (none["lam"] == 1.0).all() and (none["lam_raw"] == 1.0).all() and (none["y1"] == 0).all()


@pytest.mark.parametrize("hw", [(32, 32), (28, 28), (227, 227), (7, 13)])
def test_cutmix_boxes(hw):
    H, W = hw
    r = _draws(_cfg(cutmix_alpha=1.0), seed=7, hw=hw)
    assert (r["mode"] == mixup.MIX_CUTMIX).all() and (r["H"] == H).all() and (r["W"] == W).all()
    assert ((0 <= r["cy"]) & (r["cy"] < H) & (0 <= r["cx"]) & (r["cx"] < W)).all()
    assert ((0 <= r["y0"]) & (r["y0"] <= r["y1"]) & (r["y1"] <= H)).all()
    assert ((0 <= r["x0"]) & (r["x0"] <= r["x1"]) & (r["x1"] <= W)).all()
    area = (r["y1"] - r["y0"]).astype(np.int64) * (r["x1"] - r["x0"])
    assert np.array_equal(r["lam"], (1.0 - area / float(H * W)).astype(np.float32))
    # the box is timm's rand_bbox of the raw λ and the centre
    cut = np.sqrt(1.0 - r["lam_raw"])
    ch, cw = (H * cut).astype(np.int64), (W * cut).astype(np.int64)
    assert np.array_equal(r["y0"], np.clip(r["cy"] - ch // 2, 0, H)) and np.array_equal(r["y1"], np.clip(r["cy"] + ch // 2, 0, H))
    assert np.array_equal(r["x0"], np.clip(r["cx"] - cw // 2, 0, W)) and np.array_equal(r["x1"], np.clip(r["cx"] + cw // 2, 0, W))
    # the centre is uniform over the grid
    assert abs(float(r["cy"].mean()) - (H - 1) / 2) < 5 * H / math.sqrt(12 * N_STEPS)


def test_streams_differ_by_rank_seed_and_step():
    cfg = _cfg(alpha=1.0)
    base = _draws(cfg)["lam_raw"]
    assert np.array_equal(base, _draws(cfg)["lam_raw"])                   # deterministic
    for other in (_draws(cfg, rank=1), _draws(cfg, seed=1), _draws(cfg, seed=2 ** 32)):
        assert (other["lam_raw"] != base).mean() > 0.99
    assert len(np.unique(base)) == N_STEPS
    one = ref.mix_draw(cfg, 0, 0, 17, (32, 32))
    assert one.shape == () and float(one["lam_raw"]) == base[17]


def test_record_layout():
    assert mixup.RECORD_BYTES == 64
    r = ref.mix_draw(_cfg(cutmix_alpha=1.0), 3, 0, np.arange(5), (32, 32))
    t = mixup.encode(r)
    assert t.dtype == torch.uint8 and t.numel() == 5 * 64
    assert np.array_equal(mixup.decode(t), r)
    b = t[64:128].numpy().tobytes()
    import struct
    mode, lam, lam_raw, cy, cx, y0, y1, x0, x1, H, W = struct.unpack("<ifdiiiiiiii", b[:48])
    assert (mode, lam_raw, cy, y1, W) == (int(r[1]["mode"]), float(r[1]["lam_raw"]), int(r[1]["cy"]), int(r[1]["y1"]), 32)


# --------------------------------------------------------------------------- reference.mix_batch
def _record(mode, lam=0.6, box=(3, 9, 2, 7), hw=(12, 10)):
    r = np.zeros((), dtype=mixup.RECORD)
    r["mode"], r["lam"], r["lam_raw"], r["H"], r["W"] = mode, lam, lam, hw[0], hw[1]
    r["y0"], r["y1"], r["x0"], r["x1"] = box
    return r


@pytest.mark.parametrize("B", [1, 2, 37])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_mix_batch_matches_explicit_torch(B, dtype):
    g = torch.Generator().manual_seed(B)
    x = (torch.randn(B, 12, 10, 3, generator=g) * 4).to(dtype)
    lam = np.float32(0.3719)
    out = ref.mix_batch(x, _record(mixup.MIX_MIXUP, lam))
    l32 = torch.tensor(float(lam))
    want = (l32 * x.float() + (1 - l32) * x.float().flip(0)).to(dtype)
    assert torch.equal(out, want)
    if B % 2:
        m = B // 2
        assert (out[m].float() - x[m].float()).abs().max() <= 1e-6 * x[m].float().abs().max() + (0.02 if dtype == torch.bfloat16 else 0)
    out = ref.mix_batch(x, _record(mixup.MIX_CUTMIX, box=(3, 9, 2, 7)))
    want = x.clone()
    for i in range(B):
        want[i, 3:9, 2:7, :] = x[B - 1 - i, 3:9, 2:7, :]
    assert torch.equal(out, want)
    assert torch.equal(ref.mix_batch(x, _record(mixup.MIX_NONE)), x)
    y = x.clone()
    assert ops.mix_batch(y, mixup.encode(_record(mixup.MIX_CUTMIX))) is y and torch.equal(y, want)     # in place


# --------------------------------------------------------------------------- reference.softmax_xent(mix=)
def _oracle(lg, y, lam, eps, weight=1.0, grad_scale=1.0):
    C = lg.shape[1]
    x = lg.double().clone().requires_grad_(True)

    def soft(t):
        return (1 - eps) * F.one_hot(t, C).double() + eps / C
    q = lam * soft(y) + (1 - lam) * soft(y.flip(0))
    loss = weight * F.cross_entropy(x, q)
    loss.backward()
    return float(loss.detach()), x.grad * grad_scale


@pytest.mark.parametrize("C", [2, 10, 1000])
@pytest.mark.parametrize("B", [23, 24])
@pytest.mark.parametrize("eps", [0.0, 0.1])
@pytest.mark.parametrize("mode, lam", [(mixup.MIX_MIXUP, 0.37), (mixup.MIX_CUTMIX, 0.8125), (mixup.MIX_NONE, 1.0)])
def test_mixed_softmax_matches_torch_cross_entropy(mode, lam, eps, B, C):
    g = torch.Generator().manual_seed(B * C)
    lg = torch.randn(B, C, generator=g, dtype=torch.float64) * 3
    y = torch.randint(0, C, (B,), generator=g)
    rec = mixup.encode(_record(mode, np.float32(lam)))
    weight, grad_scale = 0.3, 0.25
    loss, e1, e5, dl = ref.softmax_xent(lg, y, grad_scale=grad_scale, weight=weight, label_smoothing=eps, mix=rec)
    want, dwant = _oracle(lg, y, float(np.float32(lam)), eps, weight, grad_scale)
    assert abs(float(loss) - want) < 1e-5 * max(1.0, abs(want)), (float(loss), want)
    assert float((dl.double() - dwant).abs().max()) < 1e-6 * float(dwant.abs().max()) + 1e-9
    ye = y if lam >= 0.5 else y.flip(0)                                    # the larger-weight label
    _, e1_0, e5_0, _ = ref.softmax_xent(lg, ye)
    assert float(e1) == float(e1_0) and float(e5) == float(e5_0)


def test_errors_follow_the_larger_weight():
    lg = torch.tensor([[5.0, 0.0, 0.0], [0.0, 5.0, 0.0]])
    y = torch.tensor([0, 2])
    for lam, want in ((0.5, 0.5), (0.75, 0.5), (0.25, 1.0)):
        _, e1, _, _ = ref.softmax_xent(lg, y, mix=mixup.encode(_record(mixup.MIX_MIXUP, lam)))
        assert float(e1) == want
    y = torch.tensor([0, 1])
    assert float(ref.softmax_xent(lg, y, mix=mixup.encode(_record(mixup.MIX_MIXUP, 0.5)))[1]) == 0.0     # y_i at λ = ½
    assert float(ref.softmax_xent(lg, y, mix=mixup.encode(_record(mixup.MIX_MIXUP, 0.49)))[1]) == 1.0    # y_j below it


def test_functional_node_and_softmax_cache_carry_the_record():
    g = torch.Generator().manual_seed(3)
    lg = torch.randn(8, 10, generator=g).requires_grad_(True)
    y = torch.randint(0, 10, (8,), generator=g)
    rec = mixup.encode(_record(mixup.MIX_MIXUP, np.float32(0.3)))
    loss, _, _ = ops.softmax_xent(lg, y, 0.1, rec)
    loss.backward()
    want, dwant = _oracle(lg.detach(), y, float(np.float32(0.3)), 0.1)
    assert abs(float(loss.detach()) - want) < 1e-5 and float((lg.grad.double() - dwant).abs().max()) < 1e-6
    layers2.reseed()
    sm = layers2.Softmax(None, 10, input_shape=(8, 16), printinfo=False)
    sm.forward(torch.randn(8, 16))
    plain = float(sm.negative_log_likelihood(y))
    mixed = float(sm.negative_log_likelihood(y, 0.0, rec))
    assert mixed != plain and float(sm.negative_log_likelihood(y)) == plain
    sm.negative_log_likelihood(y, 0.0, rec)
    assert float(sm.errors(y)) == float(ref.softmax_xent(sm.logits, y.flip(0))[1])       # the errors reuse the mixed launch


# --------------------------------------------------------------------------- configuration
def _cifar(**kw):
    from theanompi_b200.models.cifar10 import Cifar10_model
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    cfg = dict(verbose=False, rank=0, size=1, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.05,
               data_kwargs=dict(n_synthetic=640, synthetic=True))
    cfg.update(kw)
    m = Cifar10_model(cfg)
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    return m


@pytest.fixture(autouse=True)
def dropout_back_on():
    yield
    Dropout.SetDropoutOn(); Crop.SetRandCropOn()


@pytest.mark.parametrize("bad, key", [
    (0.5, "mixup"), ([1.0], "mixup"), ("alpha", "mixup"), (True, "mixup"),
    (dict(beta=1.0), "beta"), (dict(alpha=1.0, pair=True), "pair"), (dict(), "alpha"), (dict(alpha=0, cutmix_alpha=0), "alpha"),
    (dict(alpha=-0.1), "alpha"), (dict(cutmix_alpha=-1), "cutmix_alpha"), (dict(alpha=16.5), "alpha"), (dict(cutmix_alpha=17), "cutmix_alpha"),
    (dict(alpha=float("nan")), "alpha"), (dict(alpha=float("inf")), "alpha"), (dict(alpha=True), "alpha"), (dict(alpha="1"), "alpha"),
    (dict(alpha=1.0, prob=1.5), "prob"), (dict(alpha=1.0, prob=-0.1), "prob"), (dict(alpha=1.0, prob=float("nan")), "prob"),
    (dict(alpha=1.0, prob=False), "prob"), (dict(alpha=1.0, switch_prob=2.0), "switch_prob"),
    (dict(alpha=1.0, switch_prob=None), "switch_prob"), (dict(alpha=1.0, seed=1.5), "seed"), (dict(alpha=1.0, seed="0"), "seed"),
    (dict(alpha=1.0, seed=True), "seed"), (dict(alpha=1.0, seed=np.float64(2)), "seed"),
])
def test_invalid_values_are_refused(bad, key):
    m = _cifar(mixup=bad)
    with pytest.raises(ValueError, match=key):
        m.compile_iter_fns("avg")


@pytest.mark.parametrize("good", [dict(alpha=0.2), dict(cutmix_alpha=1), dict(alpha=16, cutmix_alpha=0.5, switch_prob=1, prob=0),
                                  dict(alpha=np.float32(0.4), seed=np.int64(7)), dict(alpha=1.0, seed=-3)])
def test_valid_values_are_accepted(good):
    m = _cifar(mixup=good)
    m.compile_iter_fns("avg")
    assert m.mixer is not None and m.mixer.cfg["alpha"] == float(good.get("alpha", 0)) and (m.mixer.H, m.mixer.W) == (28, 28)


def _refused_models():
    from theanompi_b200.models.alex_net_sc_outdated import AlexNet_sc
    from theanompi_b200.models.lasagne_model_zoo.lsgan import LSGAN, NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50Torch
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN, WGAN
    from theanompi_b200.models.lstm import LSTM, LSTMTorch
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNetTorch
    img = dict(batch_size=4, file_batch_size=4, n_class=8, no_paraload=True, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))
    return [(NativeWGAN, dict(data_kwargs=dict(n_synthetic=128))), (NativeLSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (WGAN, dict(data_kwargs=dict(n_synthetic=128))), (LSGAN, dict(data_kwargs=dict(n_synthetic=128))),
            (LSTM, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (LSTMTorch, dict(dim_proj=16, data_kwargs=dict(n_synthetic=64, n_words=200))),
            (ResNet50Torch, dict(img, blocks=(1, 1, 1, 1))),
            (Wide_ResNetTorch, dict(batch_size=8, file_batch_size=8, depth=10, widen=1, data_kwargs=dict(n_synthetic=64, synthetic=True))),
            (AlexNet_sc, img)]


def test_unsupported_models_refuse_mixup():
    for cls, kw in _refused_models():
        assert cls.supports_mixup is False, cls
        layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", mixup=dict(alpha=0.2), **kw))
        with pytest.raises(ValueError, match="mixup is not supported.*AlexNet, GoogLeNet, Cifar10_model, VGG16, ResNet50 and Wide_ResNet"):
            m.compile_iter_fns("avg")
        m = cls(dict(verbose=False, rank=0, size=1, device="cpu", mixup=None, **kw))
        m.compile_iter_fns("avg")
        assert m.mixer is None


def _train(m, n, rec):
    for i in range(n):
        m.train_iter(i, rec)


def test_none_is_an_absent_key():
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    a, b = _cifar(), _cifar(mixup=None)
    a.compile_iter_fns("avg"); b.compile_iter_fns("avg")
    assert a.mixer is None and b.mixer is None
    _train(a, 4, rec); _train(b, 4, rec)
    assert torch.equal(a.arena.W, b.arena.W) and torch.equal(a.arena.U, b.arena.U)


# --------------------------------------------------------------------------- training steps
def _mixed_loss(lg, y, rec, eps=0.0):
    """torch's soft-target cross-entropy (fp64) of the logits ``lg`` against the target of the record ``rec``."""
    lam = ref.mix_lambda(rec)
    C = lg.shape[1]

    def soft(t):
        return (1 - eps) * F.one_hot(t, C).double() + eps / C
    return float(F.cross_entropy(lg.double(), lam * soft(y) + (1 - lam) * soft(y.flip(0))))


def _step(m, step):
    """One training step of ``m``: (recorded cost, the step's logits, labels, mix record, the batch that entered the forward)."""
    seen = {}
    fwd, mix_input = m.forward, m.mix_input

    def spy(x):
        seen["x"] = x.detach().clone()
        out = fwd(x)
        seen["logits"] = out.detach().double().clone()
        return out

    def spy_mix(rec):
        seen["before"] = m.x_in.clone()
        mix_input(rec)
    m.forward, m.mix_input = spy, spy_mix
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.train_iter(step, rec)
    del m.forward, m.mix_input
    return (float(rec.train_info["cost"][-1]), seen["logits"], m.y_in.clone(), m.mixer.rec.clone(), seen["x"], seen["before"])


def _check_steps(m, n, eps=0.0, input_mixed=True):
    modes = set()
    for i in range(n):
        cost, lg, y, rec, x, src = _step(m, i)
        modes.add(int(mixup.decode(rec)["mode"]))
        assert abs(cost - _mixed_loss(lg, y, rec, eps)) < 1e-4 * max(1.0, cost), i
        if int(mixup.decode(rec)["mode"]):
            assert abs(cost - float(F.cross_entropy(lg, y))) > 1e-6, i
        if input_mixed:                                 # x_in is the mix point: the forward saw the mixed batch, shared_x unchanged
            assert torch.equal(x, ref.mix_batch(src, rec)), i
            B = m.batch_size
            assert any(torch.equal(m.shared_x[k * B:(k + 1) * B], src) for k in range(m.n_subb)) and not torch.equal(x, src)
    return modes


def test_cifar_steps_record_the_mixed_loss_and_validate_without_it():
    m = _cifar(mixup=dict(alpha=1.0, cutmix_alpha=1.0, seed=5))
    m.compile_iter_fns("avg")
    Crop.SetRandCropOn()                                          # the mix point is the random crop's output
    seen = {}
    mb = ops.mix_batch

    def spy(x, rec):
        seen["crop"] = x.clone()
        out = mb(x, rec)
        assert torch.equal(out, ref.mix_batch(seen["crop"], rec))
        return out
    import theanompi_b200.models.cifar10 as cm
    cm.ops.mix_batch = spy
    try:
        modes = _check_steps(m, 6, input_mixed=False)
    finally:
        cm.ops.mix_batch = mb
    assert seen["crop"].shape[1:3] == (28, 28) and modes == {1, 2}
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.reset_iter("val")
    got = {}
    fwd = m.forward
    m.forward = lambda x: got.setdefault("lg", fwd(x))
    m.val_iter(0, rec)
    m.forward = fwd
    assert abs(float(rec.val_info["cost"][-1]) - float(F.cross_entropy(got["lg"].detach().double(), m.shared_y[:m.batch_size]))) < 1e-5


def test_small_alexnet_steps_with_label_smoothing():
    from theanompi_b200.models.alex_net import AlexNet
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, n_class=16, no_paraload=True,
                     learning_rate=0.001, label_smoothing=0.1, mixup=dict(alpha=0.4, cutmix_alpha=1.0, seed=3),
                     data_kwargs=dict(n_train_files=3, n_val_files=1, synthetic=True)))
    m.compile_iter_fns("avg")
    Dropout.SetDropoutOff()
    _check_steps(m, 3, eps=0.1)


def test_wide_resnet_adam_steps():
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    m = Wide_ResNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=8, file_batch_size=16, depth=10, widen=1,
                         mixup=dict(cutmix_alpha=1.0, seed=11), data_kwargs=dict(n_synthetic=64, synthetic=True)))
    m.compile_iter_fns("avg")
    assert _check_steps(m, 3) == {2}


def test_googlenet_aux_heads_use_the_same_target():
    from theanompi_b200.models.googlenet import GoogLeNet
    layers2.reseed(); Dropout.layers.clear(); Crop.layers.clear()
    m = GoogLeNet(dict(verbose=False, rank=0, size=1, device="cpu", batch_size=4, file_batch_size=4, n_class=8, no_paraload=True,
                       mixup=dict(alpha=1.0, seed=2), data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))
    m.compile_iter_fns("avg")
    Dropout.SetDropoutOn()
    heads = [m.output_layer, m.aux1.softmax_layer, m.aux2.softmax_layer]
    rec = Recorder(None, 10 ** 6, "c", False, device="cpu")
    m.train_iter(0, rec)
    r = m.mixer.rec
    assert int(mixup.decode(r)["mode"]) == mixup.MIX_MIXUP
    parts = [_mixed_loss(h.logits.detach(), m.y_in, r) for h in heads]
    want = parts[0] + 0.3 * parts[1] + 0.3 * parts[2]
    assert abs(float(rec.train_info["cost"][-1]) - want) < 1e-4 * max(1.0, want)
    for h in heads:                                                       # every head's cached launch is the mixed one
        assert h._cache[2] is r


def test_grad_accum_micro_steps_draw_their_own_records():
    m = _cifar(batch_size=8, grad_accum=2, mixup=dict(alpha=1.0))
    m.compile_iter_fns("avg")
    lams = []
    for i in range(4):
        cost, lg, y, rec, _, _ = _step(m, i)
        assert abs(cost - _mixed_loss(lg, y, rec)) < 1e-5, i
        lams.append(float(mixup.decode(rec)["lam_raw"]))
    assert len(set(lams)) == 4, lams
    assert m.n_updates == 2


# --------------------------------------------------------------------------- distributed
def test_rule_bsp_cdd_two_gloo_ranks(tmp_path, monkeypatch):
    """BSP sync_type='cdd' over the split 'ar' strategy with mixup in rule.model_config: the key reaches both workers (an invalid
    value stops them at compile_iter_fns) and the run completes with finite mixed training costs recorded."""
    import subprocess
    import theanompi_b200 as tm
    monkeypatch.chdir(tmp_path)
    tm.BSP.sync_type, tm.BSP.exch_strategy = "cdd", "ar"
    rcs = {}
    for name, mx in (("good", dict(alpha=0.2, cutmix_alpha=1.0, seed=1)), ("bad", dict(alpha=0.2, beta=1.0))):
        rule = tm.BSP()
        rule.model_config = dict(batch_size=16, file_batch_size=16, n_epochs=1, learning_rate=0.01, max_batches=6, printFreq=4,
                                 mixup=mx, data_kwargs=dict(n_synthetic=320, synthetic=True))
        rule.env["OMP_NUM_THREADS"] = "2"
        rule.init(devices=["cpu0", "cpu1"], modelfile="theanompi_b200.models.cifar10", modelclass="Cifar10_model")
        try:
            rcs[name] = rule.proc.wait(timeout=300)
        except subprocess.TimeoutExpired:
            rule.proc.kill()
            raise
        if name == "good":
            with open(tmp_path / "inforec" / "inforec.pkl", "rb") as f:
                costs = [c for _, c, _ in pickle.load(f)["train_info"]]
            assert costs and all(math.isfinite(c) and c > 0 for c in costs), costs
    assert rcs["good"] == 0 and rcs["bad"] != 0, rcs
