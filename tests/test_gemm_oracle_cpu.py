"""The float64 GEMM / convolution references of tests/gemm_oracle.py, their bounds and the exact-integer generator (no GPU needed);
the shape table of tests/test_gpu_gemm_shapes.py against what the models launch; the launch plans its batch-reduced cases reach."""
import itertools

import pytest
import torch
import torch.nn.functional as F

import gemm_oracle as go

D = torch.float64


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


# --------------------------------------------------------------------------- the references against torch.nn.functional
CONV_CASES = [(2, 9, 7, 4, 6, 3, 3, 1, 1, 1), (2, 9, 9, 6, 4, 3, 3, 2, 1, 2), (1, 11, 10, 3, 5, 5, 5, 2, 2, 1),
              (3, 8, 8, 8, 8, 1, 1, 2, 0, 4), (1, 13, 13, 4, 6, 11, 11, 4, 0, 1), (2, 6, 6, 6, 9, 3, 3, 1, 0, 3)]


@pytest.mark.parametrize("case", CONV_CASES, ids=lambda c: "n%d-%dx%dx%d-o%d-k%dx%d-s%dp%dg%d" % c)
def test_conv_references_match_torch(case):
    N, H, W, C, O, KH, KW, s, p, g = case
    gen = torch.Generator().manual_seed(sum(case))
    x = torch.randn(N, H, W, C, generator=gen, dtype=D)
    w = torch.randn(O, KH, KW, C // g, generator=gen, dtype=D)
    b = torch.randn(O, generator=gen, dtype=D)
    y, s_ = go.conv_fwd64(x, w, s, p, g, b)
    ref = _nhwc(F.conv2d(_nchw(x), w.permute(0, 3, 1, 2), b, stride=s, padding=p, groups=g))
    torch.testing.assert_close(y, ref, rtol=1e-12, atol=1e-12)
    ys, _ = go.conv_fwd64(x.abs(), w.abs(), s, p, g, b.abs())
    torch.testing.assert_close(s_, ys, rtol=1e-12, atol=1e-12)
    dy = torch.randn(y.shape, generator=gen, dtype=D)
    dx, _ = go.conv_dgrad64(dy, w, x.shape, s, p, g)
    dw, _ = go.conv_wgrad64(dy, x, w.shape, s, p, g)
    xr, wr = _nchw(x).clone().requires_grad_(True), w.permute(0, 3, 1, 2).clone().requires_grad_(True)
    F.conv2d(xr, wr, None, stride=s, padding=p, groups=g).backward(_nchw(dy))
    torch.testing.assert_close(dx, _nhwc(xr.grad), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dw, wr.grad.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)
    db, sb = go.bias_grad64(dy)
    torch.testing.assert_close(db, dy.sum((0, 1, 2)))
    torch.testing.assert_close(sb, dy.abs().sum((0, 1, 2)))


@pytest.mark.parametrize("case", [(2, 4, 4, 8, 6, 5, 2, 2, 1), (1, 7, 5, 4, 3, 3, 2, 1, 0), (2, 3, 3, 6, 4, 4, 2, 1, 0),
                                  (1, 5, 5, 3, 2, 3, 1, 1, 0)], ids=lambda c: "n%d-%dx%dx%d-to-%d-k%d-s%dp%dop%d" % c)
def test_conv_transpose_reference_matches_torch(case):
    N, Hi, Wi, Cin, Cout, K, s, p, op = case
    gen = torch.Generator().manual_seed(sum(case))
    x = torch.randn(N, Hi, Wi, Cin, generator=gen, dtype=D)
    w = torch.randn(Cin, K, K, Cout, generator=gen, dtype=D)           # [Cin, KH, KW, Cout]: torch's [in, out, kh, kw] permuted
    y, s_, parts = go.convT_fwd64(x, w, s, p, op)
    ref = _nhwc(F.conv_transpose2d(_nchw(x), w.permute(0, 3, 1, 2), stride=s, padding=p, output_padding=op))
    torch.testing.assert_close(y, ref, rtol=1e-12, atol=1e-12)
    assert (parts >= y.abs() - 1e-9).all() and (s_ >= parts - 1e-9).all()
    # backward: dx is the convolution of dy with the same weight, dW the wgrad with x as the output gradient
    dy = torch.randn(y.shape, generator=gen, dtype=D)
    xr, wr = _nchw(x).clone().requires_grad_(True), w.permute(0, 3, 1, 2).clone().requires_grad_(True)
    F.conv_transpose2d(xr, wr, stride=s, padding=p, output_padding=op).backward(_nchw(dy))
    dx, _ = go.conv_fwd64(dy, w, s, p)
    dw, _ = go.conv_wgrad64(x, dy, w.shape, s, p)
    torch.testing.assert_close(dx, _nhwc(xr.grad), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(dw, wr.grad.permute(0, 2, 3, 1), rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("a_mn,b_mn", list(itertools.product([False, True], repeat=2)))
def test_gemm_reference_all_majors_match_linear(a_mn, b_mn):
    M, N, K = 7, 5, 9
    gen = torch.Generator().manual_seed(3)
    A = torch.randn(M, K, generator=gen, dtype=D)
    B = torch.randn(N, K, generator=gen, dtype=D)
    bias = torch.randn(N, generator=gen, dtype=D)
    # storage with a row pitch wider than the rows, as the kernel's lda / ldb allow
    lda, ldb = (M + 3 if a_mn else K + 2), (N + 1 if b_mn else K + 5)
    sa = torch.zeros((K, lda) if a_mn else (M, lda), dtype=D)
    sb = torch.zeros((K, ldb) if b_mn else (N, ldb), dtype=D)
    (sa[:, :M].copy_(A.t()) if a_mn else sa[:, :K].copy_(A))
    (sb[:, :N].copy_(B.t()) if b_mn else sb[:, :K].copy_(B))
    want, s = go.gemm64(sa, sb, M, N, K, a_mn, b_mn, lda, ldb, bias=bias, act="relu")
    torch.testing.assert_close(want, F.relu(F.linear(A, B, bias)), rtol=1e-12, atol=1e-12)
    torch.testing.assert_close(s, F.linear(A.abs(), B.abs(), bias.abs()), rtol=1e-12, atol=1e-12)


# --------------------------------------------------------------------------- exact-integer operands
def test_integer_generator_is_exact_and_the_range_assertion_holds():
    gen = torch.Generator().manual_seed(0)
    x = go.int_operands((4, 9, 9, 64), gen, "cpu", scale_exp=-3)
    w = go.int_operands((32, 3, 3, 64), gen, "cpu", scale_exp=-2)
    assert torch.equal(x.to(torch.bfloat16).float(), x) and torch.equal(w.to(torch.bfloat16).float(), w)
    y, s = go.conv_fwd64(x, w, 1, 1)
    go.assert_exact_range(s, unit=2.0 ** -5)
    # every order of the fp32 sum is the exact value: a reversed, chunked fp32 accumulation agrees bit for bit
    xs = x.reshape(-1, 64)[:50]
    ws = w[:, 1, 1, :]
    exact = xs.double() @ ws.double().t()
    acc = torch.zeros(50, 32)
    for c in reversed(range(0, 64, 16)):
        acc = acc + (xs[:, c:c + 16] @ ws[:, c:c + 16].t())
    assert torch.equal(acc.double(), exact)
    with pytest.raises(AssertionError, match="too large"):
        go.assert_exact_range(torch.tensor([2.0 ** 24]))
    with pytest.raises(AssertionError, match="not integers"):
        go.assert_exact_range(torch.tensor([0.5]))


def test_bf16_ties_are_found():
    v = torch.tensor([257.0, 258.0, 100.0, 514.0, 1028.0, -259.0], dtype=D)
    assert go.tie_fraction(v) == pytest.approx(4 / 6)
    assert float(go.bf16_round(torch.tensor([257.0, 259.0], dtype=D))[0]) == 256.0


# --------------------------------------------------------------------------- the bounds reject a lost k-step and a one-ulp error
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "tf32"])
@pytest.mark.parametrize("K", [64 * 9, 1024, 4608])
def test_bound_rejects_a_missing_kstep(K, dtype):
    """A result that lost one k-step (MMA_K terms) at a model-sized K fails the per-element bound on random data."""
    M, N = 256, 64
    gen = torch.Generator().manual_seed(K)
    a = torch.randn(M, K, generator=gen).to(dtype)
    b = (torch.randn(N, K, generator=gen) * K ** -0.5).to(dtype)
    want, s = go.gemm64(a, b, M, N, K)
    out_dtype = dtype
    bnd = go.bound(want, s, K, dtype, out_dtype, splits=4, extra=2)
    good = want.to(out_dtype)
    go.check(good, want, bnd, "rounded exact result")
    mk = go.MMA_K[dtype]
    k0 = K // 2 // mk * mk
    lost = want - a[:, k0:k0 + mk].double() @ b[:, k0:k0 + mk].double().t()
    with pytest.raises(AssertionError, match="outside the bound"):
        go.check(lost.to(out_dtype), want, bnd, "lost k-step")


def test_exact_check_rejects_one_bf16_ulp():
    gen = torch.Generator().manual_seed(1)
    a = go.int_operands((128, 576), gen, "cpu").to(torch.bfloat16)
    b = go.int_operands((64, 576), gen, "cpu").to(torch.bfloat16)
    want, s = go.gemm64(a, b, 128, 64, 576)
    go.assert_exact_range(s)
    got = want.to(torch.float32).to(torch.bfloat16)
    go.assert_exact(got, want, "exact")
    bad = got.clone()
    i = int((want.abs() > 4).nonzero()[0, 0]), int((want.abs() > 4).nonzero()[0, 1])
    bad[i] = torch.nextafter(bad[i].float(), torch.tensor(float("inf"))).to(torch.bfloat16)
    if bad[i] == got[i]:                                     # nextafter in fp32 rounds back: step one bf16 ulp explicitly
        bad[i] = (got[i].float() * (1 + 2.0 ** -7)).to(torch.bfloat16)
    assert bad[i] != got[i]
    with pytest.raises(AssertionError, match=r"first at \(r=%d, c=%d\)" % i):
        go.assert_exact(bad, want, "one ulp")
    # and on the fp32 path (wgrad / tf32 outputs): one fp32 ulp
    got32 = want.float()
    bad32 = got32.clone()
    bad32[i] = torch.nextafter(bad32[i], torch.tensor(float("inf")))
    with pytest.raises(AssertionError, match="differ from the exact result"):
        go.assert_exact(bad32, want, "one fp32 ulp")


def test_explicit_path_partials_round_before_the_sum():
    """The strided dgrad reference with per-tap partials rounded to bf16 is what a bf16 dcol + col2im computes."""
    gen = torch.Generator().manual_seed(5)
    dy = go.int_operands((1, 4, 4, 64), gen, "cpu", -15, 15)
    w = go.int_operands((64, 3, 3, 8), gen, "cpu", -15, 15)
    exact, s, parts = go.conv_dgrad64(dy, w, (1, 8, 8, 8), 2, 1, abs_partials=True)
    rounded, _ = go.conv_dgrad64(dy, w, (1, 8, 8, 8), 2, 1, partial_dtype=torch.bfloat16)
    assert (parts > 256).any()                                  # some partials are not bf16 integers
    assert ((rounded - exact).abs() <= go.U_BF16 * parts).all()


# --------------------------------------------------------------------------- the shape table stays honest
def _record(builder):
    """Every conv / transposed-conv / linear call of one forward pass on the CPU, through the ops.reference functions that
    functional._impl dispatches to."""
    from theanompi_b200.ops import reference as ref
    calls = []
    names = ("conv2d_bias_act", "linear_bias_act", "conv_transpose2d_bias_act")
    orig = {n: getattr(ref, n) for n in names}

    def wrap(n):
        def f(*a, **k):
            calls.append((n,) + tuple(tuple(t.shape) if torch.is_tensor(t) else t for t in a))
            return orig[n](*a, **k)
        return f
    try:
        for n in names:
            setattr(ref, n, wrap(n))
        with torch.no_grad():
            builder()
    finally:
        for n in names:
            setattr(ref, n, orig[n])
    return calls


def _cfg(**kw):
    return dict(verbose=False, rank=0, size=1, device="cpu", batch_size=1, file_batch_size=1, **kw)


def _image_model(cls, **kw):
    from theanompi_b200.models import layers2
    layers2.reseed()
    m = cls(_cfg(**kw))
    return lambda: m.forward(m.x_in)


def _models():
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.googlenet import GoogLeNet
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    from theanompi_b200.models.lasagne_model_zoo.vgg16 import VGG16
    img = dict(data_kwargs=dict(n_train_files=1, n_val_files=1, synthetic=True))
    small = dict(data_kwargs=dict(n_synthetic=8, synthetic=True))
    return {"alexnet": (AlexNet, img), "cifar10": (Cifar10_model, small), "wrn": (Wide_ResNet, small), "googlenet": (GoogLeNet, img),
            "resnet50": (ResNet50, img), "resnet152": (ResNet152, img), "vgg16": (VGG16, img)}


def _in_table(model, call):
    table_model = "resnet50" if model == "resnet152" else model
    rows = [l for l in go.MODEL_LAYERS if l[0] == table_model]
    n = call[0]
    if n == "linear_bias_act":
        _, x, w, b, act = call
        return any(l[2] == "fc" and (l[3], l[4]) == (x[1], w[0]) and l[5] == ("relu" if act is True else "none") for l in rows)
    _, x, w, b, s, p, g, act = call
    _, H, W, C = x
    O, KH, KW, Cg = w
    act = {True: "relu", False: "none"}.get(act, act)
    for l in rows:
        if l[2] != "conv" or (l[3], l[4], l[7], l[8], l[9], l[10], l[12], l[13]) != (H, W, KH, KW, s, p, act, b is not None):
            continue
        if (l[5], l[6], l[11]) == (C, O, g) or (l[11] == 2 and g == 1 and (l[5], l[6]) == (2 * C, 2 * O)):   # AlexNet halves
            return True
    return False


@pytest.mark.parametrize("model", ["alexnet", "cifar10", "wrn", "googlenet", "resnet50", "resnet152", "vgg16"])
def test_model_shapes_are_in_the_table(model):
    """Each conv and linear call of the model at batch 1 and its production image size is in MODEL_LAYERS (at the model's
    default batch, which the table lists)."""
    cls, kw = _models()[model]
    calls = _record(_image_model(cls, **kw))
    assert calls, model
    missing = sorted(set(c for c in calls if not _in_table(model, c)))
    assert not missing, "%s launches shapes the GPU table lacks: %s" % (model, missing)


def test_gan_and_lstm_shapes_are_in_the_table():
    """NativeWGAN's generator and critic (the LSGAN shares them) and the LSTM at their defaults."""
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN
    from theanompi_b200.models.lstm import LSTM
    from theanompi_b200.ops import precision
    m = NativeWGAN(dict(verbose=False, rank=0, size=1, device="cpu", data_kwargs=dict(n_synthetic=64)))
    assert m.batch_size == 64
    calls = _record(lambda: m.critic(m.generator(torch.rand(1, m.nz))))
    cp = go.layer_channels("cp", precision.act_dtype())
    for c in calls:
        if c[0] == "conv_transpose2d_bias_act":
            _, x, w, b, s, p, op, act, c_real = c
            Cout = "cp" if w[3] == cp else w[3]
            assert any((l[2], l[3], l[4], l[5], l[6], l[7], l[8], l[9], l[10]) == (x[1], x[2], x[3], Cout, w[1], s, p, op, act)
                       for l in go.MODEL_CONVT), c
        elif c[0] == "conv2d_bias_act":
            _, x, w, b, s, p, g, act = c
            C = "cp" if x[3] == cp else x[3]
            assert any(l[0] == "gan" and (l[3], l[4], l[5], l[6], l[7], l[9], l[10], l[12]) ==
                       (x[1], x[2], C, w[0], w[1], s, p, {False: "none"}.get(act, act)) for l in go.MODEL_LAYERS), c
        else:
            _, x, w, b, act = c
            assert any(l[0] == "gan" and l[2] == "fc" and (l[3], l[4]) == (x[1], w[0]) for l in go.MODEL_LAYERS), c
    lstm = LSTM(dict(verbose=False, rank=0, size=1, device="cpu", data_kwargs=dict(n_synthetic=64)))
    assert (lstm.dim, lstm.batch_size) == (go.LSTM_H, go.LSTM_B)


# --------------------------------------------------------------------------- plans of the batch-reduced cases
def _lib():
    from theanompi_b200.ops import native
    L = native.lib()
    if L is None:
        pytest.skip("native extension not built")
    return L


@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "tf32"])
def test_batch_reduced_cases_keep_the_production_plans(f32):
    L = _lib()
    reduced = 0
    for l in go.MODEL_LAYERS:
        if l[2] != "conv":
            continue
        b = go.test_batch(L, l)
        assert go.conv_plans(L, l, b, f32) == go.conv_plans(L, l, l[1], f32), l
        reduced += b < l[1]
    assert reduced >= 10


@pytest.mark.parametrize("f32", [False, True], ids=["bf16", "tf32"])
def test_gpu_table_reaches_every_production_plan(f32):
    """Every (pass, path, BN, MT, split-K on / off) that the production shapes launch is launched by the GPU table's cases."""
    L = _lib()
    prod, test = set(), set()
    for l in go.MODEL_LAYERS:
        if l[2] != "conv":
            continue
        for dst, b in ((prod, l[1]), (test, go.test_batch(L, l))):
            for k, (path, bn, mt, sp) in go.conv_plans(L, l, b, f32).items():
                dst.add((k, path, bn, mt, sp > 1))
    assert prod <= test, sorted(prod - test)
    kinds = {(k, bn, mt) for k, path, bn, mt, _ in test if path == "implicit"}
    assert {("fprop", 96, 2), ("fprop", 192, 1), ("dgrad", 192, 1), ("wgrad", 192, 1)} <= kinds
