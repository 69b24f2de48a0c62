"""The wgmma GEMM and the implicit / explicit convolutions at every shape the models launch and at the edges of their launch
geometry, against the float64 references of tests/gemm_oracle.py (run with ``pytest -m gpu`` on an H100).

Every case runs twice: on exact-integer operands, where the result must be the exact one rounded once to the storage type, bit
for bit, whatever the accumulation order, split-K factor or atomics; and on random-normal operands, held per element to the bound
of the path (gemm_oracle.bound).  Convolutions and FC layers are reached through the ``ops`` autograd nodes, the LSTM GEMMs and the
geometry edges through ``cuda_impl.gemm``.  Both precision modes.

``TMPI_TEST_OUT`` names the directory that ``gemm_ratios.json`` (the largest |diff| / bound per family of the random-data cases)
is written to; by default it is pytest's temporary directory."""
import gc
import json
import os
import subprocess
import sys

import pytest
import torch

import gemm_oracle as go
import layer_oracle as lo
from theanompi_b200 import ops
from theanompi_b200.ops import accum, precision

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DT = {"bf16": torch.bfloat16, "tf32": torch.float32}
DATA = ["int", "randn"]
RATIOS = {}


def _ci():
    from theanompi_b200.ops import cuda_impl
    return cuda_impl


@pytest.fixture(params=["bf16", "tf32"])
def dtype(request):
    old = precision.precision()
    precision.set_precision(request.param)
    try:
        yield DT[request.param]
    finally:
        precision.set_precision(old)


@pytest.fixture(autouse=True)
def _release_memory():
    """Hand each case's operands and float64 references back to the device when it ends: the cases reach several GB (the
    ResNet50 layers at batch 32 in float64), and blocks left in the caching allocator would stay reserved for the rest of the
    process, where a later CUDA-graph capture needs fresh device memory for its private pool."""
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _ratios(tmp_path_factory):
    yield
    out = os.environ.get("TMPI_TEST_OUT") or str(tmp_path_factory.mktemp("gemm"))
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "gemm_ratios.json"), "w") as f:
        json.dump(dict(sorted(RATIOS.items())), f, indent=1)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _operand(shape, data, g, dtype, scale=1.0):
    """Storage-type operand: integers in [-2, 2] (``int``) or N(0, scale²) (``randn``), as an fp32 tensor when ``dtype`` is fp32."""
    if data == "int":
        return go.int_operands(shape, g, DEV, dtype=torch.float32).to(dtype)
    return (torch.randn(tuple(shape), device=DEV, generator=g) * scale).to(dtype)


def _master(shape, data, g, dtype, scale=1.0):
    """fp32 parameter whose values the active precision's operand holds exactly (bf16-representable in bf16 mode)."""
    return _operand(shape, data, g, dtype, scale).float()


def _chk(got, want, s, K, dtype, out_dtype, data, what, family, **kw):
    if data == "int":
        go.assert_exact_range(s)
        go.assert_exact(got, want, what)
    else:
        go.check(got, want, go.bound(want, s, K, dtype, out_dtype, **kw), what, RATIOS, _fam(family, dtype))


def _chk_db(got, dym, data, what, op_rel=0.0):
    want, s = go.bias_grad64(dym)
    if data == "int":
        go.assert_exact_range(s)
        go.assert_exact(got.float(), want, what)
    else:
        lo.assert_reduction(got, want, s, dym.numel() // dym.shape[-1], extra_abs=op_rel * s, what=what)


KM, RNA = go.U_TF32_KMAJOR, go.U_TF32_RNA


def _fam(family, dtype):
    return family + ("-bf16" if dtype == torch.bfloat16 else "-tf32")


# =========================================================================== convolutions
def _conv_case(H, W, C, O, KH, KW, s, p, groups, act, bias, batch, dtype, data, need_dx=True, seed=0, accumulate=False, tag=""):
    """Forward + backward of one convolution through ops.conv2d_bias_act / conv2d_group2_bias_act; checks y, dx, dW and db."""
    g = _gen(seed)
    Cg, Og = C // groups, O // groups
    K = KH * KW * Cg
    x = _operand((batch, H, W, C), data, g, dtype).requires_grad_(need_dx)
    ws = [_master((Og, KH, KW, Cg), data, g, dtype, K ** -0.5) for _ in range(groups)]
    bs = [(_master((Og,), data, g, torch.float32) if bias else None) for _ in range(groups)]
    sent = []
    for t in ws + [b for b in bs if b is not None]:
        t.requires_grad_(True)
        if accumulate:
            # the G arena: the gradient is a view into a NaN-filled buffer whose view holds G0
            buf = torch.full((t.numel() + 24,), float("nan"), device=DEV)
            view = buf[8:8 + t.numel()].view(t.shape)
            view.copy_(_operand(t.shape, "int", g, torch.float32))
            t.gbuf = view
            sent.append((t, buf, view.clone()))
    relu = {"relu": True, "none": False}.get(act, act)
    if groups == 2:
        y = ops.conv2d_group2_bias_act(x, ws[0], bs[0], ws[1], bs[1], s, p, relu)
    else:
        y = ops.conv2d_bias_act(x, ws[0], bs[0], s, p, 1, relu)
    dy = _operand(y.shape, data, g, dtype)
    with accum.mode(accumulate):
        y.backward(dy)
    torch.cuda.synchronize()
    w64 = torch.cat([t.detach() for t in ws], 0)
    b64 = torch.cat([t.detach() for t in bs], 0) if bias else None
    xd = x.detach()
    fam = "conv"
    # ---- forward
    plain = act in ("relu", "none")
    yw, ys = go.conv_fwd64(xd, w64, s, p, groups, b64, act if plain else None)
    if plain:
        _chk(y.detach(), yw, ys, K, dtype, dtype, data, tag + "y", fam + "-fprop", extra=1, tf32_units=(KM, KM))
    else:
        # an fp32 GEMM, then bias_act: the pre-activation's bound passes through the activation (slope <= 1), plus the
        # fast-math exp of the sigmoid and the rounding of the stored result
        yw = lo.act_fwd64(yw, act)
        bnd = go.bound(yw, ys, K, dtype, dtype, extra=1, tf32_units=(KM, KM)) + (8 * 2.0 ** -22) * (yw.abs() + 1.0)
        go.check(y.detach(), yw, bnd, tag + "y", RATIOS, _fam(fam + "-act-fprop", dtype))
    del yw, ys
    dym, data, op_rel = _dym(dy, y, act, dtype, data)
    # ---- weight gradient
    Ho, Wo = y.shape[1], y.shape[2]
    M = batch * Ho * Wo
    dww, dws = go.conv_wgrad64(dym, xd, (O, KH, KW, Cg), s, p, groups)
    for gi, t in enumerate(ws):
        sl = slice(gi * Og, (gi + 1) * Og)
        got = t.gbuf if accumulate else t.grad
        want = dww[sl]
        if accumulate:
            want = want + sent[gi][2].double()
        _chk(got, want, dws[sl] + (sent[gi][2].double().abs() if accumulate else 0), M, dtype, torch.float32, data,
             tag + "dW[%d]" % gi, fam + "-wgrad", splits=go.ceil_div(M, go.BK[dtype]), tf32_units=(RNA, RNA), operand_rel=op_rel)
    del dww, dws
    # ---- bias gradient
    if bias:
        for gi, t in enumerate(bs):
            got = t.gbuf if accumulate else t.grad
            d = dym[..., gi * Og:(gi + 1) * Og]
            if accumulate:
                want, sabs = go.bias_grad64(d)
                g0 = sent[len(ws) + gi][2].double()
                if data == "int":
                    go.assert_exact(got, want + g0, tag + "db[%d]" % gi)
                else:
                    lo.assert_reduction(got, want + g0, sabs + g0.abs(), M + 1, extra_abs=op_rel * sabs, what=tag + "db[%d]" % gi)
            else:
                _chk_db(got, d, data, tag + "db[%d]" % gi, op_rel)
    for t, buf, g0 in sent:
        outside = torch.cat([buf[:8], buf[8 + t.numel():]])
        assert torch.isnan(outside).all(), tag + "accumulate mode wrote outside the gradient view"
    # ---- input gradient
    if need_dx:
        explicit = s > 1 or not plain
        pdt = dtype if (explicit and not (KH == 1 and KW == 1 and s == 1 and p == 0)) else None
        if explicit and pdt is not None:
            dxw, dxs, dxp = go.conv_dgrad64(dym, w64, xd.shape, s, p, groups, abs_partials=True,
                                            partial_dtype=pdt if data == "int" else None)
            taps = KH * KW
            _chk(x.grad, dxw, dxs, O // groups * taps, dtype, dtype, data, tag + "dx", fam + "-dgrad-explicit", extra=taps,
                 tf32_units=(KM, RNA), partials=dxp, store_partials=pdt, operand_rel=op_rel)
            del dxp
        else:
            dxw, dxs = go.conv_dgrad64(dym, w64, xd.shape, s, p, groups)
            _chk(x.grad, dxw, dxs, KH * KW * Og, dtype, dtype, data, tag + "dx", fam + "-dgrad", tf32_units=(KM, RNA), operand_rel=op_rel)
        del dxw, dxs


def _dym(dy, y, act, dtype, data):
    """The masked output gradient as the kernel stores it, the data kind its checks can use and the relative error of its
    elements: exact for ReLU / identity; leaky ReLU / sigmoid store dy·act'(y) rounded to the activation dtype, so the
    products that follow get that rounding as an operand error and integer data is no longer exact."""
    if act in ("relu", "none", True, False):
        return lo.act_bwd64(dy.double(), y.detach().double(), act), data, 0.0
    d = lo.act_bwd64(dy.float(), y.detach().float(), act).to(dtype).double()
    return d, "randn", go.U_STORE_REL[dtype]


def _layer_id(i):
    l = go.MODEL_LAYERS[i]
    if l[2] == "conv":
        return "%s-%dx%dx%s-%s%dx%d-s%dp%dg%d-%s" % (l[0], l[3], l[4], l[5], l[6], l[7], l[8], l[9], l[10], l[11], l[12])
    return "%s-fc%dx%d-%s" % (l[0], l[3], l[4], l[5])


def _test_batch(l):
    from theanompi_b200.ops import native
    return go.test_batch(native.require(), l)


CONV_IDX = [i for i, l in enumerate(go.MODEL_LAYERS) if l[2] == "conv"]
FC_IDX = [i for i, l in enumerate(go.MODEL_LAYERS) if l[2] == "fc"]


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("i", CONV_IDX, ids=_layer_id)
def test_model_conv(i, data, dtype):
    l = go.MODEL_LAYERS[i]
    _, _, _, H, W, C, O, KH, KW, s, p, groups, act, bias = l
    C = go.layer_channels(C, dtype)
    need_dx = not go.first_layer(i) or l[0] == "gan"             # the critic's first conv gets the generator's gradient
    _conv_case(H, W, C, O, KH, KW, s, p, groups, act, bias, _test_batch(l), dtype, data, need_dx=need_dx, seed=i)


# --------------------------------------------------------------------------- geometry edges of the implicit convolution
# (id, N, H, W, C, O, K, stride, pad, groups, act): partial last channel chunks (bf16 chunk 64, tf32 chunk 32), grouped
# convolutions whose last chunk would run into the next group's channels, M mod 128 in {1, 64, 127}, N not a multiple of BN,
# a wgrad whose second m-tile has a warpgroup without rows (O = 192), the 1x1 "activation is the matrix" path.
CONV_EDGES_BF16 = [("cg%d" % c, 4, 9, 9, c, 64, 3, 1, 1, 1, "relu") for c in (8, 16, 24, 40, 48, 72)] + [
    ("cg24-groups2", 4, 9, 9, 48, 64, 3, 1, 1, 2, "relu"),
    ("cg40-groups2", 2, 7, 7, 80, 96, 3, 1, 1, 2, "none"),
]
CONV_EDGES_TF32 = [("cg%d" % c, 4, 9, 9, c, 64, 3, 1, 1, 1, "relu") for c in (4, 12, 36)] + [
    ("cg12-groups2", 4, 9, 9, 24, 64, 3, 1, 1, 2, "relu"),
]
CONV_EDGES = [
    ("m128k+1", 1, 9, 57, 32, 64, 3, 1, 1, 1, "relu"),         # 513 rows
    ("m128k+64", 1, 8, 72, 32, 64, 3, 1, 1, 1, "relu"),        # 576
    ("m128k+127", 1, 17, 15, 32, 64, 3, 1, 1, 1, "relu"),      # 255
    ("n-not-bn-multiple", 2, 10, 10, 64, 200, 3, 1, 1, 1, "relu"),
    ("wgrad-m192-idle-warpgroup", 4, 13, 13, 64, 192, 3, 1, 1, 1, "relu"),
    ("1x1-explicit-leaky", 4, 10, 10, 64, 64, 1, 1, 0, 1, "leaky"),
    ("strided-dgrad-3x3", 4, 15, 15, 32, 64, 3, 2, 1, 1, "none"),
    ("leaky-sigmoid", 2, 12, 12, 32, 32, 3, 1, 1, 1, "sigmoid"),
]


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("case", CONV_EDGES + [("bf16-" + c[0],) + c[1:] for c in CONV_EDGES_BF16]
                         + [("tf32-" + c[0],) + c[1:] for c in CONV_EDGES_TF32], ids=lambda c: c[0])
def test_conv_edges(case, data, dtype):
    name, N, H, W, C, O, K, s, p, groups, act = case
    if name.startswith("bf16-") and dtype != torch.bfloat16 or name.startswith("tf32-") and dtype != torch.float32:
        pytest.skip("channel chunk edge of the other precision")
    _conv_case(H, W, C, O, K, K, s, p, groups, act, True, N, dtype, data, need_dx=True, seed=len(name))


# --------------------------------------------------------------------------- accumulate mode (gradient accumulation into G)
ACCUM_CASES = [i for i in CONV_IDX if go.MODEL_LAYERS[i][0] in ("alexnet", "cifar10")] + [74]


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("i", ACCUM_CASES, ids=_layer_id)
def test_accumulate_mode_conv(i, data, dtype):
    """Every wgrad and db of the layer adds into a view of a NaN-filled buffer holding G0: G = G0 + dW, nothing written outside."""
    l = go.MODEL_LAYERS[i]
    _, _, _, H, W, C, O, KH, KW, s, p, groups, act, _ = l
    _conv_case(H, W, go.layer_channels(C, dtype), O, KH, KW, s, p, groups, act, True, _test_batch(l), dtype, data,
               need_dx=False, seed=100 + i, accumulate=True, tag="accumulate: ")


# =========================================================================== FC layers
def _fc_case(I, O, act, batch, dtype, data, seed=0, accumulate=False):
    g = _gen(seed)
    x = _operand((batch, I), data, g, dtype).requires_grad_(True)
    w = _master((O, I), data, g, dtype, I ** -0.5).requires_grad_(True)
    b = _master((O,), data, g, torch.float32).requires_grad_(True)
    sent = []
    if accumulate:
        for t in (w, b):
            buf = torch.full((t.numel() + 24,), float("nan"), device=DEV)
            view = buf[8:8 + t.numel()].view(t.shape)
            view.copy_(_operand(t.shape, "int", g, torch.float32))
            t.gbuf = view
            sent.append((t, buf, view.clone()))
    y = ops.linear_bias_act(x, w, b, {"relu": True, "none": False}[act])
    dy = _operand(y.shape, data, g, dtype)
    with accum.mode(accumulate):
        y.backward(dy)
    torch.cuda.synchronize()
    yw, ys = go.gemm64(x.detach(), w.detach(), batch, O, I, bias=b.detach(), act=act)
    _chk(y.detach(), yw, ys, I, dtype, dtype, data, "y", "fc-fprop", extra=2, tf32_units=(KM, KM))
    dym, _, _ = _dym(dy, y, act, dtype, data)
    dxw, dxs = go.gemm64(dym, w.detach(), batch, I, O, b_mn=True)
    _chk(x.grad, dxw, dxs, O, dtype, dtype, data, "dx", "fc-dgrad", tf32_units=(KM, RNA))
    dww, dws = go.gemm64(dym, x.detach(), O, I, batch, a_mn=True, b_mn=True)
    gw = w.gbuf if accumulate else w.grad
    if accumulate:
        dww, dws = dww + sent[0][2].double(), dws + sent[0][2].double().abs()
    _chk(gw, dww, dws, batch, dtype, torch.float32, data, "dW", "fc-wgrad", splits=batch, extra=1, tf32_units=(RNA, RNA))
    gb = b.gbuf if accumulate else b.grad
    if accumulate:
        want, sabs = go.bias_grad64(dym)
        if data == "int":
            go.assert_exact(gb, want + sent[1][2].double(), "db")
        else:
            lo.assert_reduction(gb, want + sent[1][2].double(), sabs + sent[1][2].double().abs(), batch + 1, what="db")
        for t, buf, _ in sent:
            assert torch.isnan(torch.cat([buf[:8], buf[8 + t.numel():]])).all(), "accumulate mode wrote outside the gradient view"
    else:
        _chk_db(gb, dym, data, "db")


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("i", FC_IDX, ids=_layer_id)
def test_model_fc(i, data, dtype):
    l = go.MODEL_LAYERS[i]
    _fc_case(l[3], l[4], l[5], l[1], dtype, data, seed=i)


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("shape", [(128, 9216, 4096), (256, 256, 10), (64, 100, 1024), (64, 1024, 1), (32, 2048, 1000)],
                         ids=lambda s: "b%d-%dx%d" % s)
def test_accumulate_mode_fc(shape, data, dtype):
    B_, I, O = shape
    _fc_case(I, O, "none", B_, dtype, data, seed=sum(shape), accumulate=True)


# =========================================================================== transposed convolutions (GAN generator)
@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("case", go.MODEL_CONVT, ids=lambda c: "%s-%dx%dx%d-to-%s-%s" % (c[0], c[2], c[3], c[4], c[5], c[10]))
def test_model_conv_transpose(case, data, dtype):
    _, B_, Hi, Wi, Cin, Cout, K, s, p, op, act, c_real = case
    Cout = go.layer_channels(Cout, dtype)
    g = _gen(Hi * Cin)
    x = _operand((B_, Hi, Wi, Cin), data, g, dtype).requires_grad_(True)
    w = _master((Cin, K, K, Cout), data, g, dtype, (Cin * K * K) ** -0.5)
    if c_real is not None:
        w[..., c_real:] = 0
    w.requires_grad_(True)
    b = _master((Cout,), data, g, torch.float32)
    if c_real is not None:
        b[c_real:] = 0
    b.requires_grad_(True)
    from theanompi_b200.ops.functional import conv_transpose2d_bias_act
    y = conv_transpose2d_bias_act(x, w, b, s, p, op, act, c_real)
    dy = _operand(y.shape, data, g, dtype)
    y.backward(dy)
    torch.cuda.synchronize()
    exact_ok = data == "int" and act == "none"
    zw, zs, zp = go.convT_fwd64(x.detach(), w.detach(), s, p, op, partial_dtype=dtype if exact_ok else None)
    zw, zs = zw + b.detach().double(), zs + b.detach().double().abs()
    if c_real is not None:
        zw[..., c_real:] = float("-inf") if act == "sigmoid" else 0.0     # padded channels are stored as zeros
    taps = K * K
    if exact_ok:
        go.assert_exact_range(zs)
        go.assert_exact(y.detach(), zw, "y")
    else:
        yw = lo.act_fwd64(zw, act)
        bnd = go.bound(yw, zs, Cin * taps, dtype, dtype, extra=taps + 1, tf32_units=(KM, RNA), partials=zp, store_partials=dtype)
        if act == "sigmoid":
            bnd = bnd + (8 * 2.0 ** -22) * (yw.abs() + 1.0)      # the fast-math exp of the epilogue (slope of the sigmoid <= 1)
        go.check(y.detach(), yw, bnd, "y", RATIOS, _fam("convT-fprop", dtype))
    del zw, zs, zp
    dym, bdata, op_rel = _dym(dy, y, act, dtype, data)
    dxw, dxs = go.conv_fwd64(dym, w.detach(), s, p)
    _chk(x.grad, dxw, dxs, K * K * Cout, dtype, dtype, bdata, "dx", "convT-dgrad", tf32_units=(KM, KM), operand_rel=op_rel)
    dww, dws = go.conv_wgrad64(x.detach(), dym, (Cin, K, K, Cout), s, p)
    M = B_ * Hi * Wi
    _chk(w.grad, dww, dws, M, dtype, torch.float32, bdata, "dW", "convT-wgrad", splits=go.ceil_div(M, go.BK[dtype]),
         tf32_units=(RNA, RNA), operand_rel=op_rel)
    _chk_db(b.grad, dym, bdata, "db", op_rel)


# =========================================================================== plain GEMM: LSTM, majors, geometry edges
def _gemm_case(M, N, K, a_mn, b_mn, dtype, data, out_bf16=True, ldc=None, splitk=0, bias=False, relu=False, accumulate=False,
               seed=0, family="gemm", check_plan=None):
    g = _gen(seed)
    # MN-major operands are stored with a 16-byte row pitch, as every caller does (TMA needs it)
    lda = go.ceil_div(M, 8) * 8 if a_mn else K
    ldb = go.ceil_div(N, 8) * 8 if b_mn else K
    a = _operand((K, lda) if a_mn else (M, K), data, g, dtype)
    b = _operand((K, ldb) if b_mn else (N, K), data, g, dtype, K ** -0.5)
    bias_t = _master((N,), data, g, torch.float32) if bias else None
    fp32_out = dtype == torch.float32 or not out_bf16
    odt = torch.float32 if fp32_out else torch.bfloat16
    ld = ldc or N
    buf = torch.full((M * ld + 16,), float("nan"), device=DEV, dtype=odt)
    out = torch.as_strided(buf, (M, N), (ld, 1), 16 // buf.element_size())
    g0 = None
    if accumulate:
        g0 = _operand((M, N), "int", g, torch.float32)
        out.copy_(g0)
    before = buf.clone()
    _ci().gemm(a, b, M, N, K, a_mn=a_mn, b_mn=b_mn, out=out, out_dtype=odt, bias=bias_t, bias_mode=1 if bias else 0, relu=relu,
               lda=lda, ldb=ldb, ldc=ld, splitk=splitk, accumulate=accumulate)
    torch.cuda.synchronize()
    want, s = go.gemm64(a, b, M, N, K, a_mn, b_mn, lda, ldb, bias=bias_t, act="relu" if relu else None)
    if accumulate:
        want, s = want + g0.double(), s + g0.double().abs()
    units = (RNA if a_mn else KM, RNA if b_mn else KM)
    _chk(out, want, s, K, dtype, odt, data, "C", family, splits=go.ceil_div(K, go.BK[dtype]), extra=2, tf32_units=units)
    inside = torch.zeros(buf.numel(), dtype=torch.bool, device=DEV)
    torch.as_strided(inside, (M, N), (ld, 1), 16 // buf.element_size()).fill_(True)
    assert torch.equal(torch.isnan(buf[~inside]), torch.isnan(before[~inside])), "the GEMM wrote outside its [M, N] view of ldc %d" % ld


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("T", go.LSTM_T)
def test_lstm_gemms(T, data, dtype):
    """The LSTM's GEMMs: input gates over T·B rows, the recurrent step h·Uᵀ, its input gradient dG·U and the sequence's
    recurrent weight gradient dUᵀ = Σ_t dG_tᵀ·h_t (both operands MN-major, split-K over T·B)."""
    H, B_ = go.LSTM_H, go.LSTM_B
    _gemm_case(T * B_, 4 * H, H, False, False, dtype, data, seed=T, family="lstm")                   # x·Wᵀ (+ b)
    _gemm_case(B_, 4 * H, H, False, False, dtype, data, seed=T + 1, family="lstm")                   # h·Uᵀ
    _gemm_case(B_, H, 4 * H, False, True, dtype, data, seed=T + 2, family="lstm")                    # dG·U
    _gemm_case(4 * H, H, T * B_, True, True, dtype, data, out_bf16=False, seed=T + 3, family="lstm")  # dGᵀ·h


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("a_mn,b_mn", [(0, 0), (0, 1), (1, 0), (1, 1)], ids=["KK", "KN", "NK", "NN"])
@pytest.mark.parametrize("MNK", [(1, 64, 64), (129, 72, 200), (192, 200, 520), (383, 64, 64), (1000, 1000, 1000)],
                         ids=lambda t: "%dx%dx%d" % t)
def test_gemm_majors(MNK, a_mn, b_mn, data, dtype):
    M, N, K = MNK
    _gemm_case(M, N, K, bool(a_mn), bool(b_mn), dtype, data, out_bf16=False, seed=M + N + K + 2 * a_mn + b_mn, family="gemm-majors")
    if not a_mn:
        _gemm_case(M, N, K, False, bool(b_mn), dtype, data, out_bf16=True, bias=True, relu=True, seed=M + 1, family="gemm-majors")


GEMM_EDGES = [
    # (id, M, N, K, a_mn, b_mn, out_bf16, ldc, splitk, accumulate)
    ("m-mod128-1", 513, 128, 256, 0, 0, 1, None, 0, 0),
    ("m-mod128-64", 576, 128, 256, 0, 0, 1, None, 0, 0),
    ("m-mod128-127", 639, 128, 256, 0, 0, 1, None, 0, 0),
    ("tall-second-half-partial", 256 * 260 + 200, 128, 128, 0, 0, 1, None, 0, 0),
    ("tall-second-half-empty", 256 * 260 + 100, 128, 128, 0, 0, 1, None, 0, 0),
    ("n-not-bn-multiple", 1024, 200, 128, 0, 0, 1, None, 0, 0),
    ("splitk-forced-off", 128, 256, 8192, 1, 1, 0, None, 1, 0),
    ("splitk-forced-4", 128, 256, 8192, 1, 1, 0, None, 4, 0),
    ("splitk-forced-7", 200, 136, 4000, 0, 1, 0, None, 7, 0),
    ("ldc-gt-n-aligned", 300, 96, 192, 0, 0, 1, 136, 0, 0),
    ("ldc-unaligned-bf16", 300, 96, 192, 0, 0, 1, 101, 0, 0),
    ("ldc-unaligned-fp32", 300, 96, 192, 1, 1, 0, 99, 0, 0),
    ("ldc-unaligned-splitk", 260, 72, 4096, 1, 1, 0, 75, 3, 0),
    ("accumulate-splitk", 192, 576, 8192, 1, 1, 0, None, 0, 1),
    ("accumulate-ldc-unaligned", 130, 40, 3000, 1, 1, 0, 43, 0, 1),
]


@pytest.mark.parametrize("data", DATA)
@pytest.mark.parametrize("case", GEMM_EDGES, ids=lambda c: c[0])
def test_gemm_edges(case, data, dtype):
    name, M, N, K, a_mn, b_mn, out_bf16, ldc, splitk, acc = case
    if name.startswith("tall"):
        from theanompi_b200.ops import native
        bn, mt, _ = go.gemm_plan(native.require(), M, N, K, dtype == torch.float32, out_bf16=bool(out_bf16))
        assert mt == 2, "the case no longer reaches a 256-row tile"
    _gemm_case(M, N, K, bool(a_mn), bool(b_mn), dtype, data, out_bf16=bool(out_bf16), ldc=ldc, splitk=splitk, accumulate=bool(acc),
               seed=M + N, family="gemm-edges")


def test_bf16_output_rounds_ties_to_even():
    """Integer sums on bf16 ties above 256 (odd integers in (256, 512), where the bf16 step is 2) are rounded to even, bit for bit."""
    old = precision.precision()
    precision.set_precision("bf16")
    try:
        M, N, K = 128, 64, 64
        a = torch.zeros((M, K), device=DEV)
        b = torch.zeros((N, K), device=DEV)
        a[:, 0] = 256.0
        a[:, 1] = 1 + 2 * torch.arange(M, device=DEV).float()      # row m sums to 257 + 2m ...
        a[:, 2] = -1.0
        b[:, 0] = b[:, 1] = 1.0
        b[:, 2] = torch.arange(N, device=DEV).float() % 3           # ... minus 0, 1 or 2 by column: ties and exact values
        a, b = a.to(torch.bfloat16), b.to(torch.bfloat16)
        out = _ci().gemm(a, b, M, N, K, lda=K, ldb=K)
        torch.cuda.synchronize()
        want, s = go.gemm64(a, b, M, N, K)
        go.assert_exact_range(s)
        assert go.tie_fraction(want) > 0.3
        go.assert_exact(out, want, "bf16 ties")
    finally:
        precision.set_precision(old)


def test_tf32_kmajor_read_rounds():
    """What the TFLOAT32 TMA read of a K-major fp32 operand does to the low 13 bits: a = 1 + 0.75·2⁻¹⁰ times b = 1 gives
    1 + 2⁻¹⁰ when rounded to nearest and 1 when truncated.  The K-major bound (gemm_oracle.U_TF32_KMAJOR = 2⁻¹¹) rests on it rounding."""
    old = precision.precision()
    precision.set_precision("tf32")
    try:
        M, N, K = 128, 64, 32
        a = torch.zeros((M, K), device=DEV)
        b = torch.zeros((N, K), device=DEV)
        a[:, 0] = 1.0 + 0.75 * 2.0 ** -10
        b[:, 0] = 1.0
        out = _ci().gemm(a, b, M, N, K, lda=K, ldb=K)
        torch.cuda.synchronize()
        v = float(out[0, 0])
        assert v == 1.0 + 2.0 ** -10, "the TFLOAT32 TMA read truncated (got %r): gemm_oracle.U_TF32_KMAJOR must be 2^-10" % v
        assert (out == v).all()
    finally:
        precision.set_precision(old)


# =========================================================================== determinism
_DET_SCRIPT = r"""
import sys, torch
sys.path.insert(0, %(root)r); sys.path.insert(0, %(tests)r)
from theanompi_b200 import ops
from theanompi_b200.ops import precision
res = []
for prec in ("bf16", "tf32"):
    precision.set_precision(prec)
    dt = torch.bfloat16 if prec == "bf16" else torch.float32
    outs = []
    for run in range(2):
        g = torch.Generator(device="cuda").manual_seed(7)
        x = torch.randn((128, 27, 27, 96), device="cuda", generator=g).to(dt).requires_grad_(True)
        w0 = torch.randn((128, 5, 5, 48), device="cuda", generator=g).to(dt).float().requires_grad_(True)
        w1 = torch.randn((128, 5, 5, 48), device="cuda", generator=g).to(dt).float().requires_grad_(True)
        b0 = torch.randn(128, device="cuda", generator=g).requires_grad_(True)
        b1 = torch.randn(128, device="cuda", generator=g).requires_grad_(True)
        y = ops.conv2d_group2_bias_act(x, w0, b0, w1, b1, 1, 2, True)
        y.backward(torch.randn(y.shape, device="cuda", generator=g).to(dt))
        xf = torch.randn((128, 9216), device="cuda", generator=g).to(dt).requires_grad_(True)
        wf = torch.randn((4096, 9216), device="cuda", generator=g).to(dt).float().requires_grad_(True)
        bf = torch.randn(4096, device="cuda", generator=g).requires_grad_(True)
        yf = ops.linear_bias_act(xf, wf, bf, True)
        yf.backward(torch.randn(yf.shape, device="cuda", generator=g).to(dt))
        outs.append([t.detach().clone() for t in (y, x.grad, w0.grad, w1.grad, b0.grad, b1.grad, yf, xf.grad, wf.grad, bf.grad)])
    res.append(all(torch.equal(a, b) for a, b in zip(*outs)))
print("BITWISE", res)
"""


def test_deterministic_mode_is_bitwise_reproducible():
    """Under TMPI_DETERMINISTIC=1 (read once per process: a subprocess) two runs of a split-K conv wgrad and the FC layer on random
    data give the same bits in both precisions."""
    env = dict(os.environ, TMPI_DETERMINISTIC="1")
    r = subprocess.run([sys.executable, "-c", _DET_SCRIPT % dict(root=ROOT, tests=HERE)], env=env, stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert "BITWISE [True, True]" in r.stdout, r.stdout[-3000:]
