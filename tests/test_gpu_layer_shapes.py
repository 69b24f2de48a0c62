"""The streaming layer kernels (batch norm, pooling, LRN, softmax cross-entropy, dropout, the small elementwise passes) at the
shapes the models launch and at the edges of their launch geometry, against the float64 references of tests/layer_oracle.py with
per-element and per-sum bounds (run with ``pytest -m gpu`` on an H100).

Every kernel is reached through ``ops.*`` where an autograd node exists, in both precision modes.  fp32 storage gets twice the
elementwise unit where a result passes through ``rsqrtf`` (batch norm) and eight times where it passes through the fast exp / log
intrinsics (LRN, softmax, sigmoid): they are 2-ulp approximations under ``--use_fast_math``.

``TMPI_TEST_OUT`` names the directory the batch-norm conditioning sweep writes ``bn_conditioning.json`` to (default: pytest's
temporary directory)."""
import json
import os
import subprocess
import sys

import pytest
import torch

import layer_oracle as lo
from theanompi_b200 import ops
from theanompi_b200.ops import accum, precision
from theanompi_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DT = {"bf16": torch.bfloat16, "tf32": torch.float32}
EPS = 1e-5


def _ci():
    from theanompi_b200.ops import cuda_impl
    return cuda_impl


def _sync():
    if DEV != "cpu":
        torch.cuda.synchronize()


@pytest.fixture(params=["bf16", "tf32"])
def dtype(request):
    old = precision.precision()
    precision.set_precision(request.param)
    try:
        yield DT[request.param]
    finally:
        precision.set_precision(old)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, g, dtype=torch.float32, scale=1.0, shift=0.0):
    return (torch.randn(shape, device=DEV, generator=g) * scale + shift).to(dtype)


def _fast(dtype, k):
    """Multiple of the elementwise unit for results that pass through a fast-math intrinsic (fp32 storage only: the bf16 rounding
    dwarfs it)."""
    return float(k) if dtype == torch.float32 else 1.0


# =========================================================================== batch norm
def _bn_run(shape, dtype, act, with_res, with_drop, seed=0, mu=0.5, sigma=2.0, momentum=0.1, gamma=None, beta=None):
    """Forward (training), backward and an eval forward through ``ops.batch_norm``; returns everything the checks need."""
    g = _gen(seed)
    C, N = shape[-1], shape[0]
    x = _randn(shape, g, dtype, sigma, mu).requires_grad_(True)
    res = _randn(shape, g, dtype).requires_grad_(True) if with_res else None
    gamma = ((torch.rand(C, device=DEV, generator=g) + 0.5) if gamma is None else gamma.clone()).requires_grad_(True)
    beta = (torch.randn(C, device=DEV, generator=g) if beta is None else beta.clone()).requires_grad_(True)
    rm0 = torch.randn(C, device=DEV, generator=g) * 0.1
    rv0 = torch.rand(C, device=DEV, generator=g) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    drop = torch.where(torch.rand(N, device=DEV, generator=g) < 0.25, 0.0, 1.0 / 0.75).float() if with_drop else None
    relu = {None: False, "relu": True}.get(act, act)
    y = ops.batch_norm(x, gamma, beta, rm, rv, True, momentum, EPS, relu, res, drop)
    saved = y.grad_fn.saved_tensors                    # (x, y or empty, mean, rstd): the statistics the backward will use
    mean, rstd = saved[2].clone(), saved[3].clone()
    dy = _randn(shape, g, dtype)
    y.backward(dy)
    ye = ops.batch_norm(x.detach(), gamma.detach(), beta.detach(), rm, rv, False, momentum, EPS, relu,
                        res.detach() if with_res else None, drop)
    _sync()
    return dict(x=x.detach(), res=res.detach() if with_res else None, gamma=gamma.detach(), beta=beta.detach(), rm0=rm0, rv0=rv0, rm=rm,
                rv=rv, drop=drop, y=y.detach(), mean=mean, rstd=rstd, dy=dy, dx=x.grad, dres=res.grad if with_res else None,
                dgamma=gamma.grad, dbeta=beta.grad, ye=ye, act=act, momentum=momentum)


def _bn_check(r, dtype, tag=""):
    x, C = r["x"], r["x"].shape[-1]
    R = x.numel() // C
    act, mom = r["act"], r["momentum"]
    sl = _fast(dtype, 8 if act == "sigmoid" else 2)
    f = lo.bn_fwd64(x, r["gamma"], r["beta"], EPS, act, r["res"], r["drop"], run_mean=r["rm0"], run_var=r["rv0"], momentum=mom)
    unb = R / (R - 1) if R > 1 else 1.0
    var_terms = f["sum_x2"] + 2 * f["mean"].abs() * f["abs_x"]
    lo.assert_reduction(r["mean"].double() * R, f["sum_x"], f["abs_x"], R, what=tag + "Σx (from mean)")
    var_k = r["rstd"].double() ** -2 - EPS
    lo.assert_reduction(var_k * R, f["var"] * R, var_terms, R, extra_abs=R * (2.0 ** -20 * (f["var"] + EPS) + f["mean_abs"] ** 2),
                        what=tag + "Σ(x − mean)² (from rstd)")
    lo.assert_reduction(r["rm"], f["run_mean"], mom * f["abs_x"] / R, R, extra_abs=2.0 ** -22 * (r["rm0"].double().abs() + f["mean"].abs()),
                        what=tag + "running mean")
    lo.assert_reduction(r["rv"], f["run_var"], mom * unb * var_terms / R, R,
                        extra_abs=2.0 ** -20 * (r["rv0"].double() + unb * (f["var"] + EPS)) + mom * unb * f["mean_abs"] ** 2,
                        what=tag + "running variance")
    lo.assert_elementwise(r["y"], f["y"], dtype, s=f["s"], extra_abs=f["coef_abs"], slack=sl, what=tag + "y (training)")
    # backward: the oracle takes the mask from the kernel's own y and the statistics the forward saved
    b = lo.bn_bwd64(x, r["dy"], r["y"], r["gamma"], r["mean"], r["rstd"], act, r["drop"])
    lo.assert_reduction(r["dgamma"], b["dgamma"], b["abs_dgamma"], R, what=tag + "dγ")
    lo.assert_reduction(r["dbeta"], b["dbeta"], b["abs_dbeta"], R, what=tag + "dβ")
    lo.assert_elementwise(r["dx"], b["dx"], dtype, s=b["s_dx"], extra_abs=lo.red_rel(R) * b["s_dx"], slack=sl, what=tag + "dx")
    if r["dres"] is not None:
        assert torch.equal(r["dres"].double(), b["dres"]), tag + "dres is the masked dy, exactly"
    # eval: the running statistics the training call left
    e = lo.bn_fwd64(x, r["gamma"], r["beta"], EPS, act, r["res"], r["drop"], training=False, run_mean=r["rm"], run_var=r["rv"])
    lo.assert_elementwise(r["ye"], e["y"], dtype, s=e["s"], slack=sl, what=tag + "y (eval)")


BN_VARIANTS = [(None, False, False), ("relu", False, False), ("relu", True, False), ("relu", True, True)]
BN_VARIANT_IDS = ["plain", "relu", "res-relu", "res-relu-drop"]
# (N, H, W, C) of the batch norms of ResNet50 at batch 64 and of WRN-28-4 / WRN-28-10 at batch 128
BN_MODEL_SHAPES = [(64, 112, 112, 64), (64, 56, 56, 64), (64, 56, 56, 256), (64, 28, 28, 128), (64, 28, 28, 512), (64, 14, 14, 1024),
                   (64, 7, 7, 512), (64, 7, 7, 2048), (128, 32, 32, 16), (128, 32, 32, 64), (128, 32, 32, 160), (128, 16, 16, 320),
                   (128, 8, 8, 640)]


@pytest.mark.parametrize("variant", BN_VARIANTS, ids=BN_VARIANT_IDS)
@pytest.mark.parametrize("shape", BN_MODEL_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_bn_model_shapes(shape, variant, dtype):
    _bn_check(_bn_run(shape, dtype, *variant, seed=sum(shape)), dtype)


def _bn_geometry(C, dtype):
    """(VT, RL): channel vectors and row lanes of one 256-thread CTA of the batch-norm passes (csrc/bn_kernels.cu)."""
    nvec = C // lo.VEC[dtype]
    VT = min(nvec, 32)
    return VT, 256 // VT


@pytest.mark.parametrize("variant", [BN_VARIANTS[0], BN_VARIANTS[3]], ids=["plain", "res-relu-drop"])
@pytest.mark.parametrize("rows", ["1", "2", "7", "RL", "UR*RL-1", "UR*RL+1"])
@pytest.mark.parametrize("C", [8, 72, 264, 2048])
def test_bn_edge_rows(C, rows, variant, dtype):
    """Fewer rows than one trip of a CTA (UR = 4 rows in flight per lane in the statistics pass), a single row, and channel counts
    whose vectors do not fill the CTA (72: 9 or 18 vectors, idle threads) or the last channel group (264)."""
    _, RL = _bn_geometry(C, dtype)
    R = {"1": 1, "2": 2, "7": 7, "RL": RL, "UR*RL-1": 4 * RL - 1, "UR*RL+1": 4 * RL + 1}[rows]
    _bn_check(_bn_run((R, 1, 1, C), dtype, *variant, seed=C + R), dtype)


@pytest.mark.parametrize("shape", [(6, 5, 7, 264), (3, 37, 41, 72), (5, 3, 3, 520)], ids=lambda s: "x".join(map(str, s)))
def test_bn_ragged_slabs(shape, dtype):
    """R not a multiple of the rows per CTA (short last slab) with several rows per sample under a drop row."""
    _bn_check(_bn_run(shape, dtype, "relu", True, True, seed=7), dtype)


@pytest.mark.parametrize("act,shape", [("leaky", (64, 16, 16, 128)), ("leaky", (64, 4, 4, 512)), ("sigmoid", (64, 8, 8, 256))],
                         ids=["leaky-16x16x128", "leaky-4x4x512", "sigmoid-8x8x256"])
def test_bn_gan_activations(act, shape, dtype):
    _bn_check(_bn_run(shape, dtype, act, False, False, seed=11), dtype)


def _bn_accumulate(dtype):
    """Backward at a ragged shape with the parameter gradients stored into, then added into, arena-style views holding a previous
    gradient.  Returns the inputs and, per mode, (dx, dγ view, dβ view, y, mean, rstd)."""
    shape, C = (6, 5, 7, 264), 264
    g = _gen(3)
    x = _randn(shape, g, dtype, 2.0, 0.5)
    dy = _randn(shape, g, dtype)
    prev_g, prev_b = torch.randn(C, device=DEV, generator=g), torch.randn(C, device=DEV, generator=g)
    out = {}
    for mode in ("store", "accumulate"):
        xx = x.clone().requires_grad_(True)
        gamma = torch.full((C,), 1.5, device=DEV).requires_grad_(True)
        beta = torch.zeros(C, device=DEV).requires_grad_(True)
        gamma.gbuf, beta.gbuf = prev_g.clone(), prev_b.clone()
        with accum.mode(mode == "accumulate"):
            y = ops.batch_norm(xx, gamma, beta, None, None, True, 0.1, EPS, True)
            mean, rstd = y.grad_fn.saved_tensors[2].clone(), y.grad_fn.saved_tensors[3].clone()
            y.backward(dy)
        out[mode] = (xx.grad, gamma.gbuf, beta.gbuf, y.detach(), mean, rstd)
    _sync()
    return x, dy, prev_g, prev_b, out


def test_bn_accumulate_mode(dtype):
    """Gradient accumulation: dγ / dβ are previous + this batch, dx is that of store mode (bit-equal in deterministic mode, see
    check_bn_deterministic; here the atomics of the two launches may order the sums differently)."""
    x, dy, prev_g, prev_b, out = _bn_accumulate(dtype)
    C, R = x.shape[-1], x.numel() // x.shape[-1]
    b = lo.bn_bwd64(x, dy, out["store"][3], torch.full((C,), 1.5, device=DEV), out["store"][4], out["store"][5], "relu")
    for mode in ("store", "accumulate"):
        lo.assert_elementwise(out[mode][0], b["dx"], dtype, s=b["s_dx"], extra_abs=lo.red_rel(R) * b["s_dx"], slack=_fast(dtype, 2),
                              what="dx (%s)" % mode)
    for i, (k, prev) in enumerate((("dgamma", prev_g), ("dbeta", prev_b))):
        lo.assert_reduction(out["store"][1 + i], b[k], b["abs_" + k], R, what=k + " (store)")
        lo.assert_reduction(out["accumulate"][1 + i], prev.double() + b[k], b["abs_" + k], R,
                            extra_abs=2.0 ** -23 * (prev.double().abs() + b[k].abs()), what=k + " (accumulate)")


def check_bn_deterministic():
    """Run with TMPI_DETERMINISTIC=1 (the flag is read once per process): two calls agree bit for bit and stay inside the bounds."""
    for name in ("bf16", "tf32"):
        precision.set_precision(name)
        for shape in ((64, 14, 14, 264), (33, 7, 7, 2048)):
            a = _bn_run(shape, DT[name], "relu", True, True, seed=5)
            b = _bn_run(shape, DT[name], "relu", True, True, seed=5)
            for k in ("y", "mean", "rstd", "rm", "rv", "dx", "dres", "dgamma", "dbeta", "ye"):
                assert torch.equal(a[k], b[k]), (name, shape, k)
            _bn_check(a, DT[name], tag="deterministic %s %s: " % (name, shape))
        out = _bn_accumulate(DT[name])[4]
        assert torch.equal(out["store"][0], out["accumulate"][0]), "dx depends on the accumulation mode (%s)" % name
    return True


def test_bn_deterministic_mode():
    code = "import sys; sys.path.insert(0, %r); import test_gpu_layer_shapes as t; t.check_bn_deterministic(); print('OK')" % HERE
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", code], env=env, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


# --------------------------------------------------------------------------- conditioning of the one-pass variance
BN_RATIOS = [0, 4, 16, 64, 256]
BN_DOMAIN_RATIO = 16          # |mean| / std up to which the statistics are asserted (DESIGN.md §3 states the measured errors)
BN_DOMAIN_VAR_TOL = 2e-3      # relative error of the variance inside that domain: rstd, and with it y, is off by at most 2^-10


def test_bn_conditioning_sweep(tmp_path):
    """``bn_finalize`` takes the variance as Σx²/R − mean² from fp32 sums, which cancels ~2·log2(|mean|/std) bits.  Measures the
    relative error of the variance and the error of y (γ = 1, β = 0: unit scale; also with the per-channel common shift removed)
    over |mean|/std at a short and at the longest reduction of ResNet50, writes them to ``bn_conditioning.json`` and asserts the
    variance inside the stated domain."""
    rows = []
    old = precision.precision()
    try:
        for name in ("tf32", "bf16"):
            precision.set_precision(name)
            for shape in ((64, 7, 7, 64), (64, 112, 112, 64)):
                for ratio in BN_RATIOS:
                    C = shape[-1]
                    r = _bn_run(shape, DT[name], None, False, False, seed=ratio + 1, mu=float(ratio), sigma=1.0,
                                gamma=torch.ones(C, device=DEV), beta=torch.zeros(C, device=DEV))
                    f = lo.bn_fwd64(r["x"], r["gamma"], r["beta"], EPS)
                    var_k = r["rstd"].double() ** -2 - EPS
                    d = _rows64(r["y"]) - _rows64(f["y"])
                    rows.append(dict(dtype=name, R=r["x"].numel() // C, C=C, ratio=ratio,
                                     var_rel_err=float(((var_k - f["var"]).abs() / f["var"]).max()),
                                     mean_err_over_std=float(((r["mean"].double() - f["mean"]).abs() * f["rstd"]).max()),
                                     y_abs_err=float(d.abs().max()), y_abs_err_shift_removed=float((d - d.mean(0)).abs().max())))
                    del r, f, d
    finally:
        precision.set_precision(old)
    rec = dict(card=torch.cuda.get_device_name(0), domain_ratio=BN_DOMAIN_RATIO, var_tol=BN_DOMAIN_VAR_TOL, rows=rows)
    out_dir = os.environ.get("TMPI_TEST_OUT") or str(tmp_path)
    os.makedirs(out_dir, exist_ok=True)
    with open(os.path.join(out_dir, "bn_conditioning.json"), "w") as fh:
        json.dump(rec, fh, indent=1)
    print(json.dumps(rec))
    bad = [q for q in rows if q["ratio"] <= BN_DOMAIN_RATIO and not q["var_rel_err"] <= BN_DOMAIN_VAR_TOL]
    assert not bad, bad


def _rows64(t):
    return t.double().reshape(-1, t.shape[-1])


# =========================================================================== pooling
# (mode, k, s, p, H, W, C): every pooling layer of AlexNet, GoogLeNet, ResNet50, VGG16, the CIFAR-10 net and WRN ...
POOL_MODEL = [("max", 3, 2, 1, 112, 112, 64), ("max", 3, 2, 1, 56, 56, 192), ("max", 3, 2, 1, 28, 28, 480), ("max", 3, 2, 1, 14, 14, 832),
              ("max", 3, 2, 0, 55, 55, 96), ("max", 3, 2, 0, 27, 27, 256), ("max", 3, 2, 0, 13, 13, 256), ("max", 3, 1, 1, 28, 28, 192),
              ("max", 3, 1, 1, 14, 14, 512), ("max", 3, 1, 1, 7, 7, 832), ("max", 2, 2, 0, 224, 224, 64), ("max", 2, 2, 0, 112, 112, 128),
              ("max", 2, 2, 0, 56, 56, 256), ("max", 2, 2, 0, 28, 28, 512), ("max", 2, 2, 0, 14, 14, 512), ("max", 2, 2, 0, 32, 32, 64),
              ("avg", 5, 3, 0, 14, 14, 512), ("avg", 7, 1, 0, 7, 7, 1024), ("avg", 7, 1, 0, 7, 7, 2048), ("avg", 8, 1, 0, 8, 8, 640)]
# ... and the paths no model reaches: generic-k forward and scalar backward (k = 4, 5 at stride 1), padded strided average, odd sizes,
# W != H, narrow and ragged channel counts
POOL_EDGE = [("max", 5, 1, 0, 11, 9, 16), ("max", 5, 1, 2, 12, 12, 264), ("max", 4, 1, 0, 9, 13, 8), ("max", 4, 1, 1, 10, 10, 512),
             ("max", 3, 2, 1, 15, 15, 8), ("max", 3, 2, 1, 14, 9, 264), ("max", 3, 2, 0, 15, 16, 16), ("max", 2, 2, 0, 7, 9, 520),
             ("max", 3, 1, 1, 5, 6, 264), ("max", 3, 3, 0, 12, 12, 16), ("avg", 3, 2, 1, 14, 14, 16), ("avg", 3, 2, 1, 15, 9, 264),
             ("avg", 3, 1, 1, 13, 13, 8), ("avg", 5, 3, 0, 15, 17, 512), ("avg", 2, 2, 0, 8, 8, 16)]


@pytest.mark.parametrize("inputs", ["ties", "randn"])
@pytest.mark.parametrize("N", [1, 3])
@pytest.mark.parametrize("cfg", POOL_MODEL + POOL_EDGE, ids=lambda c: "%s-k%ds%dp%d-%dx%dx%d" % c)
def test_pool(cfg, N, inputs, dtype):
    mode, k, s, p, H, W, C = cfg
    if N == 3 and H * W * C > 60 * 60 * 256:
        pytest.skip("the large images run at N = 1")
    g = _gen(H * W + C + k)
    if inputs == "ties":           # a small integer grid: equal maxima in most windows, and sums of dy that are exact in bf16
        x = torch.randint(-3, 4, (N, H, W, C), device=DEV, generator=g).to(dtype)
    else:
        x = _randn((N, H, W, C), g, dtype)
    x.requires_grad_(True)
    y = ops.pool2d(x, k, s, p, mode)
    if inputs == "ties":
        dy = torch.randint(-4, 5, tuple(y.shape), device=DEV, generator=g).to(dtype)
    else:
        dy = _randn(tuple(y.shape), g, dtype)
    y.backward(dy)
    _sync()
    y64, arg, sy = lo.pool64(x.detach(), k, s, p, mode)
    assert tuple(y.shape) == tuple(y64.shape)
    dx64, sdx = lo.pool_bwd64(dy, arg, tuple(x.shape), k, s, p, mode)
    if mode == "max":
        assert torch.equal(y.double(), y64), "max pooling is exact"
        if inputs == "ties":
            # dx makes the argmax visible: the first maximum in window order must have won, element for element
            bad = x.grad.double() != dx64
            assert not bool(bad.any()), "dx: %d elements differ; first at %s" % (
                int(bad.sum()), lo._where(int(bad.reshape(-1).to(torch.uint8).argmax()), tuple(x.shape), dtype))
        else:
            lo.assert_elementwise(x.grad, dx64, dtype, s=sdx, what="dx")
    else:
        lo.assert_elementwise(y, y64, dtype, s=sy, what="y")
        lo.assert_elementwise(x.grad, dx64, dtype, s=sdx, what="dx")


@pytest.mark.parametrize("k,s,p,H,C,split", [(3, 2, 1, 28, 192, None), (3, 2, 1, 14, 264, 128), (3, 2, 0, 27, 256, 128), (2, 2, 0, 8, 16, None)])
def test_fused_pool_relu_bias_backward(k, s, p, H, C, split):
    """The fused conv→max-pool backward (pool scatter + ReLU mask + bias gradient, bf16) with padding: its masked gradient is
    bit-equal to the plain pool backward followed by the mask, its bias gradient a sum within the bound."""
    ci = _ci()
    g = _gen(H + C)
    N = 3
    y = torch.relu(torch.randint(-2, 4, (N, H, H, C), device=DEV, generator=g).to(torch.bfloat16))
    yp, arg = ci.pool2d_fwd(y, k, s, p, "max")
    dyp = _randn(tuple(yp.shape), g, torch.bfloat16)
    db0 = torch.empty(split or C, device=DEV)
    db1 = torch.empty(C - split, device=DEV) if split else None
    dym = ci.maxpool_relu_bias_bwd(dyp, arg, y, (k, s, p, "max"), db0, db1)
    dxp = ci.pool2d_bwd_arg(dyp, arg, tuple(y.shape), k, s, p, "max")
    _sync()
    want = torch.where(y > 0, dxp, torch.zeros_like(dxp))
    assert torch.equal(dym, want)
    db = torch.cat([db0, db1]) if split else db0
    w64 = _rows64(want)
    lo.assert_reduction(db, w64.sum(0), w64.abs().sum(0), w64.shape[0], what="bias gradient")


# =========================================================================== LRN
@pytest.mark.parametrize("scale", [1.0, 20.0])
@pytest.mark.parametrize("C", [8, 64, 96, 192, 256, 2112])
@pytest.mark.parametrize("n", [3, 5, 7, 9])
def test_lrn(n, C, scale, dtype):
    """Every window the bf16 kernels are compiled for, from one channel vector (the window leaves the tensor on both sides) to
    264 vectors per row; at scale 20 the denominator departs from k."""
    g = _gen(n * 1000 + C)
    shape = (2, 5, 5, C) if C > 256 else (4, 13, 13, C)
    x = _randn(shape, g, dtype, scale).requires_grad_(True)
    y = ops.lrn(x, n)
    dy = _randn(shape, g, dtype)
    y.backward(dy)
    _sync()
    sl = _fast(dtype, 8)
    lo.assert_elementwise(y, lo.lrn64(x.detach(), n), dtype, slack=sl, what="y")
    dx64, s = lo.lrn_bwd64(x.detach(), dy, n)
    lo.assert_elementwise(x.grad, dx64, dtype, s=s, slack=sl, what="dx")


# =========================================================================== softmax + cross-entropy + top-1 / top-5
def _logits(kind, B, C, g, dtype):
    if kind == "normal":
        z = _randn((B, C), g, dtype, 3.0)
        return z, torch.randint(0, C, (B,), device=DEV, generator=g)
    if kind == "spread":            # max − min far beyond where exp underflows in fp32
        z = _randn((B, C), g, dtype, 40.0)
        return z, torch.randint(0, C, (B,), device=DEV, generator=g)
    # ties: up to 8 classes per row share the row maximum and the label is one of them, so its rank is the number of tied classes
    # with a lower index: 0 … 7, on both sides of the top-5 cut
    z = torch.randint(-8, -3, (B, C), device=DEV, generator=g).float()
    m = min(C, 8)
    top = torch.rand(B, C, device=DEV, generator=g).argsort(1)[:, :m]
    z.scatter_(1, top, 3.0)
    lab = top.gather(1, torch.randint(0, m, (B, 1), device=DEV, generator=g))[:, 0]
    return z.to(dtype), lab


@pytest.mark.parametrize("eps,grad_scale", [(0.0, 1.0), (0.0, 0.25), (0.1, 0.25), (1.0, 1.0)])
@pytest.mark.parametrize("kind", ["normal", "ties", "spread"])
@pytest.mark.parametrize("B,C", [(1, 2), (128, 10), (100, 100), (64, 1000), (16, 1003), (8, 21841)])
def test_softmax_xent(B, C, kind, eps, grad_scale, dtype):
    g = _gen(B * 7 + C)
    z, lab = _logits(kind, B, C, g, dtype)
    z.requires_grad_(True)
    with accum.mode(False, grad_scale):
        loss, e1, e5 = ops.softmax_xent(z, lab, eps)
        loss.backward()
    _sync()
    o = lo.softmax_xent64(z.detach(), lab, eps, grad_scale)
    # the error rates are counts over B: the label's rank under the tie rule, exactly
    assert round(float(e1) * B) == round(float(o["err1"]) * B) and round(float(e5) * B) == round(float(o["err5"]) * B), (
        float(e1), float(o["err1"]), float(e5), float(o["err5"]))
    assert abs(float(e1) - float(o["err1"])) <= 2.0 ** -22 and abs(float(e5) - float(o["err5"])) <= 2.0 ** -22
    lo.assert_reduction(loss.detach(), o["loss"], o["abs_loss"], B + C, what="mean loss")
    s = torch.full_like(o["dlogits"], grad_scale / B)              # dlogits are probabilities (minus the target) times scale / B
    lo.assert_elementwise(z.grad, o["dlogits"], dtype, s=s, slack=_fast(dtype, 8), what="dlogits")


# =========================================================================== dropout
@pytest.mark.parametrize("numel", [8, 2048 * 8 + 8, 128 * 4096])
@pytest.mark.parametrize("p", [1 / 65536, 0.1, 0.5, 0.9, 1 - 1 / 65536], ids=["2^-16", "0.1", "0.5", "0.9", "1-2^-16"])
def test_dropout_mask_replay(p, numel, dtype):
    """The kernel's mask is the host replay bit for bit; y = x·mask and dx = dy·mask exactly (the backward reads the mask bytes the
    forward wrote, 8 per thread in bf16 and 4 in fp32); another layer id and the next step draw other, equally correct masks."""
    ci = _ci()
    g = _gen(numel)
    x = _randn((numel // 8, 8), g, dtype)
    x = torch.where(x == 0, torch.ones_like(x), x).requires_grad_(True)          # y != 0 shows the mask
    dy = _randn((numel // 8, 8), g, dtype)
    seed = ops.rng_state()["seed"]
    step = int(ci.step_counter(x.device).item())
    zero = torch.zeros_like(dy)
    for layer, adv in ((3, 0), (4, 0), (3, 1)):
        if adv:
            ci.advance_step(x.device)
        x.grad = None
        y = ops.dropout(x, p, True, layer_id=layer)
        y.backward(dy)
        m = ref.dropout_mask_philox(numel, p, seed, layer, step + adv).view(numel // 8, 8).to(DEV)
        assert torch.equal(y.detach() != 0, m), "mask of layer %d at step +%d" % (layer, adv)
        assert torch.equal(y.detach(), torch.where(m, x.detach(), zero))
        assert torch.equal(x.grad, torch.where(m, dy, zero))
    assert ops.dropout(x, 0.0, True) is x
    ye = ops.dropout(x.detach(), p, False)
    _sync()
    lo.assert_elementwise(ye, x.detach().double() * (1.0 - p), dtype, what="eval")


# =========================================================================== small elementwise kernels
NVECS = [1, 255, 256, 257, 100001]          # 16-byte vectors: below, at and past one 256-thread CTA, and a ragged large count


@pytest.mark.parametrize("nvec", NVECS)
def test_add_kernels(nvec, dtype):
    """add, add4 and add_scaled (with and without the second operand): the fp32 result rounded once to the storage type, bit for bit."""
    ci = _ci()
    g = _gen(nvec)
    V = lo.VEC[dtype]
    a, b, c, d = (_randn((nvec * V,), g, dtype) for _ in range(4))
    y = ops.add(a, b)
    y4 = torch.empty_like(a)
    ci.L().add4_tensors(a.data_ptr(), b.data_ptr(), c.data_ptr(), d.data_ptr(), y4.data_ptr(), a.numel(), int(dtype == torch.float32), ci._st(a))
    N = 3 if nvec % 3 == 0 else 1
    s = (torch.rand(N, device=DEV, generator=g) + 0.5).float()
    a2, b2 = a.view(N, -1), b.view(N, -1)
    ys = ops.add(a2, b2, s)
    y1 = ci.add_scaled(a2, s)
    _sync()
    assert torch.equal(y, (a.float() + b.float()).to(dtype))
    assert torch.equal(y4, ((a.float() + b.float()) + (c.float() + d.float())).to(dtype))
    fma = (s.double()[:, None] * a2.double() + b2.double()).float().to(dtype)    # the product is exact in float64: one rounding, as fmaf
    assert torch.equal(ys, fma)
    assert torch.equal(y1, (s[:, None] * a2.float()).to(dtype))


@pytest.mark.parametrize("act", ["none", "relu", "leaky", "sigmoid"])
@pytest.mark.parametrize("R,C", [(1, 8), (255, 8), (256, 8), (257, 8), (100001, 8), (37, 264)])
def test_bias_act(R, C, act, dtype):
    ci = _ci()
    g = _gen(R + C)
    acc = torch.randn(R, C, device=DEV, generator=g) * 3
    bias = torch.randn(C, device=DEV, generator=g)
    y = torch.empty(R, C, device=DEV, dtype=dtype)
    ci.L().bias_act(acc.data_ptr(), bias.data_ptr(), y.data_ptr(), R, C, ci.ACT[act], ci.LEAKY_SLOPE, int(dtype == torch.float32), ci._st(acc))
    _sync()
    v = acc + bias
    if act == "sigmoid":
        lo.assert_elementwise(y, torch.sigmoid(v.double()), dtype, slack=_fast(dtype, 8), what="sigmoid")
        return
    want = {"none": v, "relu": v.clamp_min(0), "leaky": torch.where(v > 0, v, v * torch.tensor(ci.LEAKY_SLOPE, device=DEV))}[act]
    assert torch.equal(y, want.to(dtype))


@pytest.mark.parametrize("split", [False, True])
@pytest.mark.parametrize("R,C", [(1, 8), (255, 8), (257, 8), (100001, 8), (37, 264), (1000, 72)])
def test_relu_bias_bwd(R, C, split, dtype):
    """ReLU mask + bias gradient: the masked gradient exactly, the column sums within the bound; ``c_split`` sends the channels
    from C/2 on to a second bias vector (the two parameter sets of a grouped convolution)."""
    ci = _ci()
    g = _gen(R * 3 + C)
    dy, yv = _randn((R, C), g, dtype), _randn((R, C), g, dtype)
    dym = torch.empty_like(dy)
    cs = C // 2 if split else C
    db0 = torch.empty(cs, device=DEV)
    db1 = torch.empty(C - cs, device=DEV) if split else None
    ci.L().relu_bias_bwd(dy.data_ptr(), yv.data_ptr(), dym.data_ptr(), db0.data_ptr(), ci._p(db1), cs, R, C, C, 1, 0.0, 0,
                         int(dtype == torch.float32), ci._st(dy))
    _sync()
    want = torch.where(yv > 0, dy, torch.zeros_like(dy))
    assert torch.equal(dym, want)
    db = torch.cat([db0, db1]) if split else db0
    lo.assert_reduction(db, want.double().sum(0), want.double().abs().sum(0), R, what="bias gradient")
