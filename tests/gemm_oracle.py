"""float64 references of the GEMM-shaped kernels (the wgmma GEMM and the implicit / explicit convolutions of ``csrc/gemm_wgmma.*``),
written from each operation's definition, the error bound each path is held to, and the exact-integer operand generator.

Layouts are those of ``csrc``: activations NHWC, convolution weights OHWI ``[O, KH, KW, C/groups]``, transposed-convolution
weights ``[Cin, KH, KW, Cout]`` (the OHWI weight of the forward convolution that maps y-space to x-space).  Every reference runs
on the device of its inputs in float64 (a bf16 or fp32 value is exact there), one matrix product per filter tap.  Each has a
magnitude twin: the same op on |a| and |b| gives s = Σ_k |a_k|·|b_k| per output element, the scale of every rounding error.

Bounds (``bound``), per output element, for what each path does:

* bf16 operands, fp32 accumulation.  A bf16 × bf16 product is exact in fp32, so only additions round.  An element of a K-term
  product is made by at most K − 1 additions inside and between the wgmma k-steps, one per split-K partial merged by
  ``red.global.add``, one per accumulate-mode add into G and one for the bias.  Whatever the order and grouping, and whether
  the tensor core rounds or truncates each addition, every such addition changes a partial sum of terms whose magnitudes add
  up to at most s by at most one fp32 ulp, 2⁻²³ relative: |err| ≤ n_add·2⁻²³·s.  This is the bound we can prove without
  knowing how the tensor core's adder rounds; it is not tightened here.  ``GAMMA_SLACK`` allows for the (n·u)² term.
* tf32 operands (fp32 storage): add 2·u_tf32·s for the rounding of both operands to tf32.  K-major tiles reach the tensor core
  through a ``TFLOAT32`` TMA descriptor; MN-major tiles are rounded with ``cvt.rna.tf32.f32`` (round to nearest, 2⁻¹¹) in the
  shared→shared transpose.  The TMA conversion is not documented as a rounding mode; on the H100 it rounds to nearest (a K-major
  1 + 0.75·2⁻¹⁰ is read as 1 + 2⁻¹⁰, not truncated to 1: ``test_gpu_gemm_shapes.py::test_tf32_kmajor_read_rounds``), so both
  operand kinds get u = 2⁻¹¹.  Without the TFLOAT32 descriptor the tensor core would truncate (2⁻¹⁰).
* bf16 output: add 2⁻⁸·|want| (one round-to-nearest-even).
* explicit strided dgrad and transposed-convolution forward: the per-tap partial products (``dcol``) are stored in the
  activation dtype before ``col2im`` sums the taps, so add u_store·Σ_taps|partial| (``abs_partials=True`` of :func:`conv_dgrad64`).
* FC / convolutions with a leaky-ReLU or sigmoid activation: an fp32 GEMM, then ``bias_act``: fp32 accumulation plus one rounding
  of the activation's result.

Exact-integer operands (:func:`int_operands`): small integers times a power of two, so that every partial sum of every order is
an fp32 value (:func:`assert_exact_range`: Σ|a||b| < 2²⁴ units).  The result of any accumulation order, split-K, atomics or
deterministic mode is then exactly the exact sum, and the stored output exactly its rounding to the storage type.
"""
import math

import torch
import torch.nn.functional as F

from layer_oracle import _where, act_fwd64, assert_elementwise, elementwise_violations  # noqa: F401  (re-exported)

U32 = 2.0 ** -23            # one fp32 addition, rounded or truncated
U_BF16 = 2.0 ** -8          # one bf16 round-to-nearest-even
U_TF32_RNA = 2.0 ** -11     # cvt.rna.tf32.f32 (MN-major tiles)
U_TF32_KMAJOR = 2.0 ** -11  # TFLOAT32 TMA read of K-major tiles (rounds to nearest on the H100)
GAMMA_SLACK = 1.01
U_STORE_REL = {torch.bfloat16: U_BF16, torch.float32: 2.0 ** -24}     # one round-to-nearest store
MMA_K = {torch.bfloat16: 16, torch.float32: 8}
BK = {torch.bfloat16: 64, torch.float32: 32}


# --------------------------------------------------------------------------- plain GEMM
def op64(t, rows, cols, mn, ld=None):
    """The [rows, cols] logical operand of a GEMM from its storage: K-major (``mn`` False) is [rows, cols] with row pitch ``ld``,
    MN-major is [cols, rows] with row pitch ``ld`` (read transposed)."""
    t = t.double()
    if not mn:
        return torch.as_strided(t, (rows, cols), (ld or cols, 1))
    return torch.as_strided(t, (cols, rows), (ld or rows, 1)).t()


def gemm64(a, b, M, N, K, a_mn=False, b_mn=False, lda=None, ldb=None, bias=None, act=None):
    """``act(op(a)·op(b)ᵀ + bias)`` with op(a) [M, K] and op(b) [N, K] (the ``cuda_impl.gemm`` convention: B is [N, K] K-major or
    [K, N] MN-major).  Returns (want, s)."""
    A, B = op64(a, M, K, a_mn, lda), op64(b, N, K, b_mn, ldb)
    want = A @ B.t()
    s = A.abs() @ B.abs().t()
    if bias is not None:
        want = want + bias.double()[None, :]
        s = s + bias.double().abs()[None, :]
    return act_fwd64(want, act), s


# --------------------------------------------------------------------------- convolution
def out_hw(H, W, KH, KW, s, p):
    return (H + 2 * p - KH) // s + 1, (W + 2 * p - KW) // s + 1


def _taps(KH, KW):
    return [(kh, kw) for kh in range(KH) for kw in range(KW)]


def conv_fwd64(x, w, stride=1, pad=0, groups=1, bias=None, act=None):
    """y[n, i, j, o] = Σ_{kh, kw, c} x[n, s·i + kh − p, s·j + kw − p, g·Cg + c]·w[o, kh, kw, c] (+ bias[o]), zero outside the image;
    o in group g = o // (O / groups).  Returns (y, s)."""
    x, w = x.double(), w.double()
    N, H, W, C = x.shape
    O, KH, KW, Cg = w.shape
    assert Cg * groups == C and O % groups == 0
    Og = O // groups
    Ho, Wo = out_hw(H, W, KH, KW, stride, pad)
    xp = F.pad(x, (0, 0, pad, pad, pad, pad))
    y = x.new_zeros((N, Ho, Wo, O))
    s = x.new_zeros((N, Ho, Wo, O))
    for kh, kw in _taps(KH, KW):
        patch = xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride, :]
        for g in range(groups):
            pg, wg = patch[..., g * Cg:(g + 1) * Cg], w[g * Og:(g + 1) * Og, kh, kw, :]
            y[..., g * Og:(g + 1) * Og] += pg @ wg.t()
            s[..., g * Og:(g + 1) * Og] += pg.abs() @ wg.abs().t()
    if bias is not None:
        y = y + bias.double()
        s = s + bias.double().abs()
    return act_fwd64(y, act), s


def conv_dgrad64(dy, w, xshape, stride=1, pad=0, groups=1, abs_partials=False, partial_dtype=None):
    """dx[n, h, w, g·Cg + c] = Σ over the taps (kh, kw) and outputs (i, j) with s·i + kh − p = h, s·j + kw − p = w of
    Σ_o dy[n, i, j, o]·w[o, kh, kw, c].  Returns (dx, s), and with ``abs_partials`` also Σ_taps |Σ_o dy·w| (the magnitude of the
    per-tap partials that the explicit path stores before summing them).  ``partial_dtype``: round each per-tap partial to that
    storage type first, as the explicit path does (exact-integer data: the result is then the kernel's, bit for bit)."""
    dy, w = dy.double(), w.double()
    N, H, W, C = xshape
    O, KH, KW, Cg = w.shape
    Og = O // groups
    Ho, Wo = dy.shape[1], dy.shape[2]
    shp = (N, H + 2 * pad + stride, W + 2 * pad + stride, C)
    dxp, sp, pp = dy.new_zeros(shp), dy.new_zeros(shp), (dy.new_zeros(shp) if abs_partials else None)
    for kh, kw in _taps(KH, KW):
        sl = (slice(None), slice(kh, kh + stride * (Ho - 1) + 1, stride), slice(kw, kw + stride * (Wo - 1) + 1, stride))
        for g in range(groups):
            dg, wg = dy[..., g * Og:(g + 1) * Og], w[g * Og:(g + 1) * Og, kh, kw, :]
            part = dg @ wg
            if partial_dtype is not None:
                part = part.to(torch.float32).to(partial_dtype).double()
            dxp[sl + (slice(g * Cg, (g + 1) * Cg),)] += part
            sp[sl + (slice(g * Cg, (g + 1) * Cg),)] += dg.abs() @ wg.abs()
            if abs_partials:
                pp[sl + (slice(g * Cg, (g + 1) * Cg),)] += part.abs()
    crop = (slice(None), slice(pad, pad + H), slice(pad, pad + W))
    if abs_partials:
        return dxp[crop], sp[crop], pp[crop]
    return dxp[crop], sp[crop]


def conv_wgrad64(dy, x, wshape, stride=1, pad=0, groups=1):
    """dw[o, kh, kw, c] = Σ_{n, i, j} dy[n, i, j, o]·x[n, s·i + kh − p, s·j + kw − p, g·Cg + c].  Returns (dw, s)."""
    dy, x = dy.double(), x.double()
    O, KH, KW, Cg = wshape
    Og = O // groups
    N, Ho, Wo, _ = dy.shape
    xp = F.pad(x, (0, 0, pad, pad, pad, pad))
    dw = dy.new_zeros(tuple(wshape))
    s = dy.new_zeros(tuple(wshape))
    D = dy.reshape(-1, O)
    for kh, kw in _taps(KH, KW):
        patch = xp[:, kh:kh + stride * (Ho - 1) + 1:stride, kw:kw + stride * (Wo - 1) + 1:stride, :].reshape(N * Ho * Wo, -1)
        for g in range(groups):
            dg, pg = D[:, g * Og:(g + 1) * Og], patch[:, g * Cg:(g + 1) * Cg]
            dw[g * Og:(g + 1) * Og, kh, kw, :] = dg.t() @ pg
            s[g * Og:(g + 1) * Og, kh, kw, :] = dg.abs().t() @ pg.abs()
    return dw, s


def bias_grad64(dy):
    """db[o] = Σ over every axis but the last of dy; returns (db, Σ|dy|)."""
    D = dy.double().reshape(-1, dy.shape[-1])
    return D.sum(0), D.abs().sum(0)


def convT_out_hw(Hi, Wi, KH, KW, s, p, op):
    return (Hi - 1) * s - 2 * p + KH + op, (Wi - 1) * s - 2 * p + KW + op


def convT_fwd64(x, w, stride, pad, output_padding=0, partial_dtype=None):
    """Transposed convolution without bias: the input gradient of the convolution whose OHWI weight is ``w`` [Cin, KH, KW, Cout].
    Returns (y, s, Σ_taps|partial|)."""
    N, Hi, Wi, _ = x.shape
    _, KH, KW, Cout = w.shape
    H, W = convT_out_hw(Hi, Wi, KH, KW, stride, pad, output_padding)
    return conv_dgrad64(x, w, (N, H, W, Cout), stride, pad, 1, abs_partials=True, partial_dtype=partial_dtype)


# --------------------------------------------------------------------------- bounds
def n_add(K, splits=1, extra=0):
    """Upper bound on the fp32 additions on one output element's chain: K − 1 inside and between k-steps, one per split-K
    partial, ``extra`` (bias, accumulate-mode add, col2im taps)."""
    return max(int(K) - 1, 0) + int(splits) + int(extra)


def gemm_gamma(K, splits=1, extra=0):
    return GAMMA_SLACK * n_add(K, splits, extra) * U32


def bound(want, s, K, dtype, out_dtype, splits=1, extra=0, tf32_units=(U_TF32_KMAJOR, U_TF32_KMAJOR), partials=None,
          store_partials=None, operand_rel=0.0):
    """Per-element allowance of a GEMM-shaped result: γ·s (fp32 accumulation), + (u_a + u_b)·s for tf32 operands,
    + u_store·Σ|partial| where per-tap partials were stored in ``store_partials`` dtype, + 2⁻⁸·|want| for a bf16 output.
    ``tf32_units``: rounding units of the (A, B) operands on the tf32 path; ``operand_rel``: relative error of one operand that
    was itself rounded before the product (a leaky / sigmoid gradient stored in the activation dtype)."""
    want = want.double()
    b = gemm_gamma(K, splits, extra) * s
    if dtype == torch.float32:
        b = b + (tf32_units[0] + tf32_units[1]) * s
    if operand_rel:
        b = b + operand_rel * s
    if partials is not None and store_partials is not None:
        b = b + U_STORE_REL[store_partials] * partials
    if out_dtype == torch.bfloat16:
        b = b + U_BF16 * want.abs()
    return b


def check(got, want, bnd, what, ratios=None, family=None):
    """|got − want| ≤ bnd everywhere (a NaN is a violation); a failure names the (n, h, w, c) or (r, c) of the worst element.
    ``ratios``: a dict that collects the largest diff / bound per ``family``."""
    g = got.detach().double().to(want.device)
    assert g.shape == want.shape, (what, tuple(g.shape), tuple(want.shape))
    diff = (g - want).abs()
    bad = ~(diff <= bnd)
    nbad = int(bad.sum())
    if ratios is not None and family is not None and diff.numel():
        r = float((diff / bnd.clamp_min(1e-300)).max())
        ratios[family] = max(ratios.get(family, 0.0), r)
    if nbad:
        excess = torch.where(bad, diff / bnd.clamp_min(1e-300), torch.zeros_like(diff))
        excess = torch.where(torch.isnan(excess), torch.full_like(excess, float("inf")), excess)
        w = int(excess.reshape(-1).argmax())
        dt = got.dtype if got.dtype in (torch.bfloat16, torch.float32) else torch.float32
        raise AssertionError("%s: %d of %d elements outside the bound; worst at %s: got %r want %r (|diff| %.3g, bound %.3g)" % (
            what, nbad, bad.numel(), _where(w, tuple(want.shape), dt), float(g.reshape(-1)[w]), float(want.reshape(-1)[w]),
            float(diff.reshape(-1)[w]), float(bnd.reshape(-1)[w])))


def round_to(want64, dtype):
    """The exact value rounded once to the storage type (exact integers below 2²⁴ pass through fp32 unchanged)."""
    return want64.to(dtype)


def assert_exact(got, want64, what):
    """Bitwise: ``got`` is exactly the exact result rounded to its storage type; a failure names the first mismatch."""
    exp = round_to(want64, got.dtype).to(got.device)
    if torch.equal(got, exp):
        return
    ne = (got != exp) | (torch.isnan(got) != torch.isnan(exp))
    idx = ne.reshape(-1).nonzero()
    first = int(idx[0])
    raise AssertionError("%s: %d of %d elements differ from the exact result; first at %s: got %r want %r (exact %r)" % (
        what, int(ne.sum()), ne.numel(), _where(first, tuple(exp.shape), got.dtype if got.dtype in (torch.bfloat16, torch.float32)
                                                else torch.float32),
        float(got.reshape(-1)[first]), float(exp.reshape(-1)[first]), float(want64.reshape(-1)[first])))


# --------------------------------------------------------------------------- exact-integer operands
def int_operands(shape, gen, device, lo=-2, hi=2, scale_exp=0, density=1.0, dtype=torch.float32):
    """Integers in [lo, hi] (zero with probability 1 − ``density``) times 2^``scale_exp``: exact in bf16 and in tf32."""
    v = torch.randint(lo, hi + 1, tuple(shape), generator=gen, device=device, dtype=torch.int32).double()
    if density < 1.0:
        v = v * (torch.rand(tuple(shape), generator=gen, device=device, dtype=torch.float64) < density)
    return (v * 2.0 ** scale_exp).to(dtype)


def assert_exact_range(s, unit=1.0):
    """Every partial sum of every order is an fp32 value: Σ|a||b| < 2²⁴ units (``s`` the magnitude of the products)."""
    top = float(s.max()) / unit if s.numel() else 0.0
    assert top < 2 ** 24, "integer operands too large to be exact in fp32: max Σ|a||b| = %g units" % top
    assert float((s / unit - (s / unit).round()).abs().max() if s.numel() else 0.0) == 0.0, "operands are not integers in the unit"
    return top


def tie_fraction(want64):
    """Share of the elements whose exact value is a bf16 round-to-nearest-even tie (|v| in (256, 2¹⁶), odd at the bf16 step)."""
    a = want64.abs()
    e = torch.floor(torch.log2(a.clamp_min(1.0)))
    step = 2.0 ** (e - 7)
    half = (a / step) - torch.floor(a / step)
    return float(((a > 256) & (half == 0.5)).double().mean()) if a.numel() else 0.0


def bf16_round(x):
    """bf16 round-to-nearest-even of a float64 tensor, in float64 (the value a bf16 store keeps)."""
    return x.to(torch.float32).to(torch.bfloat16).double()


# --------------------------------------------------------------------------- the models' GEMM-shaped layers
# (model, default batch, "conv", H, W, C, O, KH, KW, stride, pad, groups, act, bias) / (model, batch, "fc", in, out, act), recorded
# from the models at batch 1 (test_gemm_oracle_cpu.py::test_model_shapes_are_in_the_table) and deduplicated per model.  AlexNet's
# 2-group layers are listed with their total channels; C = "cp" is the GAN image padded to 16 bytes (8 bf16 / 4 fp32 channels).
MODEL_LAYERS = [
    ("alexnet", 128, "conv", 227, 227, 3, 96, 11, 11, 4, 0, 1, "relu", True),
    ("alexnet", 128, "conv", 27, 27, 96, 256, 5, 5, 1, 2, 2, "relu", True),
    ("alexnet", 128, "conv", 13, 13, 256, 384, 3, 3, 1, 1, 1, "relu", True),
    ("alexnet", 128, "conv", 13, 13, 384, 384, 3, 3, 1, 1, 2, "relu", True),
    ("alexnet", 128, "conv", 13, 13, 384, 256, 3, 3, 1, 1, 2, "relu", True),
    ("alexnet", 128, "fc", 9216, 4096, "relu"),
    ("alexnet", 128, "fc", 4096, 4096, "relu"),
    ("alexnet", 128, "fc", 4096, 1000, "none"),
    ("cifar10", 256, "conv", 28, 28, 3, 64, 5, 5, 1, 0, 1, "relu", True),
    ("cifar10", 256, "conv", 12, 12, 64, 128, 5, 5, 1, 0, 1, "relu", True),
    ("cifar10", 256, "conv", 4, 4, 128, 64, 3, 3, 1, 0, 1, "relu", True),
    ("cifar10", 256, "fc", 256, 256, "relu"),
    ("cifar10", 256, "fc", 256, 10, "none"),
    ("wrn", 128, "conv", 32, 32, 3, 16, 3, 3, 1, 1, 1, "none", False),
    ("wrn", 128, "conv", 32, 32, 16, 64, 1, 1, 1, 0, 1, "none", False),
    ("wrn", 128, "conv", 32, 32, 16, 64, 3, 3, 1, 1, 1, "none", False),
    ("wrn", 128, "conv", 32, 32, 64, 64, 3, 3, 1, 1, 1, "none", False),
    ("wrn", 128, "conv", 32, 32, 64, 128, 1, 1, 2, 0, 1, "none", False),
    ("wrn", 128, "conv", 32, 32, 64, 128, 3, 3, 2, 1, 1, "none", False),
    ("wrn", 128, "conv", 16, 16, 128, 128, 3, 3, 1, 1, 1, "none", False),
    ("wrn", 128, "conv", 16, 16, 128, 256, 1, 1, 2, 0, 1, "none", False),
    ("wrn", 128, "conv", 16, 16, 128, 256, 3, 3, 2, 1, 1, "none", False),
    ("wrn", 128, "conv", 8, 8, 256, 256, 3, 3, 1, 1, 1, "none", False),
    ("wrn", 128, "fc", 256, 10, "none"),
    ("googlenet", 32, "conv", 224, 224, 3, 64, 7, 7, 2, 3, 1, "relu", True),
    ("googlenet", 32, "conv", 56, 56, 64, 64, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 56, 56, 64, 192, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 192, 64, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 192, 96, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 96, 128, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 192, 16, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 16, 32, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 192, 32, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 256, 128, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 128, 192, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 256, 32, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 32, 96, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 28, 28, 256, 64, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 480, 192, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 480, 96, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 96, 208, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 480, 16, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 16, 48, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 480, 64, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 160, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 112, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 112, 224, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 24, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 24, 64, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 64, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 128, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 128, 256, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 144, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 144, 288, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 512, 32, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 32, 64, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 528, 256, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 528, 160, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 160, 320, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 528, 32, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 32, 128, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 14, 14, 528, 128, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 256, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 160, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 160, 320, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 32, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 32, 128, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 128, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 384, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 192, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 192, 384, 3, 3, 1, 1, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 832, 48, 1, 1, 1, 0, 1, "relu", True),
    ("googlenet", 32, "conv", 7, 7, 48, 128, 5, 5, 1, 2, 1, "relu", True),
    ("googlenet", 32, "fc", 1024, 1000, "none"),
    ("resnet50", 32, "conv", 224, 224, 3, 64, 7, 7, 2, 3, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 64, 256, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 64, 64, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 64, 64, 3, 3, 1, 1, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 256, 64, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 256, 512, 1, 1, 2, 0, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 256, 128, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 56, 56, 128, 128, 3, 3, 2, 1, 1, "none", False),
    ("resnet50", 32, "conv", 28, 28, 128, 512, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 28, 28, 512, 128, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 28, 28, 128, 128, 3, 3, 1, 1, 1, "none", False),
    ("resnet50", 32, "conv", 28, 28, 512, 1024, 1, 1, 2, 0, 1, "none", False),
    ("resnet50", 32, "conv", 28, 28, 512, 256, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 28, 28, 256, 256, 3, 3, 2, 1, 1, "none", False),
    ("resnet50", 32, "conv", 14, 14, 256, 1024, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 14, 14, 1024, 256, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 14, 14, 256, 256, 3, 3, 1, 1, 1, "none", False),
    ("resnet50", 32, "conv", 14, 14, 1024, 2048, 1, 1, 2, 0, 1, "none", False),
    ("resnet50", 32, "conv", 14, 14, 1024, 512, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 14, 14, 512, 512, 3, 3, 2, 1, 1, "none", False),
    ("resnet50", 32, "conv", 7, 7, 512, 2048, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 7, 7, 2048, 512, 1, 1, 1, 0, 1, "none", False),
    ("resnet50", 32, "conv", 7, 7, 512, 512, 3, 3, 1, 1, 1, "none", False),
    ("resnet50", 32, "fc", 2048, 1000, "none"),
    ("vgg16", 32, "conv", 224, 224, 3, 64, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 224, 224, 64, 64, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 112, 112, 64, 128, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 112, 112, 128, 128, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 56, 56, 128, 256, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 56, 56, 256, 256, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 28, 28, 256, 512, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 28, 28, 512, 512, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "conv", 14, 14, 512, 512, 3, 3, 1, 1, 1, "relu", True),
    ("vgg16", 32, "fc", 25088, 4096, "relu"),
    ("vgg16", 32, "fc", 4096, 4096, "relu"),
    ("vgg16", 32, "fc", 4096, 1000, "none"),
    # NativeWGAN / NativeLSGAN (batch 64, 28x28 images): the critic's leaky-ReLU first conv and its strided second conv
    ("gan", 64, "conv", 28, 28, "cp", 64, 5, 5, 2, 2, 1, "leaky", True),
    ("gan", 64, "conv", 14, 14, 64, 128, 5, 5, 2, 2, 1, "none", True),
    ("gan", 64, "fc", 100, 1024, "none"),
    ("gan", 64, "fc", 1024, 6272, "none"),
    ("gan", 64, "fc", 6272, 1024, "none"),
    ("gan", 64, "fc", 1024, 1, "none"),
]
# the generator's transposed convolutions: (model, batch, Hi, Wi, Cin, Cout, K, stride, pad, output_padding, act, c_real)
MODEL_CONVT = [
    ("gan", 64, 7, 7, 128, 64, 5, 2, 2, 1, "none", None),
    ("gan", 64, 14, 14, 64, "cp", 5, 2, 2, 1, "sigmoid", 1),
]
# AlexNet's conv -> max-pool blocks (conv layer index in MODEL_LAYERS -> pool (k, s, p)): one autograd node, fused backward
ALEX_POOL = {0: (3, 2, 0), 1: (3, 2, 0), 4: (3, 2, 0)}
# the LSTM (dim_proj 128, batch 16, sequences of 20 to 80 steps): its embedding-to-gates FC over T·B rows, the recurrent
# step GEMMs and the output head are listed by the LSTM tests of test_gpu_gemm_shapes.py
LSTM_H, LSTM_B, LSTM_T = 128, 16, (20, 80)


def layer_channels(c, dtype):
    return (8 if dtype == torch.bfloat16 else 4) if c == "cp" else c


def first_layer(i):
    """True for the first GEMM layer of each model (its input is the image: no input gradient)."""
    return i == 0 or MODEL_LAYERS[i - 1][0] != MODEL_LAYERS[i][0]


# --------------------------------------------------------------------------- launch plans (host arithmetic of csrc/gemm_wgmma.cu)
SMS = 132                   # H100 SXM
FPROP, DGRAD, WGRAD = 0, 1, 2


def gemm_plan(L, M, N, K, f32, a_mn=False, b_mn=False, out_bf16=True, fused=False, splitk=0, accumulate=False, sms=SMS):
    """(BN, MT, splits) that ``gemm_host`` launches for a plain GEMM (mirrors its tile-width rule; splits / tall tiles come from the
    exported planners)."""
    bk = 32 if f32 else 64
    if f32:
        out_bf16 = False
    can_split = not out_bf16 and not fused
    mt = ceil_div(M, 128)
    bn = 128
    if not (can_split and splitk != 1):
        if mt * ceil_div(N, 128) < sms and N >= 64:
            bn = 64
        if bn == 64 and mt * ceil_div(N, 64) < sms and not b_mn and N >= 32:
            bn = 32
    elif N <= 64:
        bn = 64
    if b_mn and bn < 64:
        bn = 64
    nt = ceil_div(N, bn)
    num_kb = ceil_div(K, bk)
    splits = 1
    if splitk > 1 and can_split:
        splits = splitk
    elif splitk == 0 and can_split:
        splits = L.gemm_plan_splits(mt * nt, num_kb, sms)
    kb_per = ceil_div(num_kb, splits)
    splits = ceil_div(num_kb, kb_per)
    tall_ok = out_bf16 if not f32 else (not a_mn and not b_mn)
    tall = splits == 1 and bn >= 64 and L.gemm_plan_tall(M, nt, int(bool(tall_ok)), sms)
    return bn, 2 if tall else 1, splits


def ceil_div(a, b):
    return -(-a // b)


def conv_plans(L, layer, batch, f32, sms=SMS):
    """{pass: ("implicit" | "gemm", BN, MT, splits)} of one MODEL_LAYERS conv at ``batch`` as ``cuda_impl`` dispatches it."""
    _, _, _, H, W, C, O, KH, KW, s, p, g, act, _bias = layer
    C = layer_channels(C, torch.float32 if f32 else torch.bfloat16)
    al, bk = (4, 32) if f32 else (8, 64)
    Cg, Og = C // g, O // g
    Ho, Wo = out_hw(H, W, KH, KW, s, p)
    M = batch * Ho * Wo
    out = {}
    ngroups = 2 if g == 2 else 1
    if act in ("leaky", "sigmoid"):
        Kp = ceil_div(KH * KW * Cg, 8) * 8
        out["fprop"] = ("gemm",) + gemm_plan(L, M, O, KH * KW * Cg, f32, out_bf16=False)
        out["wgrad"] = ("gemm",) + gemm_plan(L, O, KH * KW * Cg, M, f32, True, True, out_bf16=False)
        out["dgrad"] = ("gemm",) + gemm_plan(L, M, Kp, O, f32, False, True, out_bf16=True)
        return out
    if C < 8 and C % 4 and s > 1:                      # space-to-depth stem
        S = s
        Hs, KHs = ceil_div(H + 2 * p, S), ceil_div(KH, S)
        Cp = ceil_div(S * S * C, 8) * 8
        nkb = KHs * ceil_div(KW, S) * ceil_div(Cp, bk)
        out["fprop"] = ("implicit",) + tuple(L.gemm_plan_conv(FPROP, M, O, 1, nkb, 1, sms))
        out["wgrad"] = ("implicit",) + tuple(L.gemm_plan_conv(WGRAD, O, KHs * ceil_div(KW, S) * ceil_div(Cp, bk) * bk, 1,
                                                              ceil_div(M, bk), 0, sms))
        return out
    if Cg % al or C % al:                              # explicit im2col (first layers on RGB)
        K = KH * KW * Cg
        out["fprop"] = ("gemm",) + gemm_plan(L, M, Og, K, f32, fused=True)
        out["wgrad"] = ("gemm",) + gemm_plan(L, Og, K, M, f32, True, True, out_bf16=False)
        return out
    out["fprop"] = ("implicit",) + tuple(L.gemm_plan_conv(FPROP, M, Og, ngroups, KH * KW * ceil_div(Cg, bk), 1, sms))
    out["wgrad"] = ("implicit",) + tuple(L.gemm_plan_conv(WGRAD, Og, KH * KW * ceil_div(Cg, bk) * bk, ngroups, ceil_div(M, bk), 0, sms))
    if s == 1:
        out["dgrad"] = ("implicit",) + tuple(L.gemm_plan_conv(DGRAD, batch * H * W, Cg, ngroups, KH * KW * ceil_div(Og, bk),
                                                              0 if f32 else 1, sms))
    else:
        Kp = ceil_div(KH * KW * Cg, 8) * 8
        out["dgrad"] = ("gemm",) + gemm_plan(L, M, Kp, Og, f32, False, True, out_bf16=True)
    return out


def test_batch(L, layer):
    """The smallest batch (1, 2, 4, … up to the model's default) whose launch plans equal the default batch's for every pass in
    both precisions; the default itself when none does."""
    default = layer[1]
    if layer[2] != "conv":
        return default
    want = [conv_plans(L, layer, default, f32) for f32 in (False, True)]
    b = 1
    while b < default:
        if [conv_plans(L, layer, b, f32) for f32 in (False, True)] == want:
            return b
        b *= 2
    return default
