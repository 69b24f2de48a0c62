"""CUDA implementations of the functional ops: thin, checked wrappers that hand raw
device pointers of torch tensors to the hand-written sm_90a kernels in ``csrc/``.

GEMM-shaped work (FC forward/dgrad/wgrad; conv forward/dgrad/wgrad through an NHWC
im2col gather) runs on ONE kernel, ``gemm`` (TMA → smem → ``wgmma`` →
registers → fused epilogue, see ``csrc/gemm_wgmma.cu``).  Operand-major flags make
transposed copies unnecessary:

    forward   y  = x · Wᵀ        A = x   (K-major)   B = W   (K-major)   + bias + ReLU → bf16
    dgrad     dx = dy · W        A = dy  (K-major)   B = W   (MN-major)               → bf16
    wgrad     dW = dyᵀ · x       A = dy  (MN-major)  B = x   (MN-major)  split-K      → fp32 (straight into the arena's G)

Gradient accumulation (:mod:`.accum`): while the switch is on, every kernel that writes a parameter gradient into an arena G view
adds into it instead (GEMM / implicit-conv wgrad through the epilogue's fp32 reductions, bias and batch-norm gradients without their
clears).  A gradient of a parameter without a G view goes to a fresh scratch buffer, which is stored into as without the switch
(``functional._sink`` then adds it into its destination).

Everything raises if the extension is missing — there is no eager fallback on a GPU.
"""
from __future__ import annotations

import numpy as np
import torch

from . import accum, native, precision

_STEP = {}          # device index -> int64[1] step counter used by the dropout Philox stream
BF16 = torch.bfloat16
F32 = torch.float32


def ADT():
    """Activation dtype of the active precision mode (bf16, or fp32 for the tf32 path)."""
    return precision.act_dtype()


def _is32(t):
    return t.dtype == F32


ACT = {"none": 0, "relu": 1, "leaky": 2, "sigmoid": 3}     # activation codes of the native kernels (ACT_* in csrc/common.cuh)
LEAKY_SLOPE = 0.2                                          # negative slope of "leaky" (the DCGAN critic's LeakyReLU(0.2))


def _act(relu):
    """Activation code of a ``relu`` argument: a bool (ReLU or identity) or an activation name from :data:`ACT`."""
    return ACT[relu] if isinstance(relu, str) else int(bool(relu))


def _al(t):
    """Elements per 16 bytes (TMA / vector alignment unit): 8 for bf16, 4 for fp32."""
    return 16 // t.element_size()


def L():
    return native.require()


def _st(t):
    return torch.cuda.current_stream(t.device).cuda_stream


def _p(t):
    return 0 if t is None else t.data_ptr()


def _acc(*outs):
    """1 while the backward accumulates (:mod:`.accum`) and one of ``outs`` — the parameter-gradient outputs of one launch — is a G
    view, so the launch adds; else 0 (the launch stores)."""
    return int(accum.accumulating() and any(o is not None for o in outs))


def grad_buffer(shape, out=None, device=None, acc=0):
    """``out`` (a parameter's gradient view in the arena), else a fresh fp32 scratch buffer: uninitialised, since the launch stores
    into it, or zeros when ``acc`` — the launch that writes it also adds into another output that is a G view (two parameter sets
    in one launch, only one of them with a view)."""
    if out is not None:
        return out
    return (torch.zeros if acc else torch.empty)(shape, dtype=torch.float32, device=device)


def step_counter(device):
    idx = torch.device(device).index
    if idx is None:
        idx = torch.cuda.current_device()
    if idx not in _STEP:
        _STEP[idx] = torch.zeros(1, dtype=torch.int64, device=torch.device("cuda", idx))
    return _STEP[idx]


def advance_step(device):
    s = step_counter(device)
    L().advance_step(s.data_ptr(), _st(s))


def _bf(t):
    """Cast to the activation dtype of the active precision mode (no-op on the hot path: layers already produce it)."""
    d = ADT()
    return t if t.dtype == d else t.to(d)


def _rows8(t2d):
    """Return a 2-D tensor whose row pitch is a multiple of 16 bytes (TMA rule) — the tensor itself when it already is, else
    a zero-padded copy (rare, tiny shapes)."""
    assert t2d.dim() == 2
    al = _al(t2d)
    if t2d.stride(1) == 1 and t2d.stride(0) % al == 0 and t2d.data_ptr() % 16 == 0:
        return t2d, t2d.stride(0)
    R, C = t2d.shape
    ld = (C + al - 1) // al * al
    out = torch.zeros((R, ld), dtype=t2d.dtype, device=t2d.device)
    out[:, :C] = t2d
    return out, ld


# --------------------------------------------------------------------------- GEMM
def gemm(a, b, M, N, K, a_mn=False, b_mn=False, out=None, out_dtype=None, bias=None, bias_mode=0,
         relu=False, alpha=1.0, lda=None, ldb=None, ldc=None, bn=0, splitk=0, accumulate=False):
    """``out[M,N] = alpha * op(a) @ op(b) (+bias)(ReLU)``; ``a``/``b`` are bf16 tensors whose
    storage is described by (major flag, leading dimension).  ``accumulate``: ``out += alpha * op(a) @ op(b)`` (fp32 ``out``, no
    bias / ReLU)."""
    dev = a.device
    tf32 = _is32(a)
    assert a.dtype == b.dtype, "GEMM operands must share a dtype"
    if out is None:
        out = torch.empty((M, N), dtype=(F32 if tf32 else (out_dtype or BF16)), device=dev)
    if ldc is None:
        ldc = out.stride(0) if out.dim() == 2 else N
    if bias is not None:
        assert bias.dtype == torch.float32
    if accumulate:
        assert out.dtype == torch.float32 and bias is None and not relu, "an accumulating GEMM adds an fp32 product into out"
    L().gemm(a.data_ptr(), b.data_ptr(), out.data_ptr(), _p(bias), int(M), int(N), int(K), int(lda), int(ldb),
             int(ldc), int(bool(a_mn)), int(bool(b_mn)), int(out.dtype == BF16), int(bias_mode), int(bool(relu)),
             float(alpha), int(bn), int(splitk), int(tf32), _st(a), int(bool(accumulate)))
    return out


# --------------------------------------------------------------------------- linear
def linear_bias_act(x, w, b, relu=True):
    x2 = _bf(x).contiguous()
    B_, I = x2.shape
    O = w.shape[0]
    xa, lda = _rows8(x2)
    wa, ldb = _rows8(_bf(w))
    bias = b.float() if b is not None and b.dtype != torch.float32 else b
    if (B_ <= 128 and I >= 1024 and O % 8 == 0) or _act(relu) > 1:
        # small-batch FC forward is a weight stream: one m-tile, so the parallelism comes from n-tiles x split-K (fp32
        # reductions into a scratch tile), followed by a tiny bias + ReLU (+ bf16 cast) pass; fp32 output is finished in
        # place.  (The fused-epilogue kernel needs 32-wide tiles to fill the machine and then re-reads the activations 128
        # times through L2: 37 us vs 13 us for fc6.)  Leaky ReLU / sigmoid are not in the GEMM epilogue and take this path too.
        f32 = _is32(x2)
        acc = gemm(xa, wa, B_, O, I, out_dtype=torch.float32, lda=lda, ldb=ldb)
        y = acc if f32 else torch.empty((B_, O), dtype=BF16, device=x2.device)
        L().bias_act(acc.data_ptr(), _p(bias), y.data_ptr(), int(B_), int(O), _act(relu), LEAKY_SLOPE, int(f32), _st(x2))
        return y
    return gemm(xa, wa, B_, O, I, bias=bias, bias_mode=1 if b is not None else 0, relu=relu, lda=lda, ldb=ldb)


def _mask_and_bias_grad(dy, y, relu, db_out, R, C, ld, need_db=True, acc=None):
    """dym = dy ⊙ act'(y) (ReLU: dy ⊙ (y > 0); contiguous [R, C]) and db = Σ_rows dym in one pass.  ``acc``: add into ``db_out``
    (default: while accumulating, when ``db_out`` is a G view)."""
    dev = dy.device
    act = _act(relu)
    if not need_db and not act and ld == C:
        return dy, None                                    # bias-free linear conv (a BatchNormal follows): nothing to do
    acc = _acc(db_out) if acc is None else int(acc)
    db = grad_buffer(C, db_out, dev)
    if act or ld != C:
        dym = torch.empty((R, C), dtype=dy.dtype, device=dev)
        L().relu_bias_bwd(dy.data_ptr(), _p(y), dym.data_ptr(), db.data_ptr(), 0, int(C), int(R), int(C), int(ld), _act(relu), LEAKY_SLOPE,
                          acc, int(_is32(dy)), _st(dy))
    else:
        dym = dy
        L().relu_bias_bwd(dy.data_ptr(), 0, 0, db.data_ptr(), 0, int(C), int(R), int(C), int(ld), 0, 0.0, acc, int(_is32(dy)), _st(dy))
    return dym, db


def maxpool_relu_bias_bwd(dyp, arg, y, pool, db0, db1=None, accumulate=False):
    """Backward of conv(+ReLU)→max-pool up to the conv's masked output gradient, in one kernel: scatter the pooled
    gradient through the argmax, apply the ReLU mask, reduce the bias gradient(s) into ``db0`` (/ ``db1``), or add it there with
    ``accumulate``.  Returns dym, shaped like y."""
    dyp = _bf(dyp).contiguous()
    N, H, W, C = y.shape
    Ho, Wo = dyp.shape[1], dyp.shape[2]
    k, s_, p_ = int(pool[0]), int(pool[1]), int(pool[2])
    dym = torch.empty((N, H, W, C), dtype=BF16, device=y.device)
    c_split = C if db1 is None else int(db0.numel())
    L().maxpool_relu_bias_bwd(dyp.data_ptr(), arg.data_ptr(), y.data_ptr(), dym.data_ptr(), db0.data_ptr(), _p(db1), c_split,
                              N, H, W, C, Ho, Wo, k, s_, p_, int(bool(accumulate)), _st(y))
    return dym


def gemm_sgd(a, b, p, M, N, K, lda, ldb):
    """Weight gradient ``op(a)^T op(b)`` of the armed parameter ``p`` (``utils.opt.FlatSGD.arm``) applied as its momentum-SGD
    step inside the GEMM epilogue: ``p`` (fp32 master in the arena), its momentum and its bf16 shadow are updated in place and
    the gradient is never written.  Same arithmetic and lr source (``arena.hyper[0]``) as ``flat_update(arena, "sgd", ...)``."""
    arena, sgd = p.arena, p.sgd_epilogue
    lrm, wd, _ = _table(arena)
    g = p.arena_group
    off = p.arena_off
    u = arena.U[off:off + p.numel()]
    L().gemm_sgd(a.data_ptr(), b.data_ptr(), p.data_ptr(), u.data_ptr(), _p(p.shadow), arena.hyper.data_ptr(), float(lrm[g]),
                 float(wd[g]), float(sgd.mu), int(bool(sgd.nesterov)), 1.0, int(M), int(N), int(K), int(lda), int(ldb),
                 int(p.shape[1]), int(_is32(a)), _st(a))


def linear_bias_act_bwd(x, w, y, dy, relu, need_dx, dw_out=None, db_out=None, sgd_param=None):
    """``sgd_param``: the master weight armed for the SGD epilogue (see :func:`gemm_sgd`); its gradient is then applied rather
    than returned (``dw`` is None)."""
    x2 = _bf(x).contiguous()
    dy = _bf(dy).contiguous()
    B_, I = x2.shape
    O = w.shape[0]
    al = _al(x2)
    if sgd_param is not None and accum.accumulating():
        raise RuntimeError("linear_bias_act_bwd: weight %s is armed for the GEMM SGD epilogue, which does not accumulate gradients"
                           % (tuple(w.shape),))
    if O % al or I % al:
        if sgd_param is not None:
            raise RuntimeError("linear_bias_act_bwd: weight %s is armed for the GEMM SGD epilogue but needs the padded path"
                               % (tuple(w.shape),))
        return _linear_bwd_padded(x2, w, y, dy, relu, need_dx, dw_out, db_out)
    dym, db = _mask_and_bias_grad(dy, y, relu, db_out.view(-1) if db_out is not None else None, B_, O, O)
    wb = _bf(w)
    dx = None
    if need_dx:
        dx = gemm(dym, wb, B_, I, O, a_mn=False, b_mn=True, lda=O, ldb=I)
    if sgd_param is not None:
        # after the dx GEMM, which reads the weights of this step
        gemm_sgd(dym, x2, sgd_param, O, I, B_, lda=O, ldb=I)
        return dx, None, db
    dw = grad_buffer((O, I), dw_out, x.device)
    gemm(dym, x2, O, I, B_, a_mn=True, b_mn=True, out=dw, lda=O, ldb=I, ldc=I, accumulate=_acc(dw_out))
    return dx, dw, db


def _linear_bwd_padded(x2, w, y, dy, relu, need_dx, dw_out, db_out):
    """Shapes whose pitches violate the 16-byte TMA rule (e.g. a 10-class test head): pad to 8.  The padded product goes to a
    scratch buffer, so an accumulating backward adds it into the gradient views afterwards."""
    B_, I = x2.shape
    O = w.shape[0]
    Op, Ip = (O + 7) // 8 * 8, (I + 7) // 8 * 8
    dev = x2.device
    dt = x2.dtype
    from .reference import act_bwd
    dyf = act_bwd(dy.float(), y.float(), relu)
    db = dyf.sum(0)
    dyp = torch.zeros((B_, Op), dtype=dt, device=dev); dyp[:, :O] = dyf
    xp = torch.zeros((B_, Ip), dtype=dt, device=dev); xp[:, :I] = x2
    wp = torch.zeros((Op, Ip), dtype=dt, device=dev); wp[:O, :I] = w
    dx = gemm(dyp, wp, B_, Ip, Op, b_mn=True, lda=Op, ldb=Ip)[:, :I].contiguous() if need_dx else None
    dwp = torch.empty((Op, Ip), dtype=torch.float32, device=dev)
    gemm(dyp, xp, Op, Ip, B_, a_mn=True, b_mn=True, out=dwp, lda=Op, ldb=Ip, ldc=Ip)
    dw = dwp[:O, :I]
    acc = accum.accumulating()
    if dw_out is not None:
        (dw_out.add_ if acc else dw_out.copy_)(dw); dw = dw_out
    if db_out is not None:
        (db_out.view(-1).add_ if acc else db_out.view(-1).copy_)(db); db = db_out
    return dx, dw, db


# --------------------------------------------------------------------------- conv (NHWC, im2col + wgmma GEMM)
def _out_hw(H, W, KH, KW, s, p):
    return (H + 2 * p - KH) // s + 1, (W + 2 * p - KW) // s + 1


def _im2col(x, c_off, Cg, KH, KW, Ho, Wo, s, p):
    N, H, W, Ct = x.shape
    K = KH * KW * Cg
    al = _al(x)
    if KH == 1 and KW == 1 and s == 1 and p == 0 and c_off == 0 and Cg == Ct and Ct % al == 0:
        return x.view(N * H * W, Ct), Ct, K                     # 1x1 conv: the activation IS the matrix
    Kp = (K + 7) // 8 * 8
    col = torch.empty((N * Ho * Wo, Kp), dtype=x.dtype, device=x.device)
    L().im2col(x.data_ptr(), col.data_ptr(), N, H, W, Ct, int(c_off), int(Cg), KH, KW, Ho, Wo, int(s), int(p), Kp, int(_is32(x)), _st(x))
    return col, Kp, K


def _w2d(w, K, Kp):
    """OHWI bf16 weights as the GEMM's [O, Kp] K-major operand (zero-padded when K % 8 != 0)."""
    O = w.shape[0]
    w2 = _bf(w).reshape(O, K)
    if Kp == K and w2.data_ptr() % 16 == 0:
        return w2
    wp = torch.empty((O, Kp), dtype=w2.dtype, device=w.device)
    L().pad_rows(w2.data_ptr(), wp.data_ptr(), O, K, K, Kp, int(_is32(w2)), _st(w))
    return wp


def _implicit_ok(x, w, c_off, Cg, Ot, o_off):
    """TMA im2col needs 16-byte aligned channel slices; C = 3 (first layer) stays on the explicit path."""
    Ct = x.shape[3]
    al = _al(x)
    return (Cg % al == 0 and c_off % al == 0 and Ct % al == 0 and Ot % al == 0 and o_off % al == 0
            and w.shape[0] % al == 0 and w.is_contiguous() and w.data_ptr() % 16 == 0)


def _conv_fwd_group(x, w, b, y, o_off, c_off, Cg, s, p, relu):
    N, H, W, Ct = x.shape
    Og, KH, KW, _ = w.shape
    Ho, Wo = y.shape[1], y.shape[2]
    Ot = y.shape[3]
    wb = _bf(w)
    if _implicit_ok(x, wb, c_off, Cg, Ot, o_off):
        # implicit GEMM: the activation tile is gathered by TMA im2col loads inside the kernel — no col matrix
        yp = y.data_ptr() + o_off * y.element_size()
        L().conv_fprop(x.data_ptr(), wb.data_ptr(), yp, _p(b), N, H, W, Ct, int(c_off), int(Cg), KH, KW, Ho, Wo, int(s), int(p),
                       Og, Ot, int(bool(relu)), 0, int(_is32(x)), _st(x))
        return None
    col, Kp, K = _im2col(x, c_off, Cg, KH, KW, Ho, Wo, s, p)
    w2 = _w2d(w, K, Kp)
    M = N * Ho * Wo
    yv = y.view(M, Ot)[:, o_off:o_off + Og]
    gemm(col, w2, M, Og, K, out=yv, bias=b, bias_mode=1 if b is not None else 0, relu=relu, lda=Kp, ldb=Kp, ldc=Ot)
    return (col, Kp, K)


def _s2d_geom(H, W, C, KH, KW, stride, pad):
    """Geometry of the space-to-depth rewrite of a strided few-channel conv, or None when it does not apply.  The zero padding
    of the original convolution is folded into the space-to-depth image (the kernel reads x[S*i + dy - pad, ...])."""
    if not (C < 8 and C % 4 != 0 and stride > 1):
        return None
    S = stride
    Hp, Wp = H + 2 * pad, W + 2 * pad
    Hs, Ws = -(-Hp // S), -(-Wp // S)
    KHs, KWs = -(-KH // S), -(-KW // S)
    Ho, Wo = _out_hw(H, W, KH, KW, stride, pad)
    if Hs - KHs + 1 != Ho or Ws - KWs + 1 != Wo:
        return None
    Cp = (S * S * C + 7) // 8 * 8
    return S, Hs, Ws, KHs, KWs, Cp, Ho, Wo, int(pad)


def _conv_s2d_fwd(x, w, b, relu, g):
    """First-layer conv (e.g. AlexNet 11x11/4 on RGB) as a stride-1 conv on the space-to-depth image (implicit GEMM)."""
    S, Hs, Ws, KHs, KWs, Cp, Ho, Wo, P0 = g
    N, H, W, C = x.shape
    O, KH, KW, _ = w.shape
    dev = x.device
    f32 = int(_is32(x))
    xs = torch.empty((N, Hs, Ws, Cp), dtype=x.dtype, device=dev)
    ws = torch.empty((O, KHs, KWs, Cp), dtype=x.dtype, device=dev)
    L().space_to_depth(x.data_ptr(), xs.data_ptr(), N, H, W, C, S, Hs, Ws, Cp, P0, f32, _st(x))
    L().s2d_filter(_bf(w).contiguous().data_ptr(), ws.data_ptr(), O, KH, KW, C, S, KHs, KWs, Cp, 0, f32, _st(x))
    y = torch.empty((N, Ho, Wo, O), dtype=x.dtype, device=dev)
    L().conv_fprop(xs.data_ptr(), ws.data_ptr(), y.data_ptr(), _p(b), N, Hs, Ws, Cp, 0, Cp, KHs, KWs, Ho, Wo, 1, 0, O, O,
                   int(bool(relu)), 0, f32, _st(x))
    return y, xs


def _conv_s2d_bwd(xs, w, y, dy, relu, g, dw_out, db_out, pre_masked=False):
    S, Hs, Ws, KHs, KWs, Cp, Ho, Wo, P0 = g
    O, KH, KW, C = w.shape
    N = xs.shape[0]
    M = N * Ho * Wo
    dev = xs.device
    if pre_masked:
        dym, db = dy, db_out
    else:
        dym, db = _mask_and_bias_grad(dy.view(M, O), y.view(M, O), relu, db_out.view(-1) if db_out is not None else None, M, O, O)
    dws = torch.empty((O, KHs, KWs, Cp), dtype=torch.float32, device=dev)
    f32 = int(_is32(xs))
    L().conv_wgrad(dym.data_ptr(), xs.data_ptr(), dws.data_ptr(), N, Hs, Ws, Cp, 0, Cp, KHs, KWs, Ho, Wo, 1, 0, O, O, 0, f32, _st(xs))
    dw = grad_buffer((O, KH, KW, C), dw_out, dev)
    # the space-to-depth gradient is scratch: it is stored, and the unpack adds it into dw while the backward accumulates
    L().s2d_filter(dws.data_ptr(), dw.data_ptr(), O, KH, KW, C, S, KHs, KWs, Cp, 2 if _acc(dw_out) else 1, f32, _st(xs))
    return dw, db


def _conv_fwd_act(x, w, b, s, p, act, Ho, Wo):
    """Convolution followed by an activation the GEMM epilogue does not have (leaky ReLU, sigmoid): im2col, an fp32-output GEMM,
    then one bias + activation pass.  Returns (y, the im2col matrix for the backward)."""
    N = x.shape[0]
    O, KH, KW, _ = w.shape
    col, Kp, K = _im2col(x, 0, x.shape[3], KH, KW, Ho, Wo, s, p)
    M = N * Ho * Wo
    acc = gemm(col, _w2d(w, K, Kp), M, O, K, out_dtype=torch.float32, lda=Kp, ldb=Kp)
    f32 = _is32(x)
    y = acc.view(N, Ho, Wo, O) if f32 else torch.empty((N, Ho, Wo, O), dtype=BF16, device=x.device)
    L().bias_act(acc.data_ptr(), _p(b), y.data_ptr(), int(M), int(O), _act(act), LEAKY_SLOPE, int(f32), _st(x))
    return y, (col, Kp, K)


def conv2d_bias_act(x, w, b, stride=1, pad=0, groups=1, relu=True, return_cols=False):
    x = _bf(x).contiguous()
    N, H, W, C = x.shape
    O, KH, KW, Cg = w.shape
    assert Cg * groups == C
    if _act(relu) > 1:
        if groups != 1:
            raise RuntimeError("leaky ReLU / sigmoid convolutions are single-group")
        y, col = _conv_fwd_act(x, w, b, stride, pad, relu, *_out_hw(H, W, KH, KW, stride, pad))
        return (y, [col]) if return_cols else y
    g = _s2d_geom(H, W, C, KH, KW, stride, pad) if (groups == 1 and O % 8 == 0) else None
    if g is not None:
        y, xs = _conv_s2d_fwd(x, w, b, relu, g)
        return (y, [("s2d", xs, g)]) if return_cols else y
    Ho, Wo = _out_hw(H, W, KH, KW, stride, pad)
    y = torch.empty((N, Ho, Wo, O), dtype=x.dtype, device=x.device)
    Og = O // groups
    cols = []
    for g in range(groups):
        cols.append(_conv_fwd_group(x, w[g * Og:(g + 1) * Og], None if b is None else b[g * Og:(g + 1) * Og], y, g * Og,
                                    g * Cg, Cg, stride, pad, relu))
    return (y, cols) if return_cols else y


def _relu_only(relu, what):
    if _act(relu) > 1:
        raise RuntimeError("%s supports ReLU or no activation only" % what)


def conv2d_group2_bias_act(x, w0, b0, w1, b1, stride, pad, relu, return_cols=False):
    _relu_only(relu, "conv2d_group2_bias_act")
    x = _bf(x).contiguous()
    N, H, W, C = x.shape
    Og, KH, KW, Cg = w0.shape
    Ho, Wo = _out_hw(H, W, KH, KW, stride, pad)
    y = torch.empty((N, Ho, Wo, 2 * Og), dtype=x.dtype, device=x.device)
    wb0, wb1 = _bf(w0), _bf(w1)
    es, f32 = x.element_size(), int(_is32(x))
    if _implicit_ok(x, wb0, 0, Cg, 2 * Og, 0) and _implicit_ok(x, wb1, Cg, Cg, 2 * Og, Og) and (b0 is None) == (b1 is None):
        # both groups in ONE persistent launch: their tiles fill the SMs together instead of two under-filled waves
        L().conv_fprop2(x.data_ptr(), wb0.data_ptr(), wb1.data_ptr(), y.data_ptr(), y.data_ptr() + Og * es, _p(b0), _p(b1), N, H, W, C, 0,
                        int(Cg), int(Cg), KH, KW, Ho, Wo, int(stride), int(pad), Og, 2 * Og, int(bool(relu)), 0, f32, _st(x))
        return (y, [None, None]) if return_cols else y
    cols = [_conv_fwd_group(x, w0, b0, y, 0, 0, Cg, stride, pad, relu),
            _conv_fwd_group(x, w1, b1, y, Og, Cg, Cg, stride, pad, relu)]
    return (y, cols) if return_cols else y


def _conv_bwd_group(x, w, y, dy, dx, o_off, c_off, Cg, s, p, relu, need_dx, dw_out, db_out, col=None, pre_masked=False, need_db=True,
                    acc_w=None, acc_b=None):
    """``acc_w`` / ``acc_b``: add the weight / bias gradient into ``dw_out`` / ``db_out`` (default: while accumulating, when the
    output is a G view)."""
    acc_w = _acc(dw_out) if acc_w is None else int(acc_w)
    N, H, W, Ct = x.shape
    Og, KH, KW, _ = w.shape
    Ho, Wo, Ot = y.shape[1], y.shape[2], y.shape[3]
    M = N * Ho * Wo
    dev = x.device
    dyv = dy.view(M, Ot)[:, o_off:o_off + Og]
    yv = y.view(M, Ot)[:, o_off:o_off + Og]
    if pre_masked:
        # dy already carries the ReLU mask and db is already accumulated (fused pool backward): the GEMMs read this
        # group's channel slice of the full tensor in place (row pitch Ot)
        dym, db, ldy, dy_coff = dyv, db_out, Ot, o_off
    else:
        dym, db = _mask_and_bias_grad(dyv, yv, relu, db_out.view(-1) if db_out is not None else None, M, Og, Ot, need_db, acc=acc_b)
        ldy, dy_coff = Og, 0
    wb = _bf(w)
    if col is None and _implicit_ok(x, wb, c_off, Cg, Ot, o_off):
        # ---- implicit GEMM backward: wgrad gathers im2col(x) by TMA; dgrad (stride 1) is a forward conv of dy with the
        # flipped / transposed filter, written straight into dx's channel slice.
        dw = grad_buffer((Og, KH, KW, Cg), dw_out, dev)
        es, f32 = x.element_size(), int(_is32(x))
        L().conv_wgrad(dym.data_ptr(), x.data_ptr(), dw.data_ptr(), N, H, W, Ct, int(c_off), int(Cg), KH, KW, Ho, Wo, int(s), int(p),
                       Og, int(ldy), acc_w, f32, _st(x))
        if need_dx:
            if s == 1:
                # dgrad = forward conv of dy with the mirrored, transposed filter — which the kernel's TMA loads read straight
                # out of the forward weights (MN-major boxes of the mirrored tap): no flipped copy
                L().conv_fprop(dym.data_ptr() - dy_coff * es, wb.data_ptr(), dx.data_ptr() + c_off * es, 0, N, Ho, Wo, int(ldy), int(dy_coff),
                               Og, KH, KW, H, W, 1, KH - 1 - int(p), int(Cg), Ct, 0, 1, f32, _st(x))
            else:
                colK = KH * KW * Cg
                Kp = (colK + 7) // 8 * 8
                dcol = gemm(dym, _w2d(w, colK, Kp), M, Kp, Og, b_mn=True, lda=ldy, ldb=Kp)
                L().col2im(dcol.data_ptr(), dx.data_ptr(), N, H, W, Ct, int(c_off), int(Cg), KH, KW, Ho, Wo, int(s), int(p), Kp, f32, _st(x))
        return dw, db
    col, Kp, K = col if col is not None else _im2col(x, c_off, Cg, KH, KW, Ho, Wo, s, p)   # forward's matrix is reused
    dw = grad_buffer((Og, KH, KW, Cg), dw_out, dev)
    # wgrad: dW[Og, K] = dymᵀ[Og, M] · col[M, K]   (both operands MN-major, split-K over M)
    gemm(dym, col, Og, K, M, a_mn=True, b_mn=True, out=dw.view(Og, K), lda=ldy, ldb=Kp, ldc=K, accumulate=acc_w)
    if need_dx:
        w2 = _w2d(w, K, Kp)
        one_by_one = (KH == 1 and KW == 1 and s == 1 and p == 0 and c_off == 0 and Cg == Ct)
        if one_by_one:
            gemm(dym, w2, M, Kp, Og, b_mn=True, out=dx.view(M, Ct), lda=ldy, ldb=Kp, ldc=Ct)
        else:
            dcol = gemm(dym, w2, M, Kp, Og, b_mn=True, lda=ldy, ldb=Kp)
            L().col2im(dcol.data_ptr(), dx.data_ptr(), N, H, W, Ct, int(c_off), int(Cg), KH, KW, Ho, Wo, int(s), int(p), Kp,
                       int(_is32(x)), _st(x))
    return dw, db


def conv2d_bias_act_bwd(x, w, y, dy, stride, pad, groups, relu, need_dx, dw_out=None, db_out=None, cols=None, pre_masked=False,
                        need_db=True):
    x = _bf(x).contiguous()
    dy = _bf(dy).contiguous()
    N, H, W, C = x.shape
    O, KH, KW, Cg = w.shape
    if cols and isinstance(cols[0], tuple) and len(cols[0]) == 3 and isinstance(cols[0][0], str) and cols[0][0] == "s2d":
        if need_dx:
            raise RuntimeError("space-to-depth conv path is for the first layer only (no input gradient)")
        dw, db = _conv_s2d_bwd(cols[0][1], w, y, dy, relu, cols[0][2], dw_out, db_out, pre_masked)
        return None, dw, db
    if (Cg % _al(x) or O % _al(x)) and need_dx:
        raise RuntimeError("conv dgrad needs channel counts that are multiples of 16 bytes")
    dx = torch.empty_like(x) if need_dx else None
    Og = O // groups
    if groups == 1:
        dw, db = _conv_bwd_group(x, w, y, dy, dx, 0, 0, Cg, stride, pad, relu, need_dx, dw_out, db_out,
                                 col=cols[0] if cols else None, pre_masked=pre_masked, need_db=need_db)
        return dx, dw, db
    acc_w, acc_b = _acc(dw_out), _acc(db_out)
    dw = grad_buffer(tuple(w.shape), dw_out, x.device)
    db = grad_buffer(O, db_out, x.device)
    for g in range(groups):
        _conv_bwd_group(x, w[g * Og:(g + 1) * Og], y, dy, dx, g * Og, g * Cg, Cg, stride, pad, relu, need_dx,
                        dw[g * Og:(g + 1) * Og], db[g * Og:(g + 1) * Og], col=cols[g] if cols else None, pre_masked=pre_masked,
                        acc_w=acc_w, acc_b=acc_b)
    return dx, dw, db


def conv2d_group2_bias_act_bwd(x, w0, w1, y, dy, stride, pad, relu, need_dx, outs=(None, None, None, None), cols=None,
                               pre_masked=False):
    _relu_only(relu, "conv2d_group2_bias_act_bwd")
    x = _bf(x).contiguous()
    dy = _bf(dy).contiguous()
    Og, KH, KW, Cg = w0.shape
    dx = torch.empty_like(x) if need_dx else None
    wb0, wb1 = _bf(w0), _bf(w1)
    Ot = 2 * Og
    no_cols = not cols or (cols[0] is None and cols[1] is None)
    if (no_cols and _implicit_ok(x, wb0, 0, Cg, Ot, 0) and _implicit_ok(x, wb1, Cg, Cg, Ot, Og)
            and (not need_dx or stride == 1)):
        # ---- both groups per launch: one mask/bias pass over the full width, one wgrad launch, one dgrad launch
        N, H, W, Ct = x.shape
        Ho, Wo = y.shape[1], y.shape[2]
        M = N * Ho * Wo
        dev = x.device
        # one launch writes both groups' bias (weight) gradients: it adds when either output is a G view
        acc_b, acc_w = _acc(outs[1], outs[3]), _acc(outs[0], outs[2])
        db0, db1 = grad_buffer(Og, outs[1], dev, acc_b), grad_buffer(Og, outs[3], dev, acc_b)
        es, f32 = x.element_size(), int(_is32(x))
        if pre_masked:
            dym = dy
        else:
            dym = torch.empty((M, Ot), dtype=x.dtype, device=dev)
            L().relu_bias_bwd(dy.data_ptr(), y.data_ptr(), dym.data_ptr(), db0.data_ptr(), db1.data_ptr(), int(Og), int(M), int(Ot), int(Ot),
                              _act(relu), LEAKY_SLOPE, acc_b, f32, _st(x))
        dw0, dw1 = grad_buffer((Og, KH, KW, Cg), outs[0], dev, acc_w), grad_buffer((Og, KH, KW, Cg), outs[2], dev, acc_w)
        L().conv_wgrad2(dym.data_ptr(), dym.data_ptr() + Og * es, x.data_ptr(), dw0.data_ptr(), dw1.data_ptr(), N, H, W, Ct, 0, int(Cg), int(Cg),
                        KH, KW, Ho, Wo, int(stride), int(pad), Og, int(Ot), acc_w, f32, _st(x))
        if need_dx:
            L().conv_fprop2(dym.data_ptr(), wb0.data_ptr(), wb1.data_ptr(), dx.data_ptr(), dx.data_ptr() + Cg * es, 0, 0, N, Ho, Wo, int(Ot), 0,
                            int(Og), int(Og), KH, KW, H, W, 1, KH - 1 - int(pad), int(Cg), Ct, 0, 1, f32, _st(x))
        return dx, (dw0, db0, dw1, db1)
    dw0, db0 = _conv_bwd_group(x, w0, y, dy, dx, 0, 0, Cg, stride, pad, relu, need_dx, outs[0], outs[1],
                               col=cols[0] if cols else None, pre_masked=pre_masked)
    dw1, db1 = _conv_bwd_group(x, w1, y, dy, dx, Og, Cg, Cg, stride, pad, relu, need_dx, outs[2], outs[3],
                               col=cols[1] if cols else None, pre_masked=pre_masked)
    return dx, (dw0, db0, dw1, db1)


# --------------------------------------------------------------------------- transposed convolution (NHWC)
def _convT_out_hw(Hi, Wi, KH, KW, s, p, op):
    return (Hi - 1) * s - 2 * p + KH + op, (Wi - 1) * s - 2 * p + KW + op


def conv_transpose2d_bias_act(x, w, b, stride, pad, output_padding=0, relu=False, c_real=None):
    """Transposed convolution = the input gradient of a stride-``stride`` convolution: ``y = act(col2im(x · W) + b)``.

    ``w`` is ``[Cin, KH, KW, Cout]``, the OHWI weight of the forward convolution that maps y-space to x-space.  The product is
    the wgmma GEMM (x K-major, W MN-major); the gather, bias and activation are one ``col2im_bias_act`` pass.  Output channels
    ``>= c_real`` (zero padding of a layer narrower than 16 bytes) are written as zeros; that needs ReLU or sigmoid, whose
    backward mask is zero at a zero output, so the padded channels get zero gradient whatever the consumer sends back."""
    x = _bf(x).contiguous()
    N, Hi, Wi, Cin = x.shape
    _, KH, KW, Cout = w.shape
    assert w.shape[0] == Cin and 0 <= output_padding < stride
    if c_real is not None and c_real < Cout and _act(relu) not in (ACT["relu"], ACT["sigmoid"]):
        raise RuntimeError("conv_transpose2d: padded output channels need a ReLU or sigmoid activation")
    if Cin % _al(x) or Cout % _al(x):
        raise RuntimeError("conv_transpose2d: channel counts must be multiples of 16 bytes")
    H, W = _convT_out_hw(Hi, Wi, KH, KW, stride, pad, output_padding)
    K = KH * KW * Cout
    Kp = (K + 7) // 8 * 8
    dcol = gemm(x.view(-1, Cin), _w2d(w, K, Kp), N * Hi * Wi, Kp, Cin, b_mn=True, lda=Cin, ldb=Kp)
    y = torch.empty((N, H, W, Cout), dtype=x.dtype, device=x.device)
    L().col2im_bias_act(dcol.data_ptr(), y.data_ptr(), _p(b), N, H, W, Cout, KH, KW, Hi, Wi, int(stride), int(pad), Kp, _act(relu), LEAKY_SLOPE,
                        int(Cout if c_real is None else c_real), int(_is32(x)), _st(x))
    return y


def conv_transpose2d_bias_act_bwd(x, w, y, dy, stride, pad, relu, need_dx, dw_out=None, db_out=None):
    """Backward of :func:`conv_transpose2d_bias_act`: the activation mask and bias gradient in one pass, ``dx`` = the forward
    convolution of the masked gradient with the same weight, ``dW`` = that convolution's weight gradient with the roles of its
    input and output gradient swapped (x is the "output gradient", the masked dy the "input").  Padded output channels have
    y = 0, where the ReLU / sigmoid mask is 0: their weight and bias gradients are exactly zero."""
    x = _bf(x).contiguous()
    dy = _bf(dy).contiguous()
    N, H, W, Cout = y.shape
    M = N * H * W
    dym, db = _mask_and_bias_grad(dy.view(M, Cout), y.view(M, Cout), relu, db_out.view(-1) if db_out is not None else None, M, Cout, Cout)
    dym = dym.view(N, H, W, Cout)
    dx = conv2d_bias_act(dym, w, None, stride, pad, 1, False) if need_dx else None
    _, dw, _ = conv2d_bias_act_bwd(dym, w, x, x, stride, pad, 1, False, False, dw_out=dw_out, pre_masked=True, need_db=False)
    return dx, dw, db


# --------------------------------------------------------------------------- pool / LRN / dropout / loss
def pool2d_fwd(x, ksize, stride, pad, mode):
    x = _bf(x).contiguous()
    N, H, W, C = x.shape
    Ho, Wo = _out_hw(H, W, ksize, ksize, stride, pad)
    y = torch.empty((N, Ho, Wo, C), dtype=x.dtype, device=x.device)
    is_max = mode == "max"
    arg = torch.empty((N, Ho, Wo, C), dtype=torch.uint8, device=x.device) if is_max else None
    L().pool_fwd(x.data_ptr(), y.data_ptr(), _p(arg), N, H, W, C, Ho, Wo, int(ksize), int(stride), int(pad), int(is_max), int(_is32(x)),
                 _st(x))
    return y, arg


def pool2d_bwd_arg(dy, arg, xshape, ksize, stride, pad, mode):
    dy = _bf(dy).contiguous()
    N, H, W, C = xshape
    Ho, Wo = dy.shape[1], dy.shape[2]
    dx = torch.empty(tuple(xshape), dtype=dy.dtype, device=dy.device)
    L().pool_bwd(dy.data_ptr(), _p(arg), dx.data_ptr(), N, H, W, C, Ho, Wo, int(ksize), int(stride), int(pad), int(mode == "max"),
                 int(_is32(dy)), _st(dy))
    return dx


def lrn(x, n=5, k=2.0, alpha=1e-4, beta=0.75):
    x = _bf(x).contiguous()
    C = x.shape[-1]
    y = torch.empty_like(x)
    L().lrn_fwd(x.data_ptr(), y.data_ptr(), x.numel() // C, C, int(n), float(k), float(alpha), float(beta), int(_is32(x)), _st(x))
    return y, None


def lrn_bwd(x, dy, n=5, k=2.0, alpha=1e-4, beta=0.75):
    x = _bf(x).contiguous()
    dy = _bf(dy).contiguous()
    C = x.shape[-1]
    dx = torch.empty_like(x)
    L().lrn_bwd(x.data_ptr(), dy.data_ptr(), dx.data_ptr(), x.numel() // C, C, int(n), float(k), float(alpha), float(beta), int(_is32(x)),
                _st(x))
    return dx


def dropout_fwd(x, p_drop, layer_id):
    from .functional import rng_state
    x = _bf(x).contiguous()
    y = torch.empty_like(x)
    mask = torch.empty(x.shape, dtype=torch.uint8, device=x.device)
    step = step_counter(x.device)
    L().dropout_fwd(x.data_ptr(), y.data_ptr(), mask.data_ptr(), x.numel(), float(p_drop), int(rng_state()["seed"]), int(layer_id),
                    step.data_ptr(), int(_is32(x)), _st(x))
    return y, mask


def dropout_bwd(dy, mask):
    dy = _bf(dy).contiguous()
    dx = torch.empty_like(dy)
    L().dropout_bwd(dy.data_ptr(), mask.data_ptr(), dx.data_ptr(), dy.numel(), int(_is32(dy)), _st(dy))
    return dx


def softmax_xent(logits, labels, weight=1.0, grad_scale=1.0, label_smoothing=0.0, mix=None):
    """(weight · mean NLL, top-1 error, top-5 error, dlogits); dlogits is the gradient of the mean NLL times weight · grad_scale
    (``grad_scale`` = 1/n under gradient accumulation over n micro-batches), scaled in fp32 inside the kernel.  ``label_smoothing``
    ε > 0 makes the loss and dlogits those of the soft target (1 − ε)·onehot + ε / C, in the same launch.  ``mix`` (the step's
    Mixup / CutMix record on the device, ops/mixup.py) launches the mixing instantiation instead: the target is
    λ·s(y_i) + (1 − λ)·s(y_j) with j = B − 1 − i (see reference.softmax_xent_mix)."""
    lg = _bf(logits).contiguous()
    B_, C = lg.shape
    labels = labels.contiguous()
    assert labels.dtype == torch.int64
    dl = torch.empty_like(lg)
    rowstat = torch.empty((B_, 3), dtype=torch.float32, device=lg.device)
    out3 = torch.empty(3, dtype=torch.float32, device=lg.device)
    if mix is None:
        L().softmax_xent(lg.data_ptr(), labels.data_ptr(), dl.data_ptr(), rowstat.data_ptr(), out3.data_ptr(), B_, C, float(weight),
                         float(weight) * float(grad_scale), float(label_smoothing), int(_is32(lg)), _st(lg))
    else:
        _check_record(mix, lg.device)
        L().softmax_xent_mix(lg.data_ptr(), labels.data_ptr(), mix.data_ptr(), dl.data_ptr(), rowstat.data_ptr(), out3.data_ptr(), B_, C,
                             float(weight), float(weight) * float(grad_scale), float(label_smoothing), int(_is32(lg)), _st(lg))
    return out3[0], out3[1], out3[2], dl


def softmax_xent_kd(logits, labels, teacher, alpha, temperature, grad_scale=1.0, label_smoothing=0.0, mix=None):
    """Knowledge distillation against the teacher's logits ``teacher`` (same shape and dtype as ``logits``): (mean L, top-1 error,
    top-5 error, dlogits) with L = (1 − α)·CE_q(z) + α·T²·KL(softmax(t/T) ‖ softmax(z/T)) per row, q the target of :func:`softmax_xent`
    (``label_smoothing`` ε, ``mix``), and dlogits = [(1 − α)·(p − q) + α·T·(softmax(z/T) − softmax(t/T))] / B times ``grad_scale``,
    scaled in fp32 inside the kernel.  One ``softmax_xent_kd`` launch and one ``rowstat_mean`` (reference.softmax_xent_kd)."""
    lg = _bf(logits).contiguous()
    t = _bf(teacher).contiguous()
    B_, C = lg.shape
    if t.shape != lg.shape or t.dtype != lg.dtype:
        raise ValueError("softmax_xent_kd: the teacher's logits %s %s do not match the student's %s %s"
                         % (tuple(t.shape), t.dtype, tuple(lg.shape), lg.dtype))
    labels = labels.contiguous()
    assert labels.dtype == torch.int64
    dl = torch.empty_like(lg)
    rowstat = torch.empty((B_, 3), dtype=torch.float32, device=lg.device)
    out3 = torch.empty(3, dtype=torch.float32, device=lg.device)
    if mix is not None:
        _check_record(mix, lg.device)
    L().softmax_xent_kd(lg.data_ptr(), t.data_ptr(), labels.data_ptr(), 0 if mix is None else mix.data_ptr(), dl.data_ptr(),
                        rowstat.data_ptr(), out3.data_ptr(), B_, C, float(grad_scale), float(label_smoothing), float(alpha),
                        float(temperature), int(_is32(lg)), _st(lg))
    return out3[0], out3[1], out3[2], dl


def _check_record(rec, device):
    from .mixup import RECORD_BYTES
    if not (rec.is_cuda and rec.device == device and rec.dtype == torch.uint8 and rec.is_contiguous() and rec.numel() % RECORD_BYTES == 0
            and rec.data_ptr() % 8 == 0):
        raise ValueError("a mix record is a contiguous uint8 tensor of %d bytes on %s" % (RECORD_BYTES, device))


def mix_draw(cfg, rank, hw, step, n=1, out=None):
    """``n`` Mixup / CutMix records (uint8 [n · 64] on the step counter's device, or into ``out``): record t is the draw of step
    counter value ``*step + t`` (one ``mix_draw_kernel`` launch that reads the int64 device counter ``step``, so a replayed CUDA graph
    draws anew); ``cfg`` is a validated ``config['mixup']``, ``hw`` the image size at the mix point.  reference.mix_draw makes the
    same draw on the CPU."""
    from .mixup import RECORD_BYTES
    rec = out if out is not None else torch.empty(n * RECORD_BYTES, dtype=torch.uint8, device=step.device)
    _check_record(rec, step.device)
    if rec.numel() != n * RECORD_BYTES:
        raise ValueError("mix_draw: %d records need %d bytes, not %d" % (n, n * RECORD_BYTES, rec.numel()))
    L().mix_draw(float(cfg["alpha"]), float(cfg["cutmix_alpha"]), float(cfg["switch_prob"]), float(cfg["prob"]), int(cfg["seed"]),
                 int(rank), int(hw[0]), int(hw[1]), step.data_ptr(), rec.data_ptr(), int(n), _st(step))
    return rec


def mix_batch(x, rec):
    """Mix the NHWC batch ``x`` in place as the device record ``rec`` says (one ``mix_batch_kernel`` launch; 16-byte vectors when a
    row of H·W·C elements is a multiple of 16 bytes, else one element per thread).  Returns ``x``."""
    if x.dim() != 4 or not x.is_contiguous() or x.dtype not in (BF16, F32):
        raise ValueError("mix_batch: needs a contiguous bf16 or fp32 NHWC batch, not %s %s" % (x.dtype, tuple(x.shape)))
    _check_record(rec, x.device)
    B_, H, W, C = x.shape
    L().mix_batch(x.data_ptr(), rec.data_ptr(), B_, H, W, C, int(_is32(x)), _st(x))
    return x


def gan_loss(scores, kind, a):
    """GAN loss over a ``[B, 1]`` (or ``[B]``) score vector and its gradient in one launch; see :func:`reference.gan_loss`."""
    sc = _bf(scores).contiguous()
    d = torch.empty_like(sc)
    out = torch.empty(1, dtype=F32, device=sc.device)
    L().gan_loss(sc.data_ptr(), d.data_ptr(), out.data_ptr(), int(sc.numel()), {"wgan": 0, "lsgan": 1}[kind], float(a), int(_is32(sc)), _st(sc))
    return out[0], d


def uniform_noise(shape, seed, stream, step, dtype=None):
    """Uniform [0, 1) noise from Philox keyed by (seed, stream) and the int64 device step counter ``step`` (read by the kernel, so
    every replay of a captured step draws fresh numbers); :func:`reference.uniform_noise` draws the same numbers on the CPU."""
    out = torch.empty(tuple(shape), dtype=dtype or ADT(), device=step.device)
    L().uniform_noise(out.data_ptr(), out.numel(), int(seed), int(stream), step.data_ptr(), int(_is32(out)), _st(step))
    return out


# --------------------------------------------------------------------------- batch norm (+ residual)(+ ReLU), residual add
def _drop_row(drop, x):
    """A drop-path row for ``x``: contiguous fp32 on x's device, one scale per sample of x's leading axis."""
    if not (drop.is_cuda and drop.device == x.device and drop.dtype == F32 and drop.is_contiguous() and drop.numel() == x.shape[0]):
        raise ValueError("a drop-path row is a contiguous fp32 tensor of %d scales on %s" % (x.shape[0], x.device))
    return drop


def batch_norm_fwd(x, gamma, beta, run_mean, run_var, training, momentum, eps, relu, res=None, drop=None):
    """``drop``: a drop-path row (needs ``res``), y = act(s_n·(γ·x̂ + β) + res) in the apply pass (reference.batch_norm_fwd)."""
    x = _bf(x).contiguous()
    C = x.shape[-1]
    R = x.numel() // C
    dev = x.device
    y = torch.empty_like(x)
    mean = torch.empty(C, dtype=F32, device=dev)
    rstd = torch.empty(C, dtype=F32, device=dev)
    scratch = torch.empty(2 * C, dtype=F32, device=dev)
    if res is not None:
        res = _bf(res).contiguous()
        assert res.shape == x.shape
    assert gamma.dtype == F32 and beta.dtype == F32
    if not training:
        assert run_mean is not None and run_var is not None
    L().bn_forward(x.data_ptr(), _p(res), y.data_ptr(), gamma.data_ptr(), beta.data_ptr(), mean.data_ptr(), rstd.data_ptr(),
                   _p(run_mean), _p(run_var), scratch.data_ptr(), int(R), int(C), float(momentum), float(eps), int(bool(training)),
                   _act(relu), LEAKY_SLOPE, _p(drop if drop is None else _drop_row(drop, x)), int(x.shape[0]), int(_is32(x)), _st(x))
    return y, mean, rstd


def batch_norm_bwd(x, dy, y, gamma, mean, rstd, relu, need_dres, dgamma_out=None, dbeta_out=None, drop=None):
    """``drop``: the forward's drop-path row; dx, dγ and dβ come from s_n·g, dres is g (reference.batch_norm_bwd)."""
    x = _bf(x).contiguous()
    dy = _bf(dy).contiguous()
    C = x.shape[-1]
    R = x.numel() // C
    dev = x.device
    dx = torch.empty_like(x)
    # without a ReLU the residual branch receives dy itself: nothing to write
    dres = torch.empty_like(x) if (need_dres and relu) else None
    acc = _acc(dgamma_out, dbeta_out)
    dgamma = grad_buffer(C, dgamma_out.view(-1) if dgamma_out is not None else None, dev, acc)
    dbeta = grad_buffer(C, dbeta_out.view(-1) if dbeta_out is not None else None, dev, acc)
    # accumulating: the batch's Σg, Σg·x̂ go to the scratch (the dx coefficients need them, not the running totals in G)
    scratch = torch.empty((5 if acc else 3) * C, dtype=F32, device=dev)
    L().bn_backward(x.data_ptr(), dy.data_ptr(), _p(y) if relu else 0, dx.data_ptr(), _p(dres), gamma.data_ptr(), mean.data_ptr(),
                    rstd.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), scratch.data_ptr(), int(R), int(C), _act(relu), LEAKY_SLOPE,
                    acc, _p(drop if drop is None else _drop_row(drop, x)), int(x.shape[0]), int(_is32(x)), _st(x))
    if need_dres and not relu:
        dres = dy
    return dx, dres, dgamma, dbeta


def add(a, b):
    a = _bf(a).contiguous()
    b = _bf(b).contiguous()
    assert a.shape == b.shape
    y = torch.empty_like(a)
    L().add_tensors(a.data_ptr(), b.data_ptr(), y.data_ptr(), a.numel(), int(_is32(a)), _st(a))
    return y


def add_scaled(a, s, b=None):
    """y = s_n·a + b per sample n of the leading axis (``b`` None: s_n·a), ``s`` a drop-path row: one ``add_scaled_kernel`` launch
    (each sample's elements must fill whole 16-byte vectors)."""
    a = _bf(a).contiguous()
    if b is not None:
        b = _bf(b).contiguous()
        assert b.shape == a.shape
    y = torch.empty_like(a)
    L().add_scaled(a.data_ptr(), _p(b), _drop_row(s, a).data_ptr(), y.data_ptr(), a.numel(), int(a.shape[0]), int(_is32(a)), _st(a))
    return y


def drop_path_draw(dp, step, out):
    """The drop-path table of the device step counter ``step`` into ``out`` (fp32 [L, B]) for :class:`drop_path.DropPath` ``dp``,
    keyed by the dropout seed and dp's rank: one ``drop_path_draw_kernel`` launch (reference.drop_path_draw on the CPU)."""
    from .functional import rng_state
    if not (out.is_cuda and out.dtype == F32 and out.is_contiguous() and tuple(out.shape) == (dp.L, dp.B) and out.device == step.device):
        raise ValueError("drop_path_draw: the table is a contiguous fp32 [%d, %d] tensor on %s" % (dp.L, dp.B, step.device))
    L().drop_path_draw(dp.thresh.data_ptr(), dp.keep.data_ptr(), dp.L, dp.B, int(rng_state()["seed"]) & (2 ** 64 - 1), dp.rank,
                       step.data_ptr(), out.data_ptr(), _st(step))
    return out


def cifar_augment_draw(cfg, rank, step, offs, flips, boxes):
    """The cifar_augment draw of the device step counter ``step`` for worker ``rank`` (``cfg`` a validated config) into ``offs`` (int32
    [B, 2]), ``flips`` (uint8 [B]) and ``boxes`` (int32 [B, 4]): one ``cifar_augment_draw_kernel`` launch (reference.cifar_augment_draw
    on the CPU; ops/cifar_augment.py owns the layout)."""
    from .cifar_augment import SIZE
    B = offs.shape[0]
    for t, dt, shape in ((offs, torch.int32, (B, 2)), (flips, torch.uint8, (B,)), (boxes, torch.int32, (B, 4))):
        if not (t.is_cuda and t.dtype == dt and t.is_contiguous() and tuple(t.shape) == shape and t.device == step.device):
            raise ValueError("cifar_augment_draw: a buffer is not a contiguous %s %s tensor on %s" % (dt, shape, step.device))
    assert boxes.data_ptr() % 16 == 0 and offs.data_ptr() % 8 == 0
    L().cifar_augment_draw(B, int(cfg["pad"]), int(cfg["cutout"]), SIZE, SIZE, int(cfg["seed"]) & (2 ** 64 - 1), int(rank),
                           step.data_ptr(), offs.data_ptr(), flips.data_ptr(), boxes.data_ptr(), _st(step))


# --------------------------------------------------------------------------- loader kernel
def crop_mirror_normalize(x, mean, std_scale, crop_hw, offsets, flips, out_dtype=None, out=None, c_out=None, zero_fill=False):
    """``nn_kernels.cu: crop_mirror_norm_kernel``: image n normalised, cropped at ``offsets[n]`` (inside the image, or anywhere with
    ``zero_fill``, where a pixel outside the image is 0) and mirrored where ``flips[n]``.  See :func:`reference.crop_mirror_normalize`."""
    out_dtype = out_dtype or ADT()
    x = x.contiguous()
    N, H, W, C = x.shape
    ch, cw = crop_hw
    kind = {torch.uint8: 0, torch.bfloat16: 1, torch.float32: 2}[x.dtype]
    mean = mean.float().contiguous()
    mode = 0 if mean.numel() == 1 else (1 if mean.numel() == C else 2)
    if mode == 2:
        assert mean.numel() == H * W * C
    Cout = c_out or C
    if out is None:
        out = torch.empty((N, ch, cw, Cout), dtype=out_dtype, device=x.device)
    assert out.dtype in (BF16, torch.float32)
    offsets = offsets.to(torch.int32).contiguous()
    flips = flips.to(torch.uint8).contiguous()
    if isinstance(std_scale, torch.Tensor):                   # per-channel scale (1 / 255 / img_std)
        cs = std_scale.to(device=x.device, dtype=torch.float32).contiguous()
        assert cs.numel() == C
        sc, cs_ptr = 1.0, cs.data_ptr()
    else:
        sc, cs_ptr = float(std_scale), 0
    L().crop_mirror_norm(x.data_ptr(), kind, mean.data_ptr(), mode, sc, cs_ptr, out.data_ptr(), int(out.dtype == BF16),
                         offsets.data_ptr(), flips.data_ptr(), N, H, W, C, ch, cw, Cout, int(bool(zero_fill)), _st(x))
    return out


def multi_crop_normalize(x, mean, std_scale, crop_hw, n_views, out_dtype=None, out=None):
    """Every test-time view of a uint8 NHWC batch in one launch (``nn_kernels.cu: multi_crop_norm_kernel``): view-major
    [V, N, ch, cw, C], view v bit-equal to :func:`crop_mirror_normalize` with the view's offsets and mirror flag broadcast.  The view
    table (:func:`reference.multi_crop_views`) goes to the kernel by value.  Same mean / ``std_scale`` forms as
    :func:`crop_mirror_normalize`; see :func:`reference.multi_crop_normalize`."""
    from .reference import multi_crop_views
    out_dtype = out_dtype or ADT()
    if x.dtype != torch.uint8 or x.dim() != 4:
        raise ValueError("multi_crop_normalize takes a uint8 NHWC batch, not %s %s" % (x.dtype, tuple(x.shape)))
    x = x.contiguous()
    N, H, W, C = x.shape
    ch, cw = crop_hw
    views = multi_crop_views((H, W), crop_hw, n_views).tolist()
    V = len(views)
    mean = mean.float().contiguous()
    mode = 0 if mean.numel() == 1 else (1 if mean.numel() == C else 2)
    if mode == 2:
        assert mean.numel() == H * W * C
    if out is None:
        out = torch.empty((V, N, ch, cw, C), dtype=out_dtype, device=x.device)
    assert out.dtype in (BF16, F32) and out.is_contiguous() and tuple(out.shape) == (V, N, ch, cw, C) and out.device == x.device
    if isinstance(std_scale, torch.Tensor):
        cs = std_scale.to(device=x.device, dtype=F32).contiguous()
        assert cs.numel() == C
        sc, cs_ptr = 1.0, cs.data_ptr()
    else:
        sc, cs_ptr = float(std_scale), 0
    L().multi_crop_norm(x.data_ptr(), mean.data_ptr(), mode, sc, cs_ptr, out.data_ptr(), int(out.dtype == BF16), [v[0] for v in views],
                        [v[1] for v in views], [v[2] for v in views], N, H, W, C, ch, cw, _st(x))
    return out


def view_softmax_accum(logits, labels, acc, v, n_views, rowstat=None):
    """View ``v`` of ``n_views`` of multi-view validation (``nn_kernels.cu: view_softmax_accum_kernel``): ``acc`` (fp32 [B, C]) takes
    softmax(logits) (v = 0) or adds it; the last view divides by V, leaving p̄ in ``acc``, and returns the device scalars (cost, top-1
    error, top-5 error) of :func:`reference.view_metrics` after one more ``rowstat_mean`` launch; earlier views return None.
    ``logits``: bf16 or fp32 [B, C]."""
    lg = logits.contiguous()
    B, C = lg.shape
    if lg.dtype not in (BF16, F32):
        raise ValueError("view_softmax_accum: bf16 or fp32 logits, not %s" % lg.dtype)
    labels = labels.contiguous()
    assert labels.dtype == torch.int64 and tuple(labels.shape) == (B,)
    assert acc.dtype == F32 and acc.is_contiguous() and tuple(acc.shape) == (B, C) and acc.device == lg.device
    last = v == n_views - 1
    if rowstat is None:
        rowstat = torch.empty((B, 3), dtype=F32, device=lg.device)
    out3 = torch.empty(3, dtype=F32, device=lg.device) if last else None
    L().view_softmax_accum(lg.data_ptr(), labels.data_ptr(), acc.data_ptr(), rowstat.data_ptr(), _p(out3), B, C, int(v), int(n_views),
                           int(_is32(lg)), _st(lg))
    return (out3[0], out3[1], out3[2]) if last else None


def resized_crop_mirror_normalize(x, mean, std_scale, out_hw, boxes, flips, out_dtype=None, out=None):
    """Random-resized crop of a uint8 NHWC batch (``nn_kernels.cu: resized_crop_mirror_norm_kernel``): image n's box
    ``boxes[n] = (y0, x0, h, w)`` (int32 [N, 4] on the device, inside the image) normalised, bilinearly resampled to ``out_hw`` and
    mirrored where ``flips[n]``.  Same mean / ``std_scale`` forms as :func:`crop_mirror_normalize`; see
    :func:`reference.resized_crop_mirror_normalize`."""
    out_dtype = out_dtype or ADT()
    if x.dtype != torch.uint8:
        raise ValueError("resized_crop_mirror_normalize takes a uint8 NHWC batch, not %s" % x.dtype)
    x = x.contiguous()
    N, H, W, C = x.shape
    ch, cw = out_hw
    mean = mean.float().contiguous()
    mode = 0 if mean.numel() == 1 else (1 if mean.numel() == C else 2)
    if mode == 2:
        assert mean.numel() == H * W * C
    if out is None:
        out = torch.empty((N, ch, cw, C), dtype=out_dtype, device=x.device)
    assert out.dtype in (BF16, torch.float32) and out.is_contiguous() and tuple(out.shape) == (N, ch, cw, C)
    boxes = boxes.to(torch.int32).contiguous()
    assert tuple(boxes.shape) == (N, 4) and boxes.device == x.device and boxes.data_ptr() % 16 == 0
    flips = flips.to(torch.uint8).contiguous()
    if isinstance(std_scale, torch.Tensor):
        cs = std_scale.to(device=x.device, dtype=torch.float32).contiguous()
        assert cs.numel() == C
        sc, cs_ptr = 1.0, cs.data_ptr()
    else:
        sc, cs_ptr = float(std_scale), 0
    L().resized_crop_mirror_norm(x.data_ptr(), mean.data_ptr(), mode, sc, cs_ptr, out.data_ptr(), int(out.dtype == BF16),
                                 boxes.data_ptr(), flips.data_ptr(), N, H, W, C, ch, cw, _st(x))
    return out


def _color_inputs(name, x, boxes):
    if x.dtype != torch.uint8 or x.dim() != 4 or x.shape[3] != 3:
        raise ValueError("%s takes a uint8 NHWC batch with C = 3, not %s %s" % (name, x.dtype, tuple(x.shape)))
    x = x.contiguous()
    boxes = boxes.to(torch.int32).contiguous()
    assert tuple(boxes.shape) == (x.shape[0], 4) and boxes.device == x.device and boxes.data_ptr() % 16 == 0
    return x, boxes


def crop_mean(x, boxes, out_hw, out=None):
    """Mean RGB of each output crop (``nn_kernels.cu: crop_mean_kernel``): ``out[n, :3]`` is the mean over the ``out_hw`` pixels of the
    bilinear resample of the raw box ``boxes[n]`` of the uint8 NHWC batch (C = 3), ``out[n, 3] = 0``; fp32 [N, 4], one launch, a
    fixed-order reduction.  A box of the output's size gives the exact integer sum, divided once."""
    x, boxes = _color_inputs("crop_mean", x, boxes)
    N, H, W, _ = x.shape
    ch, cw = out_hw
    if out is None:
        out = torch.empty((N, 4), dtype=torch.float32, device=x.device)
    assert out.dtype == torch.float32 and out.is_contiguous() and tuple(out.shape) == (N, 4) and out.data_ptr() % 16 == 0
    L().crop_mean(x.data_ptr(), boxes.data_ptr(), out.data_ptr(), N, H, W, ch, cw, _st(x))
    return out


def color_crop_mirror_normalize(x, mean, std_scale, out_hw, boxes, flips, records, mu=None, out_dtype=None, out=None):
    """Colour jitter and lighting on the resized crop (``resized_crop_mirror_norm_kernel<_, true>``): with v̂ / m̂ the bilinear resample
    of image n's raw box / of the mean, the output is ``(M·v̂ + K·μ + ℓ − m̂)·std_scale``, mirrored where ``flips[n]``.  ``records``:
    fp32 [N, 24] on the device (M, K, ℓ, 0; ``utils.color_jitter_records``), 16-byte aligned; ``mu``: :func:`crop_mean`'s [N, 4], or
    None when every K is 0.  A fixed crop is the box (y0, x0, ch, cw).  See :func:`reference.color_crop_mirror_normalize`."""
    out_dtype = out_dtype or ADT()
    x, boxes = _color_inputs("color_crop_mirror_normalize", x, boxes)
    N, H, W, C = x.shape
    ch, cw = out_hw
    mean = mean.float().contiguous()
    mode = 0 if mean.numel() == 1 else (1 if mean.numel() == C else 2)
    if mode == 2:
        assert mean.numel() == H * W * C
    if out is None:
        out = torch.empty((N, ch, cw, C), dtype=out_dtype, device=x.device)
    assert out.dtype in (BF16, torch.float32) and out.is_contiguous() and tuple(out.shape) == (N, ch, cw, C)
    flips = flips.to(torch.uint8).contiguous()
    assert records.dtype == torch.float32 and records.is_contiguous() and tuple(records.shape) == (N, 24)
    assert records.device == x.device and records.data_ptr() % 16 == 0
    if mu is not None:
        assert mu.dtype == torch.float32 and mu.is_contiguous() and tuple(mu.shape) == (N, 4) and mu.data_ptr() % 16 == 0
    if isinstance(std_scale, torch.Tensor):
        cs = std_scale.to(device=x.device, dtype=torch.float32).contiguous()
        assert cs.numel() == C
        sc, cs_ptr = 1.0, cs.data_ptr()
    else:
        sc, cs_ptr = float(std_scale), 0
    L().color_crop_mirror_norm(x.data_ptr(), mean.data_ptr(), mode, sc, cs_ptr, out.data_ptr(), int(out.dtype == BF16), boxes.data_ptr(),
                               flips.data_ptr(), records.data_ptr(), 0 if mu is None else mu.data_ptr(), N, H, W, ch, cw, _st(x))
    return out


def aa_crop_u8(x, out_hw, boxes, flips, out=None):
    """auto_augment's uint8 crop (``resized_crop_mirror_norm_kernel<uint8_t>``): uint8 [N, ch, cw, 3], the bilinear resample of each
    raw box rounded half to even, mirrored where ``flips[n]``.  See :func:`reference.aa_crop_u8`."""
    x, boxes = _color_inputs("aa_crop_u8", x, boxes)
    N, H, W, _ = x.shape
    ch, cw = out_hw
    if out is None:
        out = torch.empty((N, ch, cw, 3), dtype=torch.uint8, device=x.device)
    assert out.dtype == torch.uint8 and out.is_contiguous() and tuple(out.shape) == (N, ch, cw, 3)
    flips = flips.to(torch.uint8).contiguous()
    L().aa_crop_u8(x.data_ptr(), out.data_ptr(), boxes.data_ptr(), flips.data_ptr(), N, H, W, ch, cw, _st(x))
    return out


def _aa_records(records, u):
    assert records.dtype == torch.float32 and records.is_contiguous() and records.dim() == 3 and records.shape[2] == 12
    assert records.shape[0] == u.shape[0] and records.device == u.device and records.data_ptr() % 16 == 0


def aa_lut(u, records, slot, out=None):
    """The point-op LUTs of one op slot (``aa_lut_kernel``): uint8 [N, 3, 256] for the images whose op in ``slot`` is Brightness,
    Contrast, Posterize, Solarize, AutoContrast or Equalize, computed from the uint8 crop ``u``; other images' rows are untouched."""
    _aa_records(records, u)
    N, ch, cw, _ = u.shape
    if out is None:
        out = torch.zeros((N, 3, 256), dtype=torch.uint8, device=u.device)
    L().aa_lut(u.data_ptr(), records.data_ptr(), out.data_ptr(), int(slot), records.shape[1], N, ch, cw, _st(u))
    return out


def aa_apply(u, records, slot, lut, out=None, bilinear=False):
    """One op slot on the uint8 crop (``aa_apply_kernel``), ``u`` → ``out`` (never in place); ``bilinear`` resamples the geometric ops
    bilinearly (``aa_apply_kernel<true>``).  An image whose op in ``slot`` is AA_NONE leaves its part of ``out`` untouched."""
    _aa_records(records, u)
    N, ch, cw, _ = u.shape
    if out is None:
        out = torch.empty_like(u)
    assert out.data_ptr() != u.data_ptr() and out.shape == u.shape and out.is_contiguous()
    L().aa_apply(u.data_ptr(), out.data_ptr(), records.data_ptr(), lut.data_ptr(), int(slot), records.shape[1], N, ch, cw, int(bool(bilinear)),
                 _st(u))
    return out


def aa_mix(u, chains, records, weights):
    """AugMix's mix in place on the uint8 crop ``u`` (``aa_mix_kernel``): u = trunc(m₀·u + Σ w_i·chain_i) in fp32, chain i read from
    ``chains[i, (depth − 1) & 1]`` with its depth from ``records`` (AA_NONE steps).  ``chains``: uint8 [width, 2, N, ch, cw, 3];
    ``records``: [N, 3·width, 12]; ``weights``: fp32 [N, 1 + width] on the device.  One launch.  See :func:`reference.augmix_mix`."""
    _aa_records(records, u)
    N, ch, cw, _ = u.shape
    width = records.shape[1] // 3
    assert records.shape[1] == 3 * width and tuple(chains.shape) == (width, 2) + tuple(u.shape) and chains.dtype == torch.uint8
    assert chains.is_contiguous() and u.is_contiguous() and chains.device == u.device
    assert weights.dtype == torch.float32 and weights.is_contiguous() and tuple(weights.shape) == (N, 1 + width) and weights.device == u.device
    L().aa_mix(u.data_ptr(), chains.data_ptr(), records.data_ptr(), weights.data_ptr(), width, N, ch, cw, _st(u))
    return u


def aa_normalize(u, mean, std_scale, boxes, flips, in_hw, out_dtype=None, out=None):
    """(u' − m̂)·std_scale into bf16 / fp32 NHWC (``aa_normalize_kernel``), m̂ the resample of a per-pixel mean over each mirrored box."""
    out_dtype = out_dtype or ADT()
    N, ch, cw, C = u.shape
    H, W = in_hw
    mean = mean.float().contiguous()
    mode = 0 if mean.numel() == 1 else (1 if mean.numel() == C else 2)
    if mode == 2:
        assert mean.numel() == H * W * C
    if out is None:
        out = torch.empty((N, ch, cw, C), dtype=out_dtype, device=u.device)
    assert out.dtype in (BF16, torch.float32) and out.is_contiguous() and tuple(out.shape) == (N, ch, cw, C)
    boxes = boxes.to(torch.int32).contiguous()
    assert tuple(boxes.shape) == (N, 4) and boxes.data_ptr() % 16 == 0
    flips = flips.to(torch.uint8).contiguous()
    if isinstance(std_scale, torch.Tensor):
        cs = std_scale.to(device=u.device, dtype=torch.float32).contiguous()
        sc, cs_ptr = 1.0, cs.data_ptr()
    else:
        sc, cs_ptr = float(std_scale), 0
    L().aa_normalize(u.data_ptr(), mean.data_ptr(), mode, sc, cs_ptr, out.data_ptr(), int(out.dtype == BF16), boxes.data_ptr(),
                     flips.data_ptr(), N, W, ch, cw, _st(u))
    return out


def auto_augment_crop_normalize(x, mean, std_scale, out_hw, boxes, flips, records, ops=None, out_dtype=None, out=None, ping=None,
                                pong=None, lut=None, bilinear=None, weights=None, chains=None):
    """TrivialAugmentWide / RandAugment / AutoAugment on the crop, then normalisation: :func:`aa_crop_u8` into ``ping``; per op slot
    :func:`aa_lut` (only when an image's op in the slot is a point op; ``ops`` = the host's int [N, slots] op ids, read from
    ``records`` when None) and :func:`aa_apply` ping → pong, swapping; then :func:`aa_normalize`.  ``bilinear``: the geometric ops'
    interpolation (read from ``records`` when None).  Launches: 1 + Σ over slots of (1 if a point op is drawn, + 1) + 1.

    AugMix, with ``weights`` (fp32 [N, 1 + width] on the device): the slots are ``width`` chains of 3, and ``ping`` (the crop u)
    survives them.  Step s of chain i maps u (s = 0) or ``chains[i, (s − 1) & 1]`` to ``chains[i, s & 1]`` (``chains``: uint8
    [width, 2, N, ch, cw, 3]); a step that no image of the batch reaches is not launched, and an image whose chain has ended
    (AA_NONE) returns at once, so a short chain costs no copy.  :func:`aa_mix` then mixes in place into ``ping``.  Launches:
    1 + Σ over slots of (1 if a point op is drawn, + 1 if any image's op is not AA_NONE) + 1 (mix) + 1.
    See :func:`reference.auto_augment_crop_normalize`."""
    from ..models.data.utils import AA_LUT_OPS, AA_NONE
    N, H, W, _ = x.shape
    ch, cw = out_hw
    if ops is None:
        ops = records[..., 0].to("cpu", torch.int64).numpy()
    if bilinear is None:
        bilinear = bool((records[..., 3] != 0).any())
    ping = aa_crop_u8(x, out_hw, boxes, flips, out=ping)
    lut = lut if lut is not None else torch.empty((N, 3, 256), dtype=torch.uint8, device=x.device)
    if weights is not None:
        width = records.shape[1] // 3
        if chains is None:
            chains = torch.empty((width, 2) + tuple(ping.shape), dtype=torch.uint8, device=x.device)
        for slot in range(records.shape[1]):
            i, s = divmod(slot, 3)
            live = [int(o) for o in ops[:, slot] if int(o) != AA_NONE]
            if not live:
                continue
            src = ping if s == 0 else chains[i, (s - 1) & 1]
            if any(o in AA_LUT_OPS for o in live):
                aa_lut(src, records, slot, out=lut)
            aa_apply(src, records, slot, lut, out=chains[i, s & 1], bilinear=bilinear)
        aa_mix(ping, chains, records, weights)
        return aa_normalize(ping, mean, std_scale, boxes, flips, (H, W), out_dtype, out=out)
    pong = pong if pong is not None else torch.empty_like(ping)
    for slot in range(records.shape[1]):
        if any(int(o) in AA_LUT_OPS for o in ops[:, slot]):
            aa_lut(ping, records, slot, out=lut)
        aa_apply(ping, records, slot, lut, out=pong, bilinear=bilinear)
        ping, pong = pong, ping
    return aa_normalize(ping, mean, std_scale, boxes, flips, (H, W), out_dtype, out=out)


def random_erase(x, boxes):
    """Random erasing in place (``nn_kernels.cu: erase_boxes_kernel``): every element of image n's box ``boxes[n] = (i, j, h, w)``
    (int32 [N, 4] on the device, 16-byte aligned, inside the output; h = w = 0 erases nothing) of the bf16 or fp32 NHWC batch ``x``
    is set to 0; nothing else is touched.  One launch.  Returns ``x``.  See :func:`reference.random_erase`."""
    if not (x.is_cuda and x.dtype in (BF16, torch.float32) and x.dim() == 4 and x.is_contiguous()):
        raise ValueError("random_erase takes a contiguous bf16 or fp32 NHWC batch on the device, not %s %s" % (x.dtype, tuple(x.shape)))
    N, ch, cw, C = x.shape
    assert boxes.dtype == torch.int32 and boxes.is_contiguous() and tuple(boxes.shape) == (N, 4)
    assert boxes.device == x.device and boxes.data_ptr() % 16 == 0
    L().erase_boxes(x.data_ptr(), int(x.dtype == BF16), boxes.data_ptr(), N, ch, cw, C, _st(x))
    return x


# --------------------------------------------------------------------------- optimizer
def _table(arena):
    if not hasattr(arena, "_tab_cache"):
        arena._tab_cache = (arena.group_lr_mult_np.tolist(), arena.group_wd_np.tolist(),
                            [int(v) for v in arena.group_exch_np.tolist()])
    return arena._tab_cache


def flat_update(arena, rule, hyper, state, step=None, g=None, lo=0, hi=None, filt=0, trust=None, clip=None):
    """One step of the local flat optimizer ``rule`` (a key of ``FLAT_RULES``: sgd, adam, rmsprop, adadelta,
    rmsprop_centered, lars, lamb) over arena elements [lo, hi) in one launch (``csrc/comm_kernels.cu: flat_update_kernel``; Adam
    and LAMB add the launch that advances their ``step`` counter, LAMB not after a ``filt`` = 1 pass).  ``state``: the rule's flat
    fp32 buffers, the arena's U region first when the rule uses it; ``hyper``: its float hyper-parameters (order in
    ``csrc/api.h``); ``filt`` (SGD, LARS, LAMB): 1 only non-exchanged groups, 2 only exchanged groups; ``trust`` (LARS, LAMB): the
    per-tensor trust ratios from :func:`lars_trust` / :func:`lamb_trust`; ``clip`` (the first five rules): the record
    :func:`grad_clip_norm` wrote for this step, so the step uses s·g, or changes nothing (Adam's counter included) when the
    gradient norm is not finite.  lr is read from ``arena.hyper[0]`` on the device, so a captured CUDA graph follows lr changes,
    and the bf16 shadow is refreshed in the same pass."""
    lrm, wd, ex = _table(arena)
    S = [t.data_ptr() for t in state] + [0] * (3 - len(state))
    lib = L()
    lib.flat_update(lib.FLAT_RULES[rule], arena.W.data_ptr(), (arena.G if g is None else g).data_ptr(), *S, _p(arena.H),
                    arena.block_group.data_ptr(), lrm, wd, ex, arena.hyper.data_ptr(), _p(step), [float(v) for v in hyper],
                    int(lo), int(arena.numel if hi is None else hi), int(filt),
                    0 if trust is None else arena.block_tensor.data_ptr(), _p(trust), _p(clip), _st(arena.W))


def grad_clip_norm(arena, g, max_norm, partial, rec, skipped):
    """The global L2 norm n of the gradient region ``g`` over the real elements of every arena tensor, for gradient clipping
    (two launches, ``csrc/comm_kernels.cu: lars_partial_kernel<false>, clip_finalize_kernel``): ``partial`` [n_blocks] receives
    the per-block sums of squares, ``rec`` (4 x fp32, ``csrc/api.h: ClipRecord``) n, s = min(1, max_norm / (n + 1e-6)) and the
    int32 flag "n is finite"; ``skipped`` (int64 [1]) is incremented when it is not.  ``g`` is not changed.  Every input is read
    from device memory, so the launches can be captured in a CUDA graph."""
    assert partial.dtype == torch.float32 and partial.is_contiguous() and tuple(partial.shape) == (arena.n_blocks,), tuple(partial.shape)
    assert rec.dtype == torch.float32 and rec.is_contiguous() and rec.numel() == 4, (rec.dtype, tuple(rec.shape))
    assert skipped.dtype == torch.int64 and skipped.numel() == 1 and skipped.is_cuda, (skipped.dtype, tuple(skipped.shape))
    assert g.dtype == torch.float32 and g.is_contiguous() and g.numel() == arena.numel, (g.dtype, tuple(g.shape))
    L().grad_clip_norm(g.data_ptr(), arena.block_tensor.data_ptr(), arena.tensor_span.data_ptr(), int(arena.n_blocks),
                       float(max_norm), partial.data_ptr(), rec.data_ptr(), skipped.data_ptr(), _st(arena.W))


def lars_trust(arena, g, inv_k, eta, partial, norms, trust):
    """LARS trust ratios of every arena tensor from W and the gradient region ``g`` (two launches, ``csrc/comm_kernels.cu:
    lars_partial_kernel, lars_finalize_kernel``): ``partial`` [n_blocks, 2] receives the per-block sums of squares, ``norms``
    [n_tensors, 2] ‖W‖ and ‖g·inv_k‖, ``trust`` [n_tensors] eta·‖W‖ / (‖g‖ + wd·‖W‖) for the weight group (1 elsewhere and when a
    norm is zero).  Every input is read from device memory, so the launches can be captured in a CUDA graph."""
    for t, shape in ((partial, (arena.n_blocks, 2)), (norms, (len(arena.sizes), 2)), (trust, (len(arena.sizes),))):
        assert t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, tuple(t.shape), shape)
    lrm, wd, ex = _table(arena)
    L().lars_trust(arena.W.data_ptr(), g.data_ptr(), arena.block_tensor.data_ptr(), arena.tensor_span.data_ptr(),
                   arena.block_group.data_ptr(), lrm, wd, ex, float(inv_k), float(eta), int(arena.n_blocks), len(arena.sizes),
                   partial.data_ptr(), norms.data_ptr(), trust.data_ptr(), _st(arena.W))


def lamb_trust(arena, g, m, v, step, b1, b2, eps, inv_k, filt, partial, norms, trust):
    """Passes 1 and 2 of a LAMB step over the groups that ``filt`` keeps (0 all, 1 only non-exchanged, 2 only exchanged; two
    launches, ``csrc/comm_kernels.cu: lamb_moments_kernel, lars_finalize_kernel``): advance the moments ``m`` (the arena's U) and
    ``v`` from the gradient region ``g`` times ``inv_k``, with the bias corrections of step ``step + 1`` (``step``: the device
    counter, not advanced here), then write ``norms`` [n_tensors, 2] ‖W‖ and ‖r‖ of the update direction r and ``trust``
    [n_tensors] ‖W‖ / ‖r‖ for the weight group (1 elsewhere and when a norm is zero).  ``partial`` [n_blocks, 2] receives the
    per-block sums of squares.  The ``flat_update`` pass of the ``lamb`` rule applies the step."""
    for t, shape in ((partial, (arena.n_blocks, 2)), (norms, (len(arena.sizes), 2)), (trust, (len(arena.sizes),))):
        assert t.dtype == torch.float32 and t.is_contiguous() and tuple(t.shape) == shape, (t.dtype, tuple(t.shape), shape)
    for t in (m, v):
        assert t.dtype == torch.float32 and t.is_contiguous() and t.numel() == arena.W.numel(), (t.dtype, tuple(t.shape))
    assert step.dtype == torch.int64 and step.numel() == 1 and step.is_cuda, (step.dtype, tuple(step.shape))
    lrm, wd, ex = _table(arena)
    L().lamb_trust(arena.W.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), step.data_ptr(), float(b1), float(b2), float(eps),
                   float(inv_k), int(filt), arena.block_tensor.data_ptr(), arena.tensor_span.data_ptr(), arena.block_group.data_ptr(),
                   lrm, wd, ex, int(arena.n_blocks), len(arena.sizes), partial.data_ptr(), norms.data_ptr(), trust.data_ptr(),
                   _st(arena.W))


def lr_schedule_step(arena, sched, counter):
    """One launch of ``csrc/comm_kernels.cu: lr_schedule_kernel``: with u = ``counter`` (int64 [1] on the arena's device), write the
    schedule's lr(u) to ``arena.hyper[0]`` and u + 1 to ``counter``.  ``sched``: the validated parameters (``utils/opt.py:
    LrSchedule``).  Reads only device memory, so it can be captured in a CUDA graph."""
    assert counter.dtype == torch.int64 and counter.numel() == 1 and counter.device == arena.hyper.device, (counter.dtype, counter.device)
    lib = L()
    lib.lr_schedule(lib.LR_POLICIES[sched.decay], int(sched.warmup_steps), int(sched.total_steps), float(sched.warmup_start),
                    float(sched.peak), float(sched.final_lr), float(sched.power), float(sched.gamma), [int(m) for m in sched.milestones],
                    counter.data_ptr(), arena.hyper.data_ptr(), _st(arena.hyper))


def _ema_check(arena, e, table):
    assert e.dtype == torch.float32 and e.is_contiguous() and e.numel() == arena.numel and e.device == arena.W.device, (e.dtype, e.shape)
    assert table.dtype == torch.int64 and table.dim() == 2 and table.shape[1] == 3 and table.device == arena.W.device, (table.dtype,
                                                                                                                         table.shape)


def ema_advance(state, every, warmup):
    """One single-thread launch of ``csrc/comm_kernels.cu: ema_advance_kernel``: ``state`` (int64 [3] on the device: u, n_averaged,
    mode) counts one more optimizer update and takes the mode of :func:`ema_update` (``reference.ema_advance``).  Reads only device
    memory, so it can be captured in a CUDA graph."""
    assert state.dtype == torch.int64 and state.numel() == 3 and state.is_cuda and state.is_contiguous(), (state.dtype, state.shape)
    L().ema_advance(state.data_ptr(), int(every), int(warmup), _st(state))


def ema_update(arena, e, state, table, decay, one_minus_decay):
    """One launch of ``csrc/comm_kernels.cu: ema_update_kernel``: per the mode in ``state[2]`` (skip, copy or average), nothing,
    E ← W or E ← fp32(d)·E + fp32(1 − d)·W over the arena's W region into ``e`` (fp32 [arena.numel]) and over the segments of
    ``table`` (int64 [n, 3]: E part address, statistics tensor address, n elements).  Reads only device memory."""
    _ema_check(arena, e, table)
    assert state.dtype == torch.int64 and state.numel() == 3 and state.device == arena.W.device, (state.dtype, state.shape)
    L().ema_update(arena.W.data_ptr(), e.data_ptr(), int(arena.numel), table.data_ptr(), int(table.shape[0]), state.data_ptr(),
                   float(np.float32(decay)), float(np.float32(one_minus_decay)), _st(arena.W))


def ema_swap(arena, e, table):
    """One launch of ``csrc/comm_kernels.cu: ema_swap_kernel``: W ↔ ``e``, the bf16 shadow ← bf16-RN(new W), and the two parts of
    every segment of ``table`` exchanged.  Twice is the identity."""
    _ema_check(arena, e, table)
    L().ema_swap(arena.W.data_ptr(), e.data_ptr(), _p(arena.H), int(arena.numel), table.data_ptr(), int(table.shape[0]), _st(arena.W))


def _sam_check(arena, p, rec):
    assert p.dtype == torch.float32 and p.is_contiguous() and p.numel() == arena.numel and p.device == arena.W.device, (p.dtype, p.shape)
    if rec is not None:
        assert rec.dtype == torch.float32 and rec.is_contiguous() and rec.numel() == 4 and rec.device == arena.W.device, (rec.dtype,
                                                                                                                         rec.shape)


def sam_norm(arena, rho, adaptive, partial, rec):
    """The ascent-step norm of sharpness-aware minimization (two launches, ``csrc/comm_kernels.cu: lars_partial_kernel<false>`` or
    ``sam_partial_wg_kernel``, then ``sam_finalize_kernel``): n = ‖g‖ (``adaptive``: ‖|w|⊙g‖) over the real elements of the arena's G
    and W, accumulated in fp64 in a fixed order, into ``rec`` (4 x fp32, ``csrc/api.h: ClipRecord``) with s = fp32(1 / (n + 1e-12))·ρ
    and the int32 flag "n is finite" (``reference.sam_norm`` / ``sam_scale``).  ``partial`` [n_blocks] receives the per-block sums."""
    _sam_check(arena, arena.W, rec)
    assert partial.dtype == torch.float32 and partial.is_contiguous() and tuple(partial.shape) == (arena.n_blocks,), tuple(partial.shape)
    L().sam_norm(arena.W.data_ptr(), arena.G.data_ptr(), arena.block_tensor.data_ptr(), arena.tensor_span.data_ptr(),
                 int(arena.n_blocks), float(np.float32(rho)), int(bool(adaptive)), partial.data_ptr(), rec.data_ptr(), _st(arena.W))


def sam_perturb(arena, p, rec, adaptive):
    """The ascent step (one launch of ``csrc/comm_kernels.cu: sam_perturb_kernel``): ``p`` ← W, then, when the record ``rec`` of
    :func:`sam_norm` is finite, W ← W + e on the real elements (e = g·s, ``adaptive``: ((w·w)·g)·s, each product and the sum rounded
    once) and the bf16 shadow ← bf16-RN(W) (``reference.sam_perturb``)."""
    _sam_check(arena, p, rec)
    L().sam_perturb(arena.W.data_ptr(), arena.G.data_ptr(), p.data_ptr(), _p(arena.H), arena.block_tensor.data_ptr(),
                    arena.tensor_span.data_ptr(), int(arena.n_blocks), int(bool(adaptive)), rec.data_ptr(), _st(arena.W))


def sam_restore(arena, p):
    """W ← ``p`` and the bf16 shadow ← bf16-RN(``p``) (one launch of ``csrc/comm_kernels.cu: sam_restore_kernel``)."""
    _sam_check(arena, p, None)
    L().sam_restore(arena.W.data_ptr(), p.data_ptr(), _p(arena.H), int(arena.n_blocks), _st(arena.W))


def sgd_flat(arena, g, lr, mu, nesterov, inv_k, lo, hi, only_local=False, only_exchanged=False, clip=None):
    """Fused momentum-SGD over arena elements [lo, hi): ``flat_update``'s SGD rule.  ``lr`` is not used: the kernel reads
    ``arena.hyper[0]`` on the device (so a captured CUDA graph follows lr changes)."""
    filt = 1 if only_local else (2 if only_exchanged else 0)
    flat_update(arena, "sgd", (mu, float(bool(nesterov)), inv_k), [arena.U], g=g, lo=lo, hi=hi, filt=filt, clip=clip)
