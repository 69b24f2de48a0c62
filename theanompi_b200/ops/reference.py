"""Plain-PyTorch reference implementations of every op in :mod:`theanompi_b200.ops`.

These are (a) the CPU execution path (tests, gloo plumbing runs) and (b) the
fp32 ground truth every hand-written sm_90a kernel is tested against.

Layout convention for the whole framework: activations are **NHWC**
``[N, H, W, C]`` contiguous, conv filters are **OHWI** ``[O, kh, kw, C/groups]``,
FC weights are ``[n_out, n_in]`` (K-major for the wgmma GEMM).  The reference
used c01b / bc01 (``theanompi/models/layers2.py:430-560``).
"""
from __future__ import annotations

import math

import numpy as np
import torch
import torch.nn.functional as F

LEAKY_SLOPE = 0.2        # negative slope of the "leaky" activation (the DCGAN critic's LeakyReLU(0.2))


def act_fwd(y, relu):
    """Activation named by a ``relu`` argument: a bool (ReLU or identity) or one of "none", "relu", "leaky", "sigmoid"."""
    a = relu if isinstance(relu, str) else ("relu" if relu else "none")
    if a == "relu":
        return torch.relu(y)
    if a == "leaky":
        return F.leaky_relu(y, LEAKY_SLOPE)
    if a == "sigmoid":
        return torch.sigmoid(y)
    assert a == "none", a
    return y


def act_bwd(dy, y, relu):
    """``dy`` times the activation's derivative, computed from its output ``y``."""
    a = relu if isinstance(relu, str) else ("relu" if relu else "none")
    if a == "relu":
        return dy * (y > 0).to(dy.dtype)
    if a == "leaky":
        return torch.where(y > 0, dy, dy * LEAKY_SLOPE)
    if a == "sigmoid":
        return dy * y * (1 - y)
    return dy


def _nchw(x):
    return x.permute(0, 3, 1, 2)


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous()


# --------------------------------------------------------------------------- conv
def conv2d_bias_act(x, w, b, stride=1, pad=0, groups=1, relu=True):
    """conv + bias + ReLU (ref ``layers2.py:380-388``)."""
    y = F.conv2d(_nchw(x), w.permute(0, 3, 1, 2), b, stride=stride, padding=pad, groups=groups)
    return _nhwc(act_fwd(y, relu))


def conv2d_bias_act_bwd(x, w, y, dy, stride=1, pad=0, groups=1, relu=True, need_dx=True):
    """Returns (dx, dw, db) given the forward output ``y`` (for the activation mask)."""
    dy = act_bwd(dy, y, relu)
    xn, wn, dyn = _nchw(x), w.permute(0, 3, 1, 2), _nchw(dy)
    dx = None
    if need_dx:
        dx = torch.nn.grad.conv2d_input(xn.shape, wn, dyn, stride=stride, padding=pad, groups=groups)
        dx = _nhwc(dx)
    dw = torch.nn.grad.conv2d_weight(xn, wn.shape, dyn, stride=stride, padding=pad, groups=groups)
    dw = dw.permute(0, 2, 3, 1).contiguous()
    db = dy.sum(dim=(0, 1, 2))
    return dx, dw, db


# --------------------------------------------------------------------------- transposed conv
def conv_transpose2d_bias_act(x, w, b, stride, pad, output_padding=0, relu=False, c_real=None):
    """Transposed conv + bias + activation, NHWC; ``w`` is ``[Cin, KH, KW, Cout]`` (the OHWI weight of the convolution that
    maps y-space back to x-space — ``torch.nn.ConvTranspose2d``'s ``[Cin, Cout, KH, KW]`` permuted).  Output channels
    ``>= c_real`` are zero (padding of a layer narrower than 16 bytes)."""
    if c_real is not None and c_real < w.shape[-1] and relu not in (True, "relu", "sigmoid"):
        raise RuntimeError("conv_transpose2d: padded output channels need a ReLU or sigmoid activation")
    y = F.conv_transpose2d(_nchw(x), w.permute(0, 3, 1, 2), b, stride=stride, padding=pad, output_padding=output_padding)
    y = _nhwc(act_fwd(y, relu))
    if c_real is not None and c_real < y.shape[-1]:
        y[..., c_real:] = 0
    return y


def conv_transpose2d_bias_act_bwd(x, w, y, dy, stride, pad, relu, need_dx=True):
    """Returns (dx, dw, db) of :func:`conv_transpose2d_bias_act`: dx is the forward convolution of the masked gradient, dw
    that convolution's weight gradient with x in the role of its output gradient."""
    dym = act_bwd(dy, y, relu)
    wn = w.permute(0, 3, 1, 2)                       # [Cin, Cout, KH, KW] = conv weight [O, I, KH, KW] of y-space -> x-space
    dx = _nhwc(F.conv2d(_nchw(dym), wn, None, stride=stride, padding=pad)) if need_dx else None
    dw = torch.nn.grad.conv2d_weight(_nchw(dym), wn.shape, _nchw(x), stride=stride, padding=pad).permute(0, 2, 3, 1).contiguous()
    return dx, dw, dym.sum(dim=(0, 1, 2))


# --------------------------------------------------------------------------- linear
def linear_bias_act(x, w, b, relu=True):
    """FC + bias + ReLU (ref ``layers2.py:927-929``); ``w`` is ``[n_out, n_in]``."""
    y = F.linear(x, w, b)
    return act_fwd(y, relu)


def linear_bias_act_bwd(x, w, y, dy, relu=True, need_dx=True):
    dy = act_bwd(dy, y, relu)
    dx = dy @ w if need_dx else None
    dw = dy.t() @ x
    db = dy.sum(0)
    return dx, dw, db


# --------------------------------------------------------------------------- pool
def pool2d(x, ksize, stride, pad=0, mode="max"):
    """max / average pooling (ref ``layers2.py:414-417``; cuDNN semantics: floor)."""
    xn = _nchw(x)
    if mode == "max":
        y = F.max_pool2d(xn, ksize, stride, pad)
    else:  # cuDNN 'average_exc_pad' is what theano's dnn_pool('average_exc_pad') used
        y = F.avg_pool2d(xn, ksize, stride, pad, count_include_pad=False)
    return _nhwc(y)


def pool2d_bwd(x, y, dy, ksize, stride, pad=0, mode="max"):
    xr = x.detach().clone().requires_grad_(True)
    with torch.enable_grad():
        yr = pool2d(xr, ksize, stride, pad, mode)
    (dx,) = torch.autograd.grad(yr, xr, dy)
    return dx


# --------------------------------------------------------------------------- LRN
def lrn(x, n=5, k=2.0, alpha=1e-4, beta=0.75):
    """Cross-channel LRN exactly as the reference writes it
    (``layers2.py:753-809``): ``x / (k + alpha * sum_{|j-i|<=n/2} x_j^2) ** beta``
    (alpha is NOT divided by n, unlike ``torch.nn.functional.local_response_norm``).
    Returns (y, scale)."""
    half = n // 2
    sq = x.float() ** 2
    C = x.shape[-1]
    padded = F.pad(sq, (half, half))
    s = torch.zeros_like(sq)
    for i in range(n):
        s = s + padded[..., i:i + C]
    scale = k + alpha * s
    y = x.float() * scale.pow(-beta)
    return y.to(x.dtype), scale


def lrn_bwd(x, dy, n=5, k=2.0, alpha=1e-4, beta=0.75):
    xr = x.detach().float().clone().requires_grad_(True)
    with torch.enable_grad():
        yr, _ = lrn(xr, n, k, alpha, beta)
    (dx,) = torch.autograd.grad(yr, xr, dy.float())
    return dx.to(x.dtype)


# --------------------------------------------------------------------------- dropout
def dropout_mask(shape, p_drop, seed, offset, device):
    """Deterministic keep-mask from (seed, offset) so CPU tests can reproduce it."""
    g = torch.Generator(device="cpu")
    g.manual_seed((int(seed) * 1000003 + int(offset)) & 0x7FFFFFFFFFFFFFFF)
    m = torch.rand(shape, generator=g) >= p_drop
    return m.to(device)


def dropout(x, p_drop, mask):
    """Inverted-scale-free dropout as in the reference (``layers2.py:885-891``):
    train: ``mask * x``; eval: ``(1-p) * x``."""
    return x * mask.to(x.dtype)


# --------------------------------------------------------------------------- softmax + NLL
def softmax_xent(logits, labels, grad_scale=1.0, weight=1.0, label_smoothing=0.0, mix=None):
    """weight · mean NLL, top-1 error, top-5 error, and d(mean NLL)/dlogits times weight · ``grad_scale`` (1/n under gradient
    accumulation over n micro-batches) (ref ``layers2.py:952-997``).  ``label_smoothing`` ε > 0: the loss and its gradient are those
    of the soft target (1 − ε)·onehot + ε / C (``F.cross_entropy(..., label_smoothing=ε)``); the errors do not change.  ``mix`` (a
    Mixup / CutMix record, ops/mixup.py): see :func:`softmax_xent_mix`."""
    if mix is not None:
        return softmax_xent_mix(logits, labels, mix, grad_scale, weight, label_smoothing)
    lg = logits.float()
    lsm = F.log_softmax(lg, dim=1)
    B = lg.shape[0]
    rows = torch.arange(B, device=lg.device)
    if label_smoothing:
        eps = float(label_smoothing)
        loss = -((1.0 - eps) * lsm[rows, labels] + eps * lsm.mean(1)).mean()
    else:
        loss = -lsm[rows, labels].mean()
    pred = lg.argmax(1)
    err1 = (pred != labels).float().mean()
    k = min(5, lg.shape[1])
    topk = lg.topk(k, dim=1).indices
    err5 = 1.0 - (topk == labels[:, None]).any(1).float().mean()
    dlogits = lsm.exp()
    if label_smoothing:
        dlogits[rows, labels] -= 1.0 - eps
        dlogits -= eps / lg.shape[1]
    else:
        dlogits[rows, labels] -= 1.0
    dlogits = dlogits / B
    if weight != 1.0:
        loss = loss * weight
        grad_scale = grad_scale * weight
    if grad_scale != 1.0:
        dlogits = dlogits * grad_scale
    return loss, err1, err5, dlogits


def softmax_xent_mix(logits, labels, mix, grad_scale=1.0, weight=1.0, label_smoothing=0.0):
    """:func:`softmax_xent` against the mixed soft target q = λ·s(y_i) + (1 − λ)·s(y_j) of the record ``mix``, with j = B − 1 − i
    and s(y) = (1 − ε)·onehot(y) + ε / C: the loss −Σ q·log p and its gradient (p − q) / B (times weight · grad_scale); the top-1 /
    top-5 errors count against y_i when λ ≥ ½, else against y_j."""
    lg = logits.float()
    B, C = lg.shape
    lam = mix_lambda(mix)
    eps = float(label_smoothing)
    lsm = F.log_softmax(lg, dim=1)

    def soft(y):
        return (1.0 - eps) * F.one_hot(y, C).float() + eps / C
    q = lam * soft(labels) + (1.0 - lam) * soft(labels.flip(0))
    loss = -(q * lsm).sum(1).mean()
    ye = labels if lam >= 0.5 else labels.flip(0)
    err1 = (lg.argmax(1) != ye).float().mean()
    topk = lg.topk(min(5, C), dim=1).indices
    err5 = 1.0 - (topk == ye[:, None]).any(1).float().mean()
    dlogits = (lsm.exp() - q) / B * (grad_scale * weight)
    return loss * weight, err1, err5, dlogits


def softmax_xent_kd(logits, labels, teacher, alpha, temperature, grad_scale=1.0, label_smoothing=0.0, mix=None):
    """Knowledge distillation (Hinton et al. 2015) of the student's logits z against the teacher's logits t of the same batch: per row
    L = (1 − α)·CE_q(z) + α·T²·KL(softmax(t/T) ‖ softmax(z/T)), q the target of :func:`softmax_xent` (``label_smoothing`` ε; with
    ``mix`` that of :func:`softmax_xent_mix`), the teacher's distribution never smoothed.  Returns (mean L, top-1 error, top-5 error,
    dlogits) with dlogits = [(1 − α)·(p − q) + α·T·(softmax(z/T) − softmax(t/T))] / B times ``grad_scale``; the errors are the student's,
    ranked as :func:`softmax_xent_mix` ranks them.  Computed in fp64 when the logits are fp64, else in fp32."""
    dt = torch.float64 if logits.dtype == torch.float64 else torch.float32
    z, t = logits.to(dt), teacher.to(dt)
    B, C = z.shape
    lam = 1.0 if mix is None else mix_lambda(mix)
    eps, a, T = float(label_smoothing), float(alpha), float(temperature)

    def soft(y):
        return (1.0 - eps) * F.one_hot(y, C).to(dt) + eps / C
    q = soft(labels) if lam == 1.0 else lam * soft(labels) + (1.0 - lam) * soft(labels.flip(0))
    lsm = F.log_softmax(z, dim=1)
    ls_s, ls_t = F.log_softmax(z / T, dim=1), F.log_softmax(t / T, dim=1)
    p_t = ls_t.exp()
    rows = (1.0 - a) * -(q * lsm).sum(1) + a * T * T * (p_t * (ls_t - ls_s)).sum(1)
    ye = labels if lam >= 0.5 else labels.flip(0)
    err1 = (z.argmax(1) != ye).to(dt).mean()
    topk = z.topk(min(5, C), dim=1).indices
    err5 = 1.0 - (topk == ye[:, None]).any(1).to(dt).mean()
    dlogits = ((1.0 - a) * (lsm.exp() - q) + a * T * (ls_s.exp() - p_t)) / B * grad_scale
    return rows.mean(), err1, err5, dlogits


# --------------------------------------------------------------------------- GAN losses / noise
def gan_loss(scores, kind, a):
    """Loss over the critic's scores and d loss / d scores.
    ``wgan``:  ``a * mean(o)``            (a = +1 fake / -1 real batch of the critic loss, -1 for the generator)
    ``lsgan``: ``0.5 * mean((o - a)^2)``  (a = target: 1 real / 0 fake, 1 for the generator)."""
    o = scores.float()
    B = o.numel()
    if kind == "wgan":
        return a * o.mean(), torch.full_like(o, a / B)
    assert kind == "lsgan", kind
    e = o - a
    return 0.5 * (e * e).mean(), e / B


_PHILOX_M = (0xD2511F53, 0xCD9E8D57)
_PHILOX_W = (0x9E3779B9, 0xBB67AE85)


def _philox4x32(c, k0, k1):
    """Philox4x32-10 over uint64 arrays holding 32-bit words (csrc/nn_kernels.cu: philox4x32)."""
    M32 = np.uint64(0xFFFFFFFF)
    c0, c1, c2, c3 = (np.asarray(v, dtype=np.uint64) & M32 for v in c)
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = c0 * np.uint64(_PHILOX_M[0])
        p1 = c2 * np.uint64(_PHILOX_M[1])
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32)
        k0, k1 = (k0 + np.uint64(_PHILOX_W[0])) & M32, (k1 + np.uint64(_PHILOX_W[1])) & M32
    return c0, c1, c2, c3


def uniform_noise(shape, seed, stream, step, device="cpu"):
    """Uniform [0, 1) noise, bit-identical (in fp32) to the CUDA ``uniform_noise`` kernel: element i is word i % 4 of
    Philox(counter = (i // 4, step), key = (seed, stream)) with its low 8 bits dropped, times 2^-24."""
    n = int(np.prod(shape))
    q = np.arange((n + 3) // 4, dtype=np.uint64)
    seed, step = int(seed) & (2 ** 64 - 1), int(step)
    r = _philox4x32((q, q >> np.uint64(32), np.full_like(q, step & 0xFFFFFFFF), np.full_like(q, step >> 32)),
                    seed & 0xFFFFFFFF, ((seed >> 32) ^ int(stream)) & 0xFFFFFFFF)
    words = np.stack(r, axis=1).reshape(-1)[:n]
    u = (words >> np.uint64(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
    return torch.from_numpy(u.reshape(shape)).to(device)


def dropout_mask_philox(n, p_drop, seed, layer, step):
    """Keep-mask (bool [n], n a multiple of 8) of the CUDA ``dropout_fwd`` kernel, bit for bit: group j of 8 elements draws
    Philox(counter = (j, step), key = (seed_lo, seed_hi ^ layer·0x9E3779B9)); element i of the group takes 16-bit half i & 1 of
    word i >> 1 and is kept iff it is >= the threshold (uint32)(float(p_drop)·65536), so P(keep) = 1 − ⌊p·65536⌋ / 65536.
    (:func:`dropout_mask` is the CPU execution path's own mask; this one is the kernel's host twin for tests.)"""
    n = int(n)
    if n % 8:
        raise ValueError("dropout_mask_philox: n must be a multiple of 8")
    j = np.arange(n // 8, dtype=np.uint64)
    seed, step, layer = int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1), int(layer) & 0xFFFFFFFF
    r = _philox4x32((j, j >> np.uint64(32), np.full_like(j, step & 0xFFFFFFFF), np.full_like(j, step >> 32)),
                    seed & 0xFFFFFFFF, ((seed >> 32) ^ (layer * 0x9E3779B9)) & 0xFFFFFFFF)
    words = np.stack(r, axis=1)                                                           # [groups, 4]
    halves = np.stack([words & np.uint64(0xFFFF), words >> np.uint64(16)], axis=2)      # [groups, 4, 2]: element i = (i >> 1, i & 1)
    thr = np.uint64(int(np.float32(p_drop) * np.float32(65536.0)))
    return torch.from_numpy((halves.reshape(-1) >= thr))


# --------------------------------------------------------------------------- Mixup / CutMix
_MIX_TAG = 0xFFFFFFFF          # second counter word of every mix block (csrc/nn_kernels.cu: kMixCounterTag)
_MIX_ATTEMPTS = 16             # Marsaglia–Tsang attempts per Gamma variate (kMixAttempts)


def _mix_block(j, s, k0, k1):
    """Philox block j of the mix draws of the steps ``s`` (uint64 array): counter (j, 0xFFFFFFFF, s_lo, s_hi)."""
    M32 = np.uint64(0xFFFFFFFF)
    return _philox4x32((np.full_like(s, j), np.full_like(s, _MIX_TAG), s & M32, s >> np.uint64(32)), k0, k1)


def _mix_u01(w):
    return (w.astype(np.float64) + 0.5) * 2.3283064365386963e-10


def _mix_gamma(a, boost_u, j0, s, k0, k1):
    """Gamma(a) per step (``a``: fp64 array) by Marsaglia–Tsang from Box–Muller normals, a < 1 boosted by U^(1/a), the operations in
    the kernel's order; (values, accepted)."""
    ae = np.where(a < 1.0, a + 1.0, a)
    d = ae - 1.0 / 3.0
    c = 1.0 / np.sqrt(9.0 * d)
    g = np.zeros_like(a)
    done = np.zeros(a.shape, dtype=bool)
    with np.errstate(divide="ignore", invalid="ignore"):
        for k in range(_MIX_ATTEMPTS):
            r = _mix_block(j0 + k, s, k0, k1)
            x = np.sqrt(-2.0 * np.log(_mix_u01(r[0]))) * np.cos(6.283185307179586 * _mix_u01(r[1]))
            v = 1.0 + c * x
            ok = v > 0.0
            v = (v * v) * v
            u, x2 = _mix_u01(r[2]), x * x
            acc = ok & ((u < 1.0 - (0.0331 * x2) * x2) | (np.log(u) < 0.5 * x2 + d * ((1.0 - v) + np.log(v))))
            new = acc & ~done
            g = np.where(new, d * v, g)
            done |= acc
    boost = np.power(boost_u, 1.0 / a)
    return np.where(a < 1.0, g * boost, g), done


def mix_draw(cfg, seed, rank, step, hw):
    """The Mixup / CutMix draw of step counter value ``step`` (an int, or an array of them) for worker ``rank``, as the CUDA
    ``mix_draw_kernel`` makes it (ops/mixup.py: RECORD; one record for an int step).  ``cfg`` is a validated ``config['mixup']``
    (mixup.check_config), ``hw`` = (H, W) the image size at the mix point.

    Philox4x32-10, key (seed_lo, seed_hi ^ rank), counter (j, 0xFFFFFFFF, step_lo, step_hi).  Block 0: the gate (mix when
    U < prob), the switch (CutMix when both α > 0 and U < switch_prob) and the CutMix centre (⌊w·H / 2^32⌋, ⌊w·W / 2^32⌋); block 1
    the U^(1/α) boosts of X and Y; blocks 2 + k and 2 + 16 + k attempt k of X and of Y ~ Gamma(α).  λ = X / (X + Y) in fp64.
    Mixup: effective λ = fp32(λ).  CutMix (timm's rand_bbox): r = √(1 − λ), the box of ⌊H·r⌋ × ⌊W·r⌋ centred on (cy, cx) clipped to
    the image, effective λ = fp32(1 − area / (H·W)).  A Gamma draw that rejects all 16 attempts leaves the step unmixed."""
    from . import mixup
    H, W = int(hw[0]), int(hw[1])
    scalar = np.ndim(step) == 0
    s = np.atleast_1d(np.asarray(step, dtype=np.int64)).astype(np.uint64)
    seed = int(seed) & (2 ** 64 - 1)
    k0, k1 = seed & 0xFFFFFFFF, ((seed >> 32) ^ int(rank)) & 0xFFFFFFFF
    out = np.zeros(s.shape, dtype=mixup.RECORD)
    out["mode"], out["lam"], out["lam_raw"], out["H"], out["W"] = mixup.MIX_NONE, 1.0, 1.0, H, W
    w0 = _mix_block(0, s, k0, k1)
    w1 = _mix_block(1, s, k0, k1)
    gate = _mix_u01(w0[0]) < cfg["prob"]
    if cfg["alpha"] > 0.0 and cfg["cutmix_alpha"] > 0.0:
        cut = _mix_u01(w0[1]) < cfg["switch_prob"]
    else:
        cut = np.full(s.shape, cfg["cutmix_alpha"] > 0.0)
    a = np.where(cut, cfg["cutmix_alpha"], cfg["alpha"])
    gx, okx = _mix_gamma(a, _mix_u01(w1[0]), 2, s, k0, k1)
    gy, oky = _mix_gamma(a, _mix_u01(w1[1]), 2 + _MIX_ATTEMPTS, s, k0, k1)
    mix = gate & okx & oky
    tot = gx + gy
    with np.errstate(divide="ignore", invalid="ignore"):
        lam = np.where(tot > 0.0, gx / tot, 0.5)
    mu, cm = mix & ~cut, mix & cut
    out["mode"][mu], out["lam_raw"][mu], out["lam"][mu] = mixup.MIX_MIXUP, lam[mu], lam[mu].astype(np.float32)
    r = np.sqrt(1.0 - lam[cm])
    ch, cw = (H * r).astype(np.int64), (W * r).astype(np.int64)
    cy = ((w0[2][cm] * np.uint64(H)) >> np.uint64(32)).astype(np.int64)
    cx = ((w0[3][cm] * np.uint64(W)) >> np.uint64(32)).astype(np.int64)
    y0, y1 = np.clip(cy - ch // 2, 0, H), np.clip(cy + ch // 2, 0, H)
    x0, x1 = np.clip(cx - cw // 2, 0, W), np.clip(cx + cw // 2, 0, W)
    area = (y1 - y0) * (x1 - x0)
    out["mode"][cm], out["lam_raw"][cm] = mixup.MIX_CUTMIX, lam[cm]
    out["lam"][cm] = (1.0 - area.astype(np.float64) / float(H * W)).astype(np.float32)
    for name, v in (("cy", cy), ("cx", cx), ("y0", y0), ("y1", y1), ("x0", x0), ("x1", x1)):
        out[name][cm] = v
    return out[0] if scalar else out


def mix_lambda(rec):
    """The weight of y_i in the step's target: the record's effective λ (an fp32 value), 1 when it does not mix."""
    from . import mixup
    r = mixup.decode(rec)
    return float(np.float32(r["lam"])) if int(r["mode"]) != mixup.MIX_NONE else 1.0


def mix_batch(x, rec):
    """The batch ``x`` [B, H, W, C] mixed as the record says, sample i with j = B − 1 − i (``x.flip(0)``): Mixup
    λ·x + (1 − λ)·x.flip(0) in fp32, rounded once to x's dtype; CutMix x with the box taken from x.flip(0); unmixed a copy."""
    from . import mixup
    r = mixup.decode(rec)
    mode = int(r["mode"])
    if mode == mixup.MIX_MIXUP:
        xf = x.float()
        lam = torch.tensor(float(r["lam"]), dtype=torch.float32)
        return (lam * xf + (1.0 - lam) * xf.flip(0)).to(x.dtype)
    out = x.clone()
    if mode == mixup.MIX_CUTMIX:
        if (int(r["H"]), int(r["W"])) != tuple(x.shape[1:3]):
            raise ValueError("mix_batch: the record's box refers to %dx%d images, not %s" % (int(r["H"]), int(r["W"]), tuple(x.shape[1:3])))
        y0, y1, x0, x1 = (int(r[k]) for k in ("y0", "y1", "x0", "x1"))
        out[:, y0:y1, x0:x1, :] = x.flip(0)[:, y0:y1, x0:x1, :]
    return out


# --------------------------------------------------------------------------- drop-path (stochastic depth)
def drop_path_draw(p_list, seed, rank, step, B):
    """The drop-path table of step counter value ``step`` for worker ``rank`` (fp32 ``[L, B]``, ops/drop_path.py), as the CUDA
    ``drop_path_draw_kernel`` writes it: entry (l, n) is 0 when (w >> 8)·2^-24 < p_l, else fp32(1 / (1 − p_l)), w word 0 of
    Philox4x32-10 with key (seed_lo, seed_hi ^ rank) and counter (n, l ^ TAG, step_lo, step_hi).  ``p_list``: the block rates p_l."""
    from . import drop_path
    rates = np.asarray(p_list, dtype=np.float64)
    L, B = rates.shape[0], int(B)
    thresh, keep = drop_path.thresholds(rates).astype(np.uint64), drop_path.keep_scales(rates)
    M32 = 0xFFFFFFFF
    seed, step = int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1)
    l = np.repeat(np.arange(L, dtype=np.uint64), B)
    n = np.tile(np.arange(B, dtype=np.uint64), L)
    w0 = _philox4x32((n, l ^ np.uint64(drop_path.TAG), np.full_like(n, step & M32), np.full_like(n, step >> 32)),
                     seed & M32, ((seed >> 32) ^ (int(rank) & M32)) & M32)[0]
    li = l.astype(np.int64)
    out = np.where((w0 >> np.uint64(8)) < thresh[li], np.float32(0.0), keep[li]).astype(np.float32)
    return torch.from_numpy(out.reshape(L, B))


# --------------------------------------------------------------------------- CIFAR augmentation (cifar_augment)
def cifar_augment_draw(cfg, seed, rank, step, B):
    """(offs int32 [B, 2], flips uint8 [B], boxes int32 [B, 4]) of step counter value ``step`` for worker ``rank``, as the CUDA
    ``cifar_augment_draw_kernel`` writes them (ops/cifar_augment.py owns the layout).  ``cfg`` is a validated ``config['cifar_augment']``.

    Philox4x32-10, key (seed_lo, seed_hi ^ rank), counter (n, TAG, step_lo, step_hi) for block 0 and (n, TAG + 1, ...) for block 1;
    each value ⌊w·k / 2^32⌋: oy, ox (k = 2·pad + 1) from block 0 words 0, 1; flip = word 2 >> 31; cy (k = 32) from word 3; cx from
    block 1 word 0.  offs = (oy − pad, ox − pad); the Cutout box is DeVries & Taylor's clamp of cy ± L//2, cx ± L//2."""
    from . import cifar_augment as ca
    M32 = 0xFFFFFFFF
    seed, step = int(seed) & (2 ** 64 - 1), int(step) & (2 ** 64 - 1)
    k0, k1 = seed & M32, ((seed >> 32) ^ (int(rank) & M32)) & M32
    n = np.arange(int(B), dtype=np.uint64)
    lo, hi = np.full_like(n, step & M32), np.full_like(n, step >> 32)
    a = _philox4x32((n, np.full_like(n, ca.TAG), lo, hi), k0, k1)
    b = _philox4x32((n, np.full_like(n, ca.TAG + 1), lo, hi), k0, k1)
    pad, L, S = cfg["pad"], cfg["cutout"], ca.SIZE

    def pick(w, k):
        return ((w * np.uint64(k)) >> np.uint64(32)).astype(np.int64)
    oy, ox = pick(a[0], 2 * pad + 1), pick(a[1], 2 * pad + 1)
    offs = np.stack([oy - pad, ox - pad], axis=1).astype(np.int32)
    flips = (a[2] >> np.uint64(31)).astype(np.uint8)
    boxes = ca.cutout_boxes(pick(a[3], S), pick(b[0], S), L)
    return torch.from_numpy(offs), torch.from_numpy(flips), torch.from_numpy(boxes)


# --------------------------------------------------------------------------- optimizer (flat arena)
def clip_scale(g, offsets, sizes, max_norm):
    """Global gradient-norm clipping (``torch.nn.utils.clip_grad_norm_``) over a flat fp32 gradient laid out as a :class:`FlatArena`
    (tensor ``i`` is ``[offsets[i], offsets[i] + sizes[i])``; the padding between tensors is ignored):

        n = ‖g‖₂ over the real elements, accumulated in fp64
        s = min(1, max_norm / (n + 1e-6))      rounded to fp32, as the device record holds it

    Returns ``(n, s, finite)``.  When n is NaN or Inf, ``finite`` is False, s = 0 and the step is to be skipped."""
    sq = 0.0
    for o, s in zip(offsets, sizes):
        v = g[o:o + s].double()
        sq += float(torch.dot(v, v))
    n = math.sqrt(sq)
    if not math.isfinite(n):
        return n, 0.0, False
    return n, float(np.float32(min(1.0, float(np.float32(max_norm)) / (n + 1e-6)))), True


def lr_at(u, peak, decay="constant", warmup_steps=0, warmup_start=0.0, total_steps=None, final_lr=0.0, power=1.0, gamma=0.1,
          milestones=()):
    """Learning rate of optimizer update ``u`` (0, 1, 2, ...) under a per-update schedule (``csrc/comm_kernels.cu:
    lr_schedule_kernel``), evaluated in fp64 and rounded once to fp32:

        u < W (warm-up)   peak·(s + (1 − s)·u / W)                                 W = warmup_steps, s = warmup_start
        then, with p = clamp((u − W) / (T − W), 0, 1), T = total_steps:
          constant        peak
          cosine          final + (peak − final)·½(1 + cos πp)
          poly            final + (peak − final)·(1 − p)^power
          multistep       peak·gamma^(number of milestones ≤ u)                    (gamma multiplied in once per milestone)"""
    u, W, peak = int(u), int(warmup_steps), float(peak)
    if u < W:
        s = float(warmup_start)
        return np.float32(peak * (s + (1.0 - s) * u / W))
    if decay == "constant":
        return np.float32(peak)
    if decay == "multistep":
        lr = peak
        for m in milestones:
            if u >= m:
                lr *= float(gamma)
        return np.float32(lr)
    p = min(max((u - W) / (int(total_steps) - W), 0.0), 1.0)
    final = float(final_lr)
    f = 0.5 * (1.0 + math.cos(math.pi * p)) if decay == "cosine" else (1.0 - p) ** float(power)
    return np.float32(final + (peak - final) * f)


def sgd_flat(w, g, u, lr_mult, wd, lr, mu, nesterov, inv_k, w_half=None):
    """One momentum-SGD step over flat fp32 buffers with per-element
    ``lr_mult`` / ``wd`` vectors (broadcastable).  Semantics of the reference's
    ``BSP_MSGD`` collapsed into one pass (``theanompi/lib/opt.py:181-268``):

        g_eff = g * inv_k + wd * w
        u     = mu * u + g_eff
        w    -= lr * lr_mult * (u            if not nesterov
                                g_eff + mu*u if nesterov)
    """
    g_eff = g * inv_k + wd * w
    u.mul_(mu).add_(g_eff)
    step = g_eff + mu * u if nesterov else u
    w.sub_(lr * lr_mult * step)
    if w_half is not None:
        w_half.copy_(w)
    return w, u


def adam_flat(w, g, m, v, lr_mult, wd, lr, b1=0.9, b2=0.999, eps=1e-8, t=1, w_half=None):
    """One Adam step over flat fp32 buffers (Keras / ``torch.optim.Adam``), ``t`` = the 1-based step number:

        g_eff = g + wd * w
        m     = b1 * m + (1 - b1) * g_eff
        v     = b2 * v + (1 - b2) * g_eff^2
        w    -= lr * lr_mult * (m / (1 - b1^t)) / (sqrt(v / (1 - b2^t)) + eps)
    """
    g_eff = g + wd * w
    m.mul_(b1).add_(g_eff, alpha=1 - b1)
    v.mul_(b2).addcmul_(g_eff, g_eff, value=1 - b2)
    mh, vh = m / (1 - b1 ** t), v / (1 - b2 ** t)
    w.sub_(lr * lr_mult * mh / (vh.sqrt() + eps))
    if w_half is not None:
        w_half.copy_(w)
    return w, m, v


def rmsprop_flat(w, g, v, lr_mult, wd, lr, alpha=0.99, eps=1e-8, clip=0.0, w_half=None):
    """One RMSProp step over flat fp32 buffers, ``torch.optim.RMSprop`` without momentum, plus an optional clip:

        g_eff = g + wd * w
        v     = alpha * v + (1 - alpha) * g_eff^2
        w    -= lr * lr_mult * g_eff / (sqrt(v) + eps)
        w     = clamp(w, -clip, clip)                  (clip > 0: the WGAN critic's weight clipping)
    """
    g_eff = g + wd * w
    v.mul_(alpha).addcmul_(g_eff, g_eff, value=1 - alpha)
    w.sub_(lr * lr_mult * g_eff / (v.sqrt() + eps))
    if clip > 0:
        w.clamp_(-clip, clip)
    if w_half is not None:
        w_half.copy_(w)
    return w, v


def adadelta_flat(w, g, u, v, lr_mult, wd, lr, rho=0.95, eps=1e-6, w_half=None):
    """One Adadelta step over flat fp32 buffers, ``torch.optim.Adadelta`` (the reference LSTM's ``adadelta`` at lr = 1):

        g_eff = g + wd * w
        v     = rho * v + (1 - rho) * g_eff^2
        d     = sqrt(u + eps) / sqrt(v + eps) * g_eff
        u     = rho * u + (1 - rho) * d^2
        w    -= lr * lr_mult * d
    """
    g_eff = g + wd * w
    v.mul_(rho).addcmul_(g_eff, g_eff, value=1 - rho)
    d = (u + eps).sqrt_().div_((v + eps).sqrt_()).mul_(g_eff)
    u.mul_(rho).addcmul_(d, d, value=1 - rho)
    w.sub_(lr * lr_mult * d)
    if w_half is not None:
        w_half.copy_(w)
    return w, u, v


def rmsprop_centered_flat(w, g, m, r, s, lr_mult, wd, lr, rho=0.95, mu=0.9, eps=1e-4, w_half=None):
    """One step of the reference LSTM's ``rmsprop`` (centred, with momentum, eps inside the square root) over flat fp32 buffers:

        g_eff = g + wd * w
        r     = rho * r + (1 - rho) * g_eff
        s     = rho * s + (1 - rho) * g_eff^2
        m     = mu * m - lr * lr_mult * g_eff / sqrt(s - r^2 + eps)
        w    += m
    """
    g_eff = g + wd * w
    r.mul_(rho).add_(g_eff, alpha=1 - rho)
    s.mul_(rho).addcmul_(g_eff, g_eff, value=1 - rho)
    m.mul_(mu).sub_(lr * lr_mult * g_eff / (s - r * r + eps).sqrt())
    w.add_(m)
    if w_half is not None:
        w_half.copy_(w)
    return w, m, r, s


def lars_flat(w, g, u, offsets, sizes, groups, group_lr_mult, group_wd, lr, mu, nesterov, eta=0.001, inv_k=1.0, update=None,
              w_half=None):
    """One LARS step (layer-wise adaptive rate scaling) over flat fp32 buffers laid out as a :class:`FlatArena`: tensor ``i`` is
    ``[offsets[i], offsets[i] + sizes[i])`` in hyper-parameter group ``groups[i]``.  Per tensor, with g = G·inv_k:

        trust = eta·‖W‖ / (‖g‖ + wd·‖W‖)   for the weight group when ‖W‖ > 0 and ‖g‖ > 0, else 1
        momentum SGD (:func:`sgd_flat`) with inv_k·trust and wd·trust in place of inv_k and wd

    Norms are accumulated in fp64 over the tensor's real elements.  ``update``: per-tensor booleans, the tensors to update (all
    when None); the trust ratios of every tensor are computed.  Returns (trust [n] fp32, norms [n, 2] fp32: ‖W‖, ‖g‖)."""
    from ..parallel.arena import G_W
    n, eta = len(offsets), float(np.float32(eta))
    trust = torch.ones(n, dtype=torch.float32)
    norms = torch.zeros(n, 2, dtype=torch.float32)
    for i, (o, s, grp) in enumerate(zip(offsets, sizes, groups)):
        sl = slice(o, o + s)
        wn = float(w[sl].double().norm())
        gn = float(g[sl].double().norm()) * float(np.float32(inv_k))
        wd = float(group_wd[grp])
        norms[i, 0], norms[i, 1] = wn, gn
        if grp == G_W and wn > 0 and gn > 0:
            trust[i] = eta * wn / (gn + wd * wn)
        if update is not None and not update[i]:
            continue
        t = np.float32(trust[i])
        sgd_flat(w[sl], g[sl], u[sl], float(group_lr_mult[grp]), float(np.float32(wd) * t), lr, mu, nesterov,
                 float(np.float32(inv_k) * t))
        if w_half is not None:
            w_half[sl].copy_(w[sl])
    return trust, norms


def lamb_flat(w, g, m, v, trust, norms, offsets, sizes, groups, group_lr_mult, group_wd, lr, b1=0.9, b2=0.999, eps=1e-6, t=1,
              inv_k=1.0, update=None, w_half=None):
    """One LAMB step (You et al., 2019) over flat fp32 buffers laid out as a :class:`FlatArena` (see :func:`lars_flat`), ``t`` = the
    1-based step number.  Per tensor, with g = G·inv_k:

        m     = b1·m + (1 − b1)·g
        v     = b2·v + (1 − b2)·g²
        r     = (m / (1 − b1^t)) / (sqrt(v / (1 − b2^t)) + eps) + wd·w          (decoupled weight decay)
        trust = ‖W‖ / ‖r‖   for the weight group when ‖W‖ > 0 and ‖r‖ > 0, else 1
        w    -= lr·lr_mult·trust·r

    Norms are accumulated in fp64 over the tensor's real elements.  ``update``: per-tensor booleans, the tensors to update (all when
    None); only their rows of ``trust`` [n] and ``norms`` [n, 2] (‖W‖, ‖r‖) are written, as on the device."""
    from ..parallel.arena import G_W
    b1, b2, inv_k = float(np.float32(b1)), float(np.float32(b2)), float(np.float32(inv_k))
    c1, c2 = 1.0 / (1.0 - b1 ** t), 1.0 / (1.0 - b2 ** t)
    for i, (o, s, grp) in enumerate(zip(offsets, sizes, groups)):
        if update is not None and not update[i]:
            continue
        sl = slice(o, o + s)
        ge = g[sl] * inv_k
        m[sl].mul_(b1).add_(ge, alpha=1 - b1)
        v[sl].mul_(b2).addcmul_(ge, ge, value=1 - b2)
        r = (m[sl] * c1) / ((v[sl] * c2).sqrt() + eps) + float(group_wd[grp]) * w[sl]
        wn, rn = float(w[sl].double().norm()), float(r.double().norm())
        norms[i, 0], norms[i, 1] = wn, rn
        trust[i] = wn / rn if (grp == G_W and wn > 0 and rn > 0) else 1.0
        w[sl].sub_(lr * float(group_lr_mult[grp]) * float(trust[i]) * r)
        if w_half is not None:
            w_half[sl].copy_(w[sl])
    return trust, norms


def easgd_elastic(w, c, alpha):
    """EASGD elastic move (ref ``exchanger.py:188-211``) with both sides updated
    from the SAME difference: ``d = alpha (w - c); w -= d; c += d``."""
    d = alpha * (w - c)
    w.sub_(d)
    c.add_(d)
    return w, c


def gosgd_merge(w, b, alpha_self, alpha_src):
    """GOSGD weighted merge (ref ``exchanger.py:450-462``)."""
    w.mul_(alpha_self).add_(b, alpha=alpha_src).div_(alpha_self + alpha_src)
    return w


EMA_SKIP, EMA_COPY, EMA_AVERAGE = 0, 1, 2


def ema_advance(u, n_averaged, every, warmup):
    """Model EMA bookkeeping after one more optimizer update: returns (u + 1, n_averaged', mode).  Update u + 1 averages iff it is a
    multiple of ``every``; it copies (mode EMA_COPY, n_averaged becomes 1) when nothing has been averaged yet or u + 1 <= ``warmup``,
    else it averages (EMA_AVERAGE, n_averaged + 1).  Otherwise EMA_SKIP."""
    u += 1
    if u % every:
        return u, n_averaged, EMA_SKIP
    if n_averaged == 0 or u <= warmup:
        return u, 1, EMA_COPY
    return u, n_averaged + 1, EMA_AVERAGE


def ema_update(pairs, mode, decay, one_minus_decay):
    """One model-EMA step over ``pairs`` of fp32 tensors (e, w), e updated in place: nothing (EMA_SKIP), e = w (EMA_COPY), or
    e = fp32(d)·e + fp32(1 − d)·w (EMA_AVERAGE) with both products and the sum each rounded once to fp32, which is what torch's
    fp32 expression ``d * e + (1 - d) * w`` gives (``torch.optim.swa_utils.AveragedModel`` with that ``avg_fn``).
    ``one_minus_decay``: 1 − d evaluated in float64, then rounded to fp32."""
    if mode == EMA_SKIP:
        return
    d = torch.tensor(float(np.float32(decay)), dtype=torch.float32)
    omd = torch.tensor(float(np.float32(one_minus_decay)), dtype=torch.float32)
    for e, w in pairs:
        if mode == EMA_COPY:
            e.copy_(w)
        else:
            e.copy_(torch.add(torch.mul(e, d.to(e.device)), torch.mul(w, omd.to(w.device))))


def ema_swap(pairs, w_half=None):
    """Exchange the contents of every pair (a, b) of equal-sized fp32 tensors; ``w_half`` (the bf16 shadow of the first pair's
    first tensor, or None) then takes bf16-RN of that tensor's new value.  Applying it twice restores every tensor."""
    for a, b in pairs:
        t = a.clone()
        a.copy_(b)
        b.copy_(t)
    if w_half is not None:
        w_half.copy_(pairs[0][0])


def sam_norm(w, g, offsets, sizes, adaptive=False):
    """The ascent-step norm of sharpness-aware minimization over a flat fp32 arena (tensor ``i`` is ``[offsets[i], offsets[i] +
    sizes[i])``, the padding ignored): n = ‖g‖₂, or with ``adaptive`` (ASAM) ‖|w|⊙g‖₂ with each w·g rounded once to fp32; the squares
    are summed in fp64 and n is rounded once to fp32.  Returns n as an np.float32."""
    sq = 0.0
    for o, s in zip(offsets, sizes):
        v = (w[o:o + s] * g[o:o + s] if adaptive else g[o:o + s]).double()
        sq += float(torch.dot(v, v))
    return np.float32(math.sqrt(sq))


def sam_scale(n, rho):
    """(s, finite) for the norm ``n`` (an fp32 value): s = rho / (n + 1e-12) as torch evaluates it on an fp32 tensor,
    fp32(1 / fp32(n + 1e-12)) · fp32(rho) (``Tensor.__rtruediv__`` is ``reciprocal() * other``); finite is False, and s = 0, when n is
    NaN or Inf."""
    n = torch.tensor(float(n), dtype=torch.float32)
    if not bool(torch.isfinite(n)):
        return 0.0, False
    return float(rho / (n + 1e-12)), True


def sam_perturb(w, g, p, s, finite, offsets, sizes, adaptive=False, w_half=None):
    """The ascent step of SAM over a flat fp32 arena laid out as in :func:`sam_norm`: ``p`` ← w; when ``finite``, w ← w + e on the real
    elements with e = g·s (``adaptive``: ((w·w)·g)·s), each product and the sum rounded once to fp32 (torch's ``p.add_(e_w)`` of the
    SAM wrapper), and ``w_half`` (the bf16 shadow, or None) ← bf16(w).  A non-finite norm leaves w as it is."""
    p.copy_(w)
    if not finite:
        return
    st = torch.tensor(float(s), dtype=torch.float32)
    for o, n in zip(offsets, sizes):
        wv, gv = w[o:o + n], g[o:o + n]
        e = (wv * wv * gv if adaptive else gv) * st
        wv.add_(e)
    if w_half is not None:
        w_half.copy_(w)


def sam_restore(w, p, w_half=None):
    """The end of a SAM step: w ← ``p`` and ``w_half`` (the bf16 shadow, or None) ← bf16(p)."""
    w.copy_(p)
    if w_half is not None:
        w_half.copy_(p)


# --------------------------------------------------------------------------- data aug
def crop_mirror_normalize(x_u8, mean, std_scale, crop_hw, offsets, flips, out_dtype=torch.float32, zero_fill=False):
    """``(x - mean) * std_scale`` → crop at per-image ``offsets`` → optional
    horizontal flip (ref ``data/utils.py:42-129`` + ``proc_load_mpi.py:99-104``).
    ``zero_fill``: the crop may reach outside the image, whose pixels are then 0 (the normalised image zero-padded, then cropped).

    x_u8   : [N, H, W, C] uint8 or float
    mean   : [H, W, C] or [C] float
    offsets: [N, 2] int (y0, x0);  flips: [N] bool
    """
    N, H, W, C = x_u8.shape
    ch, cw = crop_hw
    if isinstance(std_scale, torch.Tensor):
        std_scale = std_scale.to(device=x_u8.device, dtype=torch.float32)
    x = (x_u8.float() - mean.float()) * std_scale
    out = torch.empty((N, ch, cw, C), dtype=torch.float32, device=x.device)
    for i in range(N):
        y0, x0 = int(offsets[i, 0]), int(offsets[i, 1])
        if zero_fill:
            patch = torch.zeros((ch, cw, C), dtype=torch.float32, device=x.device)
            ys, ye, xs, xe = max(0, -y0), min(ch, H - y0), max(0, -x0), min(cw, W - x0)
            if ye > ys and xe > xs:
                patch[ys:ye, xs:xe] = x[i, y0 + ys:y0 + ye, x0 + xs:x0 + xe, :]
        else:
            patch = x[i, y0:y0 + ch, x0:x0 + cw, :]
        if bool(flips[i]):
            patch = patch.flip(1)
        out[i] = patch
    return out.to(out_dtype)


MULTI_CROP_VIEWS = (1, 2, 10)


def multi_crop_views(in_hw, crop_hw, n_views):
    """The (y0, x0, mirror) table of the ``n_views`` test-time views of a ``crop_hw`` crop of an ``in_hw`` image, int32 [V, 3], in
    the order of torchvision's ``ten_crop(img, size)``: top-left, top-right, bottom-left, bottom-right, centre, then the same five
    regions of the horizontally flipped image, whose view k + 5 is (y0_k, dx − x0_k, 1) with dx = W − cw.  V = 2 is views 4 and 9 (the
    centre crop and the centre crop of the mirrored image); V = 1 is view 4, the validation crop of :func:`crop_mirror_normalize`.
    The centre is (dy // 2, dx // 2); torchvision's ``center_crop`` anchors at round(d / 2), which differs only when d ≡ 3 (mod 4)."""
    H, W = in_hw
    ch, cw = crop_hw
    dy, dx = H - ch, W - cw
    if dy < 0 or dx < 0:
        raise ValueError("multi_crop_views: a %d x %d crop does not fit a %d x %d image" % (ch, cw, H, W))
    five = [(0, 0), (0, dx), (dy, 0), (dy, dx), (dy // 2, dx // 2)]
    ten = [(y, x, 0) for y, x in five] + [(y, dx - x, 1) for y, x in five]
    pick = {1: [4], 2: [4, 9], 10: list(range(10))}
    if n_views not in pick:
        raise ValueError("multi_crop_views: n_views must be one of %s, not %r" % (MULTI_CROP_VIEWS, n_views))
    return torch.tensor([ten[k] for k in pick[n_views]], dtype=torch.int32)


def multi_crop_normalize(x_u8, mean, std_scale, crop_hw, n_views, out_dtype=torch.float32):
    """The ``n_views`` test-time views (:func:`multi_crop_views`) of every image, view-major [V, N, ch, cw, C]: view v is
    :func:`crop_mirror_normalize` with the view's offsets and mirror flag broadcast to every image."""
    N, H, W, C = x_u8.shape
    views = multi_crop_views((H, W), crop_hw, n_views)
    out = []
    for y0, x0, m in views.tolist():
        offs = torch.tensor([[y0, x0]], dtype=torch.int32).expand(N, 2)
        out.append(crop_mirror_normalize(x_u8, mean, std_scale, crop_hw, offs, torch.full((N,), m, dtype=torch.uint8), out_dtype))
    return torch.stack(out)


def view_metrics(pbar, labels):
    """(mean −log max(p̄_y, FLT_MIN), top-1 error, top-5 error) of the averaged prediction ``pbar`` [B, C] in its own dtype, with the
    rank rule of the native kernels: rank = #{p̄_c > p̄_y} + #{c < y : p̄_c = p̄_y}; an error when rank ≥ 1 (top-1) or ≥ 5 (top-5)."""
    B, C = pbar.shape
    py = pbar.gather(1, labels.view(B, 1))
    cols = torch.arange(C, device=pbar.device).view(1, C)
    rank = ((pbar > py) | ((pbar == py) & (cols < labels.view(B, 1)))).sum(1)
    cost = -torch.log(py.view(B).clamp_min(float(np.finfo(np.float32).tiny))).mean()
    return cost, (rank >= 1).to(pbar.dtype).mean(), (rank >= 5).to(pbar.dtype).mean()


def multi_view_xent(logits_per_view, labels, dtype=torch.float64):
    """Multi-view validation of V views' logits (a list of [B, C], or [V, B, C]): p̄ = (1/V)·Σ_v softmax(z_v), each softmax
    computed in ``dtype``, the probabilities averaged (not the logits, as Krizhevsky et al. 2012 average the ten patches'
    predictions).  Returns (cost, top-1 error, top-5 error, p̄) with :func:`view_metrics`."""
    V = len(logits_per_view)
    pbar = sum(torch.softmax(z.to(dtype), dim=1) for z in logits_per_view) / V
    return view_metrics(pbar, labels.to(pbar.device)) + (pbar,)


def resized_crop_mirror_normalize(x_u8, mean, std_scale, out_hw, boxes, flips, out_dtype=torch.float32):
    """Random-resized crop: ``(x - mean) * std_scale`` (each source pixel with its own mean) → image i's box
    ``boxes[i] = (y0, x0, h, w)`` → ``F.interpolate(size=out_hw, mode='bilinear', align_corners=False, antialias=False)`` → optional
    horizontal flip, as torchvision's ``RandomResizedCrop`` then ``RandomHorizontalFlip`` without the antialiasing filter.

    x_u8 : [N, H, W, C] uint8;  mean: [H, W, C], [C] or scalar;  boxes: [N, 4] int, inside the image;  flips: [N] bool
    """
    import torch.nn.functional as F
    N, H, W, C = x_u8.shape
    if isinstance(std_scale, torch.Tensor):
        std_scale = std_scale.to(device=x_u8.device, dtype=torch.float32)
    x = (x_u8.float() - mean.float()) * std_scale
    out = torch.empty((N,) + tuple(out_hw) + (C,), dtype=torch.float32, device=x.device)
    for i in range(N):
        y0, x0, h, w = (int(v) for v in boxes[i])
        if not (h > 0 and w > 0 and 0 <= y0 <= H - h and 0 <= x0 <= W - w):
            raise ValueError("resized_crop_mirror_normalize: box %r of image %d is not inside %d x %d" % ((y0, x0, h, w), i, H, W))
        box = x[i, y0:y0 + h, x0:x0 + w, :].permute(2, 0, 1).unsqueeze(0)
        y = F.interpolate(box, size=tuple(out_hw), mode="bilinear", align_corners=False, antialias=False)[0].permute(1, 2, 0)
        out[i] = y.flip(1) if bool(flips[i]) else y
    return out.to(out_dtype)


def color_crop_mirror_normalize(x_u8, mean, std_scale, out_hw, boxes, flips, records, out_dtype=torch.float32):
    """Colour jitter and lighting on the (resized) crop: v = image i's raw box ``boxes[i] = (y0, x0, h, w)`` resampled to ``out_hw``
    (``F.interpolate``, bilinear, ``align_corners=False``, no antialias), m̂ = the same resample of a per-pixel mean (a [C] or scalar
    mean as it is), μ = the mean of v over the output pixels; the output is ``(M·v + K·μ + ℓ − m̂) * std_scale`` with (M, K, ℓ) from
    ``records[i]`` (``models/data/utils.py: color_jitter_records``), then the optional horizontal flip.  A fixed crop is the box of
    the output's size.  Values of M·v + K·μ + ℓ may leave [0, 255]: nothing is clamped, as in fb.resnet.torch.

    x_u8 : [N, H, W, 3] uint8;  mean: [H, W, 3], [3] or scalar;  boxes: [N, 4] int, inside the image;  flips: [N];  records: [N, 24]
    """
    import torch.nn.functional as F
    N, H, W, C = x_u8.shape
    if isinstance(std_scale, torch.Tensor):
        std_scale = std_scale.to(device=x_u8.device, dtype=torch.float32)
    mean = torch.as_tensor(mean).float()
    rec = torch.as_tensor(records).to(device=x_u8.device, dtype=torch.float32)
    out = torch.empty((N,) + tuple(out_hw) + (C,), dtype=torch.float32, device=x_u8.device)

    def resample(img, y0, x0, h, w):
        box = img[y0:y0 + h, x0:x0 + w, :].permute(2, 0, 1).unsqueeze(0)
        return F.interpolate(box, size=tuple(out_hw), mode="bilinear", align_corners=False, antialias=False)[0].permute(1, 2, 0)

    for i in range(N):
        y0, x0, h, w = (int(v) for v in boxes[i])
        if not (h > 0 and w > 0 and 0 <= y0 <= H - h and 0 <= x0 <= W - w):
            raise ValueError("color_crop_mirror_normalize: box %r of image %d is not inside %d x %d" % ((y0, x0, h, w), i, H, W))
        v = resample(x_u8[i].float(), y0, x0, h, w)
        m = resample(mean, y0, x0, h, w) if mean.dim() == 3 else mean
        M, K, ell = rec[i, 0:9].view(3, 3), rec[i, 9:18].view(3, 3), rec[i, 18:21]
        mu = v.reshape(-1, C).mean(0)
        y = (v @ M.T + (K @ mu + ell) - m) * std_scale
        out[i] = y.flip(1) if bool(flips[i]) else y
    return out.to(out_dtype)


def aa_crop_u8(x_u8, out_hw, boxes, flips):
    """auto_augment's uint8 crop: image i's raw box ``boxes[i] = (y0, x0, h, w)`` resampled to ``out_hw`` (``F.interpolate``, bilinear,
    ``align_corners=False``, no antialias), rounded half to even to uint8 and mirrored where ``flips[i]``.  Returns uint8 [N, ch, cw, C]."""
    import torch.nn.functional as F
    N, H, W, C = x_u8.shape
    out = torch.empty((N,) + tuple(out_hw) + (C,), dtype=torch.uint8, device=x_u8.device)
    for i in range(N):
        y0, x0, h, w = (int(v) for v in boxes[i])
        if not (h > 0 and w > 0 and 0 <= y0 <= H - h and 0 <= x0 <= W - w):
            raise ValueError("aa_crop_u8: box %r of image %d is not inside %d x %d" % ((y0, x0, h, w), i, H, W))
        box = x_u8[i, y0:y0 + h, x0:x0 + w, :].float().permute(2, 0, 1).unsqueeze(0)
        v = F.interpolate(box, size=tuple(out_hw), mode="bilinear", align_corners=False, antialias=False)[0].permute(1, 2, 0)
        v = v.round().to(torch.uint8)
        out[i] = v.flip(1) if bool(flips[i]) else v
    return out


def _aa_blend(img, other, f, d):
    return img.mul(f).add_(other, alpha=d).clamp_(0, 255).to(torch.uint8)


def _aa_gray(img):
    r, g, b = img.unbind(0)
    return r.mul(0.2989).add_(g, alpha=0.587).add_(b, alpha=0.114).floor_().unsqueeze(0)


def aa_apply_op(img, rec):
    """One op of TrivialAugmentWide / RandAugment / AutoAugment / AugMix on a uint8 CHW image (C = 3), as
    ``torchvision.transforms.v2.functional`` computes it (fill 0), from its 12-float record (``models/data/utils.py:
    auto_augment_records``): op id, scalar (factor, Solarize threshold or Posterize bits), 1 − factor, the interpolation of a
    geometric op (0 nearest, 1 bilinear), the fp32 inverse affine matrix.  Invert (op 14) is 255 − v; op 15 (an AugMix step past its
    chain's depth) returns the image as it is.

    The bilinear geometry is torchvision's ``_apply_grid_transform`` with fill None: ``grid_sample(mode="bilinear",
    padding_mode="zeros", align_corners=False)`` of the fp32 image (a tap outside the image contributes 0), ``round_()`` (half to
    even) and a cast to uint8."""
    import torch.nn.functional as F
    rec = [float(v) for v in rec]
    op, f, d = int(rec[0]), rec[1], rec[2]
    C, h, w = img.shape
    if op == 0 or op == 15:
        return img.clone()
    if op == 14:
        return 255 - img
    if 1 <= op <= 5:                                          # torchvision's _affine_grid and grid_sample(nearest / bilinear, zeros)
        theta = torch.tensor(rec[4:10], dtype=torch.float32).reshape(1, 2, 3)
        base = torch.empty(1, h, w, 3, dtype=torch.float32)
        base[..., 0].copy_(torch.linspace((1.0 - w) * 0.5, (w - 1.0) * 0.5, steps=w))
        base[..., 1].copy_(torch.linspace((1.0 - h) * 0.5, (h - 1.0) * 0.5, steps=h).unsqueeze_(-1))
        base[..., 2].fill_(1)
        rescaled = theta.transpose(1, 2).div_(torch.tensor([0.5 * w, 0.5 * h], dtype=torch.float32))
        grid = base.view(1, h * w, 3).bmm(rescaled).view(1, h, w, 2)
        mode = "bilinear" if rec[3] != 0.0 else "nearest"
        out = F.grid_sample(img.float().unsqueeze(0), grid, mode=mode, padding_mode="zeros", align_corners=False)
        return out[0].round_().to(torch.uint8)
    if op == 6:
        return img.mul(f).clamp_(0, 255).to(torch.uint8)
    if op == 7:
        return _aa_blend(img, _aa_gray(img), f, d)
    if op == 8:
        return _aa_blend(img, torch.mean(_aa_gray(img), dim=(-3, -2, -1), keepdim=True), f, d)
    if op == 9:
        if h <= 2 or w <= 2:
            return img.clone()
        a, b = 1.0 / 13.0, 5.0 / 13.0
        kernel = torch.tensor([[a, a, a], [a, b, a], [a, a, a]], dtype=torch.float32).expand(C, 1, 3, 3)
        out = img.to(torch.float32, copy=True)
        blurred = F.conv2d(out.unsqueeze(0), kernel, groups=C)[0].round_()
        view = out[..., 1:-1, 1:-1]
        view.add_(blurred.sub_(view), alpha=d)
        return out.clamp_(0, 255).to(torch.uint8)
    if op == 10:
        bits = int(f)
        return img.clone() if bits >= 8 else img & (((1 << bits) - 1) << (8 - bits))
    if op == 11:
        return torch.where(img >= f, 255 - img, img)
    if op == 12:
        fimg = img.to(torch.float32)
        lo = fimg.amin(dim=(-2, -1), keepdim=True)
        hi = fimg.amax(dim=(-2, -1), keepdim=True)
        eq = hi == lo
        inv = hi.sub_(lo).mul_(1.0 / 255)
        lo[eq] = 0.0
        inv[eq] = 1.0
        return fimg.sub_(lo).div_(inv).clamp_(0, 255).to(torch.uint8)
    if op == 13:                                              # PIL's equalize LUT, per channel; step == 0 leaves the channel as it is
        flat = img.flatten(start_dim=-2).to(torch.long)
        hist = torch.zeros((C, 256), dtype=torch.int32).scatter_add_(-1, flat, torch.ones_like(flat, dtype=torch.int32))
        cum = hist.cumsum(-1)
        last = cum.argmax(-1, keepdim=True)
        step = (flat.shape[-1] - hist.gather(-1, last)).div(255, rounding_mode="floor")
        lut = (cum[:, :-1] + step // 2).div(step.clamp(min=1), rounding_mode="floor").clamp_(0, 255).to(torch.uint8)
        lut = torch.cat([torch.zeros((C, 1), dtype=torch.uint8), lut], -1)
        eqd = lut.gather(-1, flat).view_as(img)
        return torch.where(step.ne(0).view(C, 1, 1), eqd, img)
    raise ValueError("aa_apply_op: unknown op %d" % op)


def augmix_mix(u, chains, weights):
    """AugMix's mix of one image, as torchvision's ``AugMix.forward`` computes it in fp32: mix = m₀·u, then mix.add_(w_i·chain_i)
    for each chain in order (a separate multiply and add each), then ``.to(uint8)``, which truncates.  ``u`` and ``chains[i]``: uint8
    tensors of one shape; ``weights``: (m₀, w_0, …) as fp32."""
    wt = torch.as_tensor(weights).float().cpu()
    mix = wt[0] * u
    for i, c in enumerate(chains):
        mix.add_(wt[1 + i] * c)
    return mix.to(torch.uint8)


def auto_augment_crop_normalize(x_u8, mean, std_scale, out_hw, boxes, flips, records, out_dtype=torch.float32, weights=None):
    """TrivialAugmentWide / RandAugment / AutoAugment on the (resized) crop, then normalisation: u = :func:`aa_crop_u8`; each op
    slot of ``records[i]`` (float32 [N, slots, 12]) applied in order by :func:`aa_apply_op`; out = (u' − m̂) * std_scale with m̂ the
    bilinear resample of a per-pixel mean over the same (mirrored) box (a [C] or scalar mean as it is).  Fill pixels become
    −m̂ * std_scale.  With ``weights`` (AugMix's float32 [N, 1 + width]) the slots are ``width`` chains of 3 that each start from u,
    and u' is :func:`augmix_mix` of u and the chains."""
    import torch.nn.functional as F
    N, H, W, C = x_u8.shape
    if isinstance(std_scale, torch.Tensor):
        std_scale = std_scale.to(dtype=torch.float32)
    mean = torch.as_tensor(mean).float()
    rec = torch.as_tensor(records).float().cpu()
    u = aa_crop_u8(x_u8.cpu(), out_hw, boxes, flips)
    out = torch.empty((N,) + tuple(out_hw) + (C,), dtype=torch.float32)
    for i in range(N):
        img = u[i].permute(2, 0, 1).contiguous()
        if weights is None:
            for r in rec[i]:
                img = aa_apply_op(img, r)
        else:
            chains = []
            for chain in rec[i].view(-1, 3, rec.shape[-1]):
                aug = img
                for r in chain:
                    aug = aa_apply_op(aug, r)
                chains.append(aug)
            img = augmix_mix(img, chains, weights[i])
        if mean.dim() == 3:
            y0, x0, h, w = (int(v) for v in boxes[i])
            box = mean.cpu()[y0:y0 + h, x0:x0 + w, :].permute(2, 0, 1).unsqueeze(0)
            m = F.interpolate(box, size=tuple(out_hw), mode="bilinear", align_corners=False, antialias=False)[0].permute(1, 2, 0)
            m = m.flip(1) if bool(flips[i]) else m
        else:
            m = mean.cpu()
        out[i] = (img.permute(1, 2, 0).float() - m) * (std_scale.cpu() if isinstance(std_scale, torch.Tensor) else std_scale)
    return out.to(device=x_u8.device, dtype=out_dtype)


def random_erase(x, boxes):
    """torchvision's ``RandomErasing(value=0)`` on an NHWC batch, given its boxes: a copy of ``x`` with every element of image i's box
    ``boxes[i] = (i0, j0, h, w)`` (output coordinates, inside the image; h = w = 0 erases nothing) set to 0.

    x: [N, H, W, C] float;  boxes: [N, 4] int (``models/data/utils.py: draw_erase_boxes``)
    """
    N, H, W, _ = x.shape
    out = x.clone()
    for n in range(N):
        i, j, h, w = (int(v) for v in boxes[n])
        if not (h >= 0 and w >= 0 and 0 <= i <= H - h and 0 <= j <= W - w):
            raise ValueError("random_erase: box %r of image %d is not inside %d x %d" % ((i, j, h, w), n, H, W))
        out[n, i:i + h, j:j + w, :] = 0
    return out


# --------------------------------------------------------------------------- batch norm (+ residual)(+ ReLU), NHWC
def _per_sample(s, x):
    """A drop-path row (one scale per sample of x's leading axis) shaped to broadcast over x."""
    return s.float().reshape((x.shape[0],) + (1,) * (x.dim() - 1))


def batch_norm_fwd(x, gamma, beta, run_mean, run_var, training, momentum, eps, relu, res=None, drop=None):
    """y = γ·(x − mean)·rstd + β [+ res] [ReLU]; statistics over all but the last (channel) axis.  Updates the running
    statistics in place (momentum form, unbiased variance) when training.  ``drop`` (a drop-path row, one scale s_n per sample,
    needs ``res``): y = act(s_n·(γ·x̂ + β) + res), the statistics still those of the whole batch.  Returns (y, mean, rstd)."""
    if drop is not None and res is None:
        raise ValueError("batch_norm: a drop-path row scales the branch of a residual add: needs res")
    xf = x.float()
    C = x.shape[-1]
    x2 = xf.reshape(-1, C)
    R = x2.shape[0]
    if training:
        mean = x2.mean(0)
        var = (x2 * x2).mean(0) - mean * mean
        var = var.clamp_min(0)
        if run_mean is not None:
            with torch.no_grad():
                run_mean.mul_(1 - momentum).add_(momentum * mean)
                run_var.mul_(1 - momentum).add_(momentum * var * (R / max(1, R - 1)))
    else:
        mean, var = run_mean.float(), run_var.float()
    rstd = torch.rsqrt(var + eps)
    y = (xf - mean) * (rstd * gamma.float()) + beta.float()
    if drop is not None:
        y = y * _per_sample(drop, x)
    if res is not None:
        y = y + res.float()
    return act_fwd(y, relu).to(x.dtype), mean, rstd


def batch_norm_bwd(x, dy, y, gamma, mean, rstd, relu, need_dres, drop=None):
    """Returns (dx, dres, dgamma, dbeta) for :func:`batch_norm_fwd` in training mode.  ``drop``: dx, dγ and dβ come from s_n·g,
    the residual gets g."""
    C = x.shape[-1]
    g = dy.float()
    if relu:
        g = act_bwd(g, y.float(), relu)
    gb = g if drop is None else g * _per_sample(drop, x)
    xh = (x.float() - mean) * rstd
    g2, xh2 = gb.reshape(-1, C), xh.reshape(-1, C)
    R = g2.shape[0]
    dbeta = g2.sum(0)
    dgamma = (g2 * xh2).sum(0)
    dx = (gamma.float() * rstd) * (gb - dbeta / R - xh * (dgamma / R))
    return dx.to(x.dtype), (g.to(x.dtype) if need_dres else None), dgamma, dbeta


def add_scaled(a, s, b=None):
    """s_n·a + b per sample n of the leading axis (b None: s_n·a) in fp32, rounded once to a's dtype: the drop-path merge of a
    pre-activation block (y = s·branch + shortcut) and its branch gradient s·dy."""
    y = a.float() * _per_sample(s, a)
    if b is not None:
        y = y + b.float()
    return y.to(a.dtype)
