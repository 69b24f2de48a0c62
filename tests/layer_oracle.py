"""float64 references of the streaming layer kernels (batch norm, pooling, LRN, softmax cross-entropy) written from each operation's
definition, and the two comparisons every test of those kernels goes through.  No GPU is needed: the functions run on the device of
their inputs, which the callers pass as float64 (a bf16 or fp32 value is exact in float64).

Conventions (those of the kernels in ``csrc/bn_kernels.cu`` / ``csrc/nn_kernels.cu``):

* activations are NHWC; batch norm reduces over all axes but the last, variance is the biased one, the running variance gets the
  unbiased one (R / (R − 1), 1 when R = 1), ``running ← (1 − momentum)·running + momentum·batch``;
* the backward of an activation takes its mask from the forward OUTPUT y (ReLU / leaky: y > 0, sigmoid: y·(1 − y));
* max pooling: padding never wins, the first maximum in window order t = kh·k + kw wins and t is the argmax; average pooling divides by
  the number of in-image taps (``count_include_pad=False``);
* LRN: ``y = x·(k + α·Σ_{|j − c| ≤ n/2} x_j²)^−β`` — α multiplies the window SUM (torch's ``local_response_norm`` divides α by n);
* softmax: label smoothing ε gives the target (1 − ε)·onehot + ε / C; the label's rank is #{z_c > z_y} + #{c < y : z_c = z_y}, the
  top-1 / top-5 error of a row is rank ≥ 1 / rank ≥ 5; dlogits is the gradient of the MEAN loss times ``grad_scale``.

Bounds.  ``assert_elementwise``: |got − want| ≤ u·|want| + u·s per element, u the unit roundoff class of the storage type and s the
magnitude of what was added up to make that element, so that cancellation is allowed for and nothing else.  ``assert_reduction``:
|got − want| ≤ RED_C·√n·2⁻²⁴·Σ|term| for an fp32 sum of n terms whose order the kernel is free to choose.
"""
import math

import torch
import torch.nn.functional as F

U_STORE = {torch.bfloat16: 2.0 ** -8, torch.float32: 2.0 ** -22}     # one bf16 rounding / a few fp32 roundings
VEC = {torch.bfloat16: 8, torch.float32: 4}                           # elements per 16-byte vector
RED_C = 4.0            # fp32 accumulation in per-thread, per-CTA and atomic stages: a random walk of 2^-24 steps, times this margin


def red_rel(n_terms):
    """Relative (to Σ|term|) error allowed to an fp32 sum of ``n_terms`` terms."""
    return RED_C * math.sqrt(max(int(n_terms), 1)) * 2.0 ** -24


def _where(flat, shape, dtype):
    idx = []
    for d in reversed(shape):
        idx.append(flat % d)
        flat //= d
    idx = tuple(reversed(idx))
    names = "nhwc" if len(shape) == 4 else ("rc" if len(shape) == 2 else None)
    pos = ", ".join("%s=%d" % (names[i], v) for i, v in enumerate(idx)) if names else str(idx)
    C = shape[-1] if shape else 1
    row = 0
    for d, v in zip(shape[:-1], idx[:-1]):
        row = row * d + v
    rows = 1
    for d in shape[:-1]:
        rows *= d
    vec = VEC[dtype]
    return "(%s): row %d of %d, channel vector %d of %d" % (pos, row, rows, idx[-1] // vec if shape else 0, (C + vec - 1) // vec)


def elementwise_violations(got, want64, dtype, s=None, extra_abs=None, slack=1.0):
    """(bad mask, |got − want|, bound) of :func:`assert_elementwise`."""
    want64 = want64.double()
    g = got.detach().to(want64.device).double()
    assert g.shape == want64.shape, (tuple(g.shape), tuple(want64.shape))
    u = U_STORE[dtype] * slack
    bound = u * want64.abs()
    if s is not None:
        bound = bound + u * s
    if extra_abs is not None:
        bound = bound + extra_abs
    diff = (g - want64).abs()
    return ~(diff <= bound), diff, bound           # ~(<=) so that a NaN is a violation


def assert_elementwise(got, want64, dtype, s=None, extra_abs=None, slack=1.0, what="output"):
    """Every element of ``got`` (storage type ``dtype``) is within u·|want| + u·s (+ ``extra_abs``) of the float64 ``want64``.
    ``s``: the magnitude of the terms that were added to make each element (broadcastable); ``extra_abs``: an absolute allowance
    the caller derived from a reduction bound (per-channel coefficients of a batch norm); ``slack`` multiplies u where the kernel
    uses the fast-math exp / log intrinsics."""
    bad, diff, bound = elementwise_violations(got, want64, dtype, s, extra_abs, slack)
    nbad = int(bad.sum())
    if nbad:
        excess = torch.where(bad, diff / bound.clamp_min(1e-300), torch.zeros_like(diff))
        excess = torch.where(torch.isnan(excess), torch.full_like(excess, float("inf")), excess)
        w = int(excess.reshape(-1).argmax())
        raise AssertionError("%s: %d of %d elements outside the bound; worst at %s: got %r want %r (|diff| %.3g, bound %.3g)" % (
            what, nbad, bad.numel(), _where(w, tuple(want64.shape), dtype), float(got.reshape(-1)[w]), float(want64.reshape(-1)[w]),
            float(diff.reshape(-1)[w]), float(bound.reshape(-1)[w])))


def assert_reduction(got, want64, abs_sum64, n_terms, extra_abs=None, what="sum"):
    """fp32 sums ``got`` against their float64 values: |got − want| ≤ RED_C·√n_terms·2⁻²⁴·Σ|term| (``abs_sum64``)."""
    want64 = torch.as_tensor(want64).double()
    g = torch.as_tensor(got).detach().to(want64.device).double()
    bound = red_rel(n_terms) * torch.as_tensor(abs_sum64).double().to(want64.device)
    if extra_abs is not None:
        bound = bound + extra_abs
    diff = (g - want64).abs()
    bad = ~(diff <= bound)
    if int(bad.sum()):
        w = int(torch.where(bad, diff / bound.clamp_min(1e-300), torch.zeros_like(diff)).reshape(-1).argmax())
        raise AssertionError("%s: %d of %d sums of %d terms outside the bound; worst at index %d: got %r want %r (|diff| %.3g, bound %.3g)" % (
            what, int(bad.sum()), bad.numel(), n_terms, w, float(g.reshape(-1)[w]), float(want64.reshape(-1)[w]),
            float(diff.reshape(-1)[w]), float(bound.reshape(-1)[w])))


def old_rel_err(a, b):
    """The metric of tests/test_gpu_kernels.py (largest error over the largest reference element), kept to show what it cannot see."""
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


# --------------------------------------------------------------------------- activations
def act_fwd64(z, act, slope=0.2):
    if act in (None, False, "none"):
        return z
    if act in (True, "relu"):
        return z.clamp_min(0.0)
    if act == "leaky":
        return torch.where(z > 0, z, z * slope)
    if act == "sigmoid":
        return torch.sigmoid(z)
    raise ValueError(act)


def act_bwd64(dy, y, act, slope=0.2):
    """Gradient through the activation, masked by its OUTPUT ``y`` (the kernel's own, rounded to storage)."""
    if act in (None, False, "none"):
        return dy
    if act in (True, "relu"):
        return torch.where(y > 0, dy, torch.zeros_like(dy))
    if act == "leaky":
        return torch.where(y > 0, dy, dy * slope)
    if act == "sigmoid":
        return dy * y * (1.0 - y)
    raise ValueError(act)


# --------------------------------------------------------------------------- batch norm
def _rows(t):
    return t.reshape(-1, t.shape[-1])


def _sample_scale(drop, x):
    """The drop-path row (one scale per sample of the leading axis) broadcast to the rows of ``x``."""
    per = x.numel() // x.shape[-1] // x.shape[0]
    return drop.double().repeat_interleave(per)[:, None]


def bn_fwd64(x, gamma, beta, eps=1e-5, act=None, res=None, drop=None, slope=0.2, training=True, run_mean=None, run_var=None, momentum=0.1):
    """``act(s_n·(γ·x̂ + β) + res)`` with batch (``training``) or running statistics.  Returns a dict: y, mean, var (biased), rstd,
    run_mean / run_var after the momentum update, the statistics' sums and Σ|term| (sum_x, sum_x2, abs_x), ``s`` (the magnitude of
    the terms of each y element) and ``coef_abs``: the absolute error of y that the reduction bound on Σx, Σx² allows through the
    per-channel scale and mean."""
    X = _rows(x.double())
    R = X.shape[0]
    gamma, beta = gamma.double(), beta.double()
    out = {}
    if training:
        mean = X.mean(0)
        var = ((X - mean) ** 2).mean(0)
        out["sum_x"], out["sum_x2"], out["abs_x"] = X.sum(0), (X * X).sum(0), X.abs().sum(0)
        if run_mean is not None:
            out["run_mean"] = (1 - momentum) * run_mean.double() + momentum * mean
            out["run_var"] = (1 - momentum) * run_var.double() + momentum * var * (R / (R - 1) if R > 1 else 1.0)
        d_mean = red_rel(R) * out["abs_x"] / R
        d_var = red_rel(R) * (out["sum_x2"] + 2 * mean.abs() * out["abs_x"]) / R + d_mean ** 2
        out["mean_abs"], out["var_abs"] = d_mean, d_var
    else:
        mean, var = run_mean.double(), run_var.double()
        d_mean = torch.zeros_like(mean)
        d_var = torch.zeros_like(var)
    rstd = (var + eps).rsqrt()
    scale = gamma * rstd
    shift = beta - mean * scale
    z = X * scale + shift
    s = (X * scale).abs() + (mean * scale).abs() + beta.abs()          # the shift β − mean·scale may itself have cancelled
    coef_abs = 0.5 * d_var / (var + eps) * (scale * (X - mean)).abs() + scale.abs() * d_mean
    if drop is not None:
        sn = _sample_scale(drop, x)
        z, s, coef_abs = z * sn, s * sn.abs(), coef_abs * sn.abs()
    if res is not None:
        z = z + _rows(res.double())
        s = s + _rows(res.double()).abs()
    out.update(y=act_fwd64(z, act, slope).reshape(x.shape), mean=mean, var=var, rstd=rstd, s=s.reshape(x.shape),
               coef_abs=coef_abs.reshape(x.shape))
    return out


def bn_bwd64(x, dy, y, gamma, mean, rstd, act=None, drop=None, slope=0.2):
    """Backward of :func:`bn_fwd64` from the statistics the forward SAVED (``mean``, ``rstd``: the kernel's own) and the mask of the
    kernel's own output ``y``: g = act'(y)·dy, g̃ = s_n·g; dβ = Σg̃, dγ = Σg̃·x̂, dx = γ·rstd·(g̃ − dβ/R − x̂·dγ/R), dres = g.  Returns a dict
    with those, Σ|term| of the two sums (abs_dbeta, abs_dgamma) and ``s_dx``: the magnitude of the terms of each dx element, the
    parts that come from the sums taken at Σ|term|."""
    X, DY = _rows(x.double()), _rows(dy.double())
    R = X.shape[0]
    gamma, mean, rstd = gamma.double(), mean.double(), rstd.double()
    g = act_bwd64(DY, _rows(y.double()), act, slope) if act not in (None, False, "none") else DY
    gt = g * _sample_scale(drop, x) if drop is not None else g
    xh = (X - mean) * rstd
    dbeta, dgamma = gt.sum(0), (gt * xh).sum(0)
    abs_db, abs_dg = gt.abs().sum(0), (gt * xh).abs().sum(0)
    k1 = gamma * rstd
    dx = k1 * (gt - dbeta / R - xh * dgamma / R)
    s_dx = k1.abs() * (gt.abs() + abs_db / R + (X.abs() + mean.abs()) * rstd * abs_dg / R)
    return dict(dx=dx.reshape(x.shape), dres=g.reshape(x.shape), dgamma=dgamma, dbeta=dbeta, abs_dgamma=abs_dg, abs_dbeta=abs_db,
                s_dx=s_dx.reshape(x.shape))


# --------------------------------------------------------------------------- pooling
def pool_out_hw(H, W, k, s, p):
    return (H + 2 * p - k) // s + 1, (W + 2 * p - k) // s + 1


def _windows(x, k, s, p, fill):
    """[N, Ho, Wo, C, k·k] taps of the NHWC ``x`` in window order t = kh·k + kw; out-of-image taps hold ``fill``."""
    xp = F.pad(x.permute(0, 3, 1, 2), (p, p, p, p), value=fill)
    w = xp.unfold(2, k, s).unfold(3, k, s)                       # [N, C, Ho, Wo, k, k]
    return w.reshape(*w.shape[:4], k * k).permute(0, 2, 3, 1, 4)


def pool64(x, k, s, p, mode):
    """Returns (y, arg, s): ``arg`` the winning tap t per output for max pooling (None for avg), ``s`` the largest |tap| of each
    output (the magnitude an average is built from)."""
    x = x.double()
    if mode == "max":
        w = _windows(x, k, s, p, float("-inf"))
        y = w.max(-1).values
        t = torch.arange(k * k, device=x.device)
        arg = torch.where(w == y[..., None], t, torch.full_like(t, k * k)).min(-1).values      # first maximum in window order
        return y, arg, None
    w = _windows(x, k, s, p, 0.0)
    cnt = _windows(torch.ones_like(x[..., :1]), k, s, p, 0.0).sum(-1)
    return w.sum(-1) / cnt, None, w.abs().max(-1).values


def pool_bwd64(dy, arg, xshape, k, s, p, mode):
    """Returns (dx, s): dx[n, h, w, c] = Σ over the windows whose argmax is (h, w) of dy (max) or Σ over covering windows of
    dy / in-image count (avg); ``s`` the same sum over |dy|."""
    N, H, W, C = xshape
    dy = dy.double()
    Ho, Wo = dy.shape[1], dy.shape[2]
    if mode == "max":
        contrib = F.one_hot(arg, k * k).double() * dy[..., None]                               # [N, Ho, Wo, C, k·k]
    else:
        cnt = _windows(torch.ones(N, H, W, 1, dtype=torch.float64, device=dy.device), k, s, p, 0.0).sum(-1)
        contrib = (dy / cnt)[..., None].expand(N, Ho, Wo, C, k * k)
    dxp = torch.zeros(N, H + 2 * p, W + 2 * p, C, dtype=torch.float64, device=dy.device)
    sp = torch.zeros_like(dxp)
    for kh in range(k):
        for kw in range(k):
            sl = (slice(None), slice(kh, kh + s * (Ho - 1) + 1, s), slice(kw, kw + s * (Wo - 1) + 1, s))
            dxp[sl] += contrib[..., kh * k + kw]
            sp[sl] += contrib[..., kh * k + kw].abs()
    return dxp[:, p:p + H, p:p + W], sp[:, p:p + H, p:p + W]


# --------------------------------------------------------------------------- LRN
def _chan_window_sum(t, n):
    h = n // 2
    return F.pad(t, (h, h)).unfold(-1, n, 1).sum(-1)


def lrn64(x, n=5, k=2.0, alpha=1e-4, beta=0.75):
    """y = x·(k + α·Σ_{window} x²)^−β over the channel (last) axis, any odd n."""
    assert n % 2 == 1
    x = x.double()
    return x * (k + alpha * _chan_window_sum(x * x, n)) ** -beta


def lrn_bwd64(x, dy, n=5, k=2.0, alpha=1e-4, beta=0.75):
    """Returns (dx, s): dx_c = dy_c·d_c^−β − 2αβ·x_c·Σ_{|i − c| ≤ n/2} dy_i·x_i·d_i^(−β−1) and the magnitude of its terms."""
    assert n % 2 == 1
    x, dy = x.double(), dy.double()
    d = k + alpha * _chan_window_sum(x * x, n)
    t = dy * x * d ** (-beta - 1)
    a = dy * d ** -beta
    dx = a - 2 * alpha * beta * x * _chan_window_sum(t, n)
    return dx, a.abs() + 2 * alpha * beta * x.abs() * _chan_window_sum(t.abs(), n)


# --------------------------------------------------------------------------- softmax + cross-entropy + top-k
def label_rank(z, labels):
    """rank = #{z_c > z_y} + #{c < y : z_c = z_y}: the number of classes placed before the label."""
    zy = z.gather(1, labels[:, None])
    c = torch.arange(z.shape[1], device=z.device)[None, :]
    return (z > zy).sum(1) + ((z == zy) & (c < labels[:, None])).sum(1)


def softmax_xent64(z, labels, label_smoothing=0.0, grad_scale=1.0):
    """Returns a dict: loss (mean over rows of −Σ q·log p), dlogits ((p − q)/B·grad_scale), err1 / err5 (mean of rank ≥ 1 / rank ≥ 5),
    abs_loss (mean over rows of the magnitudes the row loss is computed from: |z_y − max|, |log Σe^(z − max)|, ε/C·Σ|z − max|, and 1 for
    the absolute error of the exp / log intrinsics)."""
    z = z.double()
    B, C = z.shape
    eps = float(label_smoothing)
    lsm = torch.log_softmax(z, 1)
    q = torch.full_like(z, eps / C)
    q.scatter_add_(1, labels[:, None], torch.full((B, 1), 1.0 - eps, dtype=z.dtype, device=z.device))
    rows = -(q * lsm).sum(1)
    rank = label_rank(z, labels)
    zm = z - z.max(1, keepdim=True).values
    abs_rows = zm.gather(1, labels[:, None])[:, 0].abs() + zm.exp().sum(1).log().abs() + eps / C * zm.abs().sum(1) + 1.0
    return dict(loss=rows.mean(), dlogits=(lsm.exp() - q) / B * grad_scale, err1=(rank >= 1).double().mean(),
                err5=(rank >= 5).double().mean(), abs_loss=abs_rows.mean(), rank=rank)
