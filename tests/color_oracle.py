"""Float64 oracle of colour jitter and PCA lighting on the loader's crops (``config['color_jitter']``).

The oracle applies fb.resnet.torch's operations one at a time, as that code writes them, on the resampled raw crop v (0…255 RGB):
brightness v ← a·v; saturation v ← s·v + (1 − s)·gray(v); contrast v ← c·v + (1 − c)·mean(gray(v)), the mean over the crop; in the
drawn order; then lighting v ← v + 255·E·(α ∘ λ).  Then (v − m̂)·s_c and the flip.  The composed per-image records of
``utils.color_jitter_records`` are checked against it, and it gives the references and bounds of the GPU tests.

The resample is the kernel's definition: per axis of box length L and output length n, the fp32 source coordinate
s = max(fl(fl(L / n)·(o + ½) − ½), 0) (one rounding, as the kernel's fused multiply-add), i0 = ⌊s⌋ clamped to L − 1,
i1 = i0 + (i0 < L − 1), λ = fl(s − i0) and 1 − λ rounded to fp32; the blend of the four taps with these weights is then exact (fp64).
"""
import numpy as np

from theanompi_b200.models.data.utils import CJ_EIGVAL, CJ_EIGVEC, CJ_GRAY

EPS32 = 2.0 ** -24


def axis_taps(L, n):
    """(i0, i1, w0, w1) of the n output positions of an axis of length L, with the kernel's fp32 weights."""
    ratio = np.float32(L) / np.float32(n)
    o = np.arange(n, dtype=np.float64)
    s = np.maximum((np.float64(ratio) * (o + 0.5) - 0.5).astype(np.float32), np.float32(0))
    i0 = np.minimum(s.astype(np.int64), L - 1)
    i1 = i0 + (i0 < L - 1)
    lam = np.clip(s - i0.astype(np.float32), np.float32(0), np.float32(1)).astype(np.float32)
    return i0, i1, (np.float32(1) - lam).astype(np.float64), lam.astype(np.float64)


def resample(img, box, out_hw):
    """Bilinear resample of ``img[y0:y0+h, x0:x0+w]`` ([H, W, C], float64) to ``out_hw``, unmirrored."""
    y0, x0, h, w = (int(v) for v in box)
    yi0, yi1, wy0, wy1 = axis_taps(h, out_hw[0])
    xi0, xi1, wx0, wx1 = axis_taps(w, out_hw[1])
    b = np.asarray(img, np.float64)[y0:y0 + h, x0:x0 + w]
    r0 = wx0[None, :, None] * b[yi0][:, xi0] + wx1[None, :, None] * b[yi0][:, xi1]
    r1 = wx0[None, :, None] * b[yi1][:, xi0] + wx1[None, :, None] * b[yi1][:, xi1]
    return wy0[:, None, None] * r0 + wy1[:, None, None] * r1


def lighting(alpha):
    """ℓ = 255·E·(α ∘ λ) for α [n, 3]."""
    return 255.0 * (np.asarray(alpha, np.float64) * CJ_EIGVAL) @ CJ_EIGVEC.T


def apply_sequential(v, factors, order, alpha):
    """fb.resnet.torch's ColorJitter (operation k of ``order``: 0 brightness, 1 saturation, 2 contrast, with factors (a, s, c))
    then Lighting, one step at a time on one image's crop v [h, w, 3] (float64)."""
    v = np.array(v, np.float64)
    a, s, c = factors
    for op in order:
        if op == 0:
            v = a * v
        elif op == 1:
            v = s * v + (1.0 - s) * (v @ CJ_GRAY)[..., None]
        else:
            v = c * v + (1.0 - c) * (v @ CJ_GRAY).mean()
    return v + lighting(np.asarray(alpha)[None])[0]


def _mean_hat(mean, box, out_hw):
    m = np.asarray(mean, np.float64)
    return resample(m, box, out_hw) if m.ndim == 3 else np.broadcast_to(m.reshape(-1), tuple(out_hw) + (3,))


def oracle(x_u8, mean, std_scale, out_hw, boxes, flips, factors, order, alpha, records):
    """(want, S): the float64 model input [N, h, w, 3] of the sequential application, and the per-element magnitude
    S = (|M|·v̂ + |K|·μ + |ℓ| + |m̂|)·s_c of the terms the kernel sums, with (M, K, ℓ) from ``records``."""
    x = np.asarray(x_u8)
    sc = np.broadcast_to(np.asarray(std_scale, np.float64).reshape(-1), (3,))
    rec = np.asarray(records, np.float64)
    want = np.empty((x.shape[0],) + tuple(out_hw) + (3,))
    S = np.empty_like(want)
    for i in range(x.shape[0]):
        v = resample(x[i], boxes[i], out_hw)
        m = _mean_hat(mean, boxes[i], out_hw)
        y = (apply_sequential(v, factors[i], order[i], alpha[i]) - m) * sc
        M, K, ell = np.abs(rec[i, 0:9].reshape(3, 3)), np.abs(rec[i, 9:18].reshape(3, 3)), np.abs(rec[i, 18:21])
        mu = v.reshape(-1, 3).mean(0)
        s = (v @ M.T + K @ mu + ell + np.abs(m)) * sc
        if flips[i]:
            y, s = y[:, ::-1], s[:, ::-1]
        want[i], S[i] = y, s
    return want, S


def crop_sums(x_u8, boxes, out_hw):
    """Float64 sums of v̂ over each output crop, [N, 3]."""
    return np.stack([resample(np.asarray(x_u8[i]), boxes[i], out_hw).reshape(-1, 3).sum(0) for i in range(len(boxes))])


def assert_bounded(got, want, S, u, what=""):
    """|got − want| ≤ u·|want| + u·S per element; a failure names the (n, y, x, c) of the worst element."""
    got = np.asarray(got, np.float64)
    err = np.abs(got - want)
    bound = u * np.abs(want) + u * S
    bad = err > bound
    if bad.any():
        r = err / np.maximum(bound, 1e-300)
        idx = np.unravel_index(np.argmax(r), r.shape)
        raise AssertionError("%s: %d elements out of bound; worst (n, y, x, c) = %s: got %r want %r bound %.3g (err / bound %.3g)" % (
            what, int(bad.sum()), idx, float(got[idx]), float(want[idx]), float(bound[idx]), float(r[idx])))
    return float((err / np.maximum(bound, 1e-300)).max())
