"""Data helpers (ref ``theanompi/models/data/utils.py``): ``unpickle`` (``:3-12``),
``get_bad_list``/``extend_data`` — pad the file list to a multiple of the world
size (``:15-40``), ``get_rand3d`` and the CPU ``crop_and_mirror`` (``:42-129``).

Images are NHWC ``[N, H, W, C]`` here (the reference used c01b).  The CPU
``crop_and_mirror`` is kept as the host fallback and as ground truth for the device
kernel (``csrc/data_kernels.cu``), which does normalise + crop + mirror + bf16 cast in
one pass after the pinned H2D copy.
"""
from __future__ import annotations

import math
import os
import pickle

import numpy as np

_COPY_POOL = None


def parallel_copyto(out, src, threads=None, min_bytes=4 << 20):
    """``np.copyto(out, src)`` split over a few threads along the first axis.  One core moves a 25 MB file batch out of the
    page cache at 4–6 GB/s (≈ 4–6 ms) — slower than an H100 consumes it (AlexNet-128b: one batch per 3 ms), so the host copy of
    the loader can be spread over ``TMPI_LOADER_THREADS`` cores (default 1; numpy releases the GIL inside each slice copy).  On a
    host where one core already saturates the memory bandwidth more threads do not help (``scripts/loader_host_bench.py``
    measures it)."""
    global _COPY_POOL
    n = int(threads or os.environ.get("TMPI_LOADER_THREADS", "1"))
    n = max(1, min(n, len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else n, int(out.shape[0]) if out.ndim else 1))
    if n == 1 or out.nbytes < min_bytes:
        np.copyto(out, src)
        return
    if _COPY_POOL is None or _COPY_POOL._max_workers < n:
        from concurrent.futures import ThreadPoolExecutor
        _COPY_POOL = ThreadPoolExecutor(max_workers=n, thread_name_prefix="tmpi-copy")
    rows = int(out.shape[0])
    step = (rows + n - 1) // n
    futs = [_COPY_POOL.submit(np.copyto, out[a:a + step], src[a:a + step]) for a in range(0, rows, step)]
    for f in futs:
        f.result()


def unpickle(path):
    with open(path, "rb") as f:
        try:
            return pickle.load(f, encoding="latin1")
        except TypeError:
            return pickle.load(f)


def get_bad_list(n_batches, commsize):
    bad_left = n_batches % commsize
    return [n_batches - (bad + 1) for bad in range(bad_left)]


def extend_data(rank, size, img_batches, label_batches, verbose=False):
    """Repeat trailing batches so ``len % size == 0`` (every rank gets the same
    number of file batches)."""
    _img = list(img_batches)
    n_files = len(_img)
    _lab = list(label_batches[:n_files])
    bad_left_list = get_bad_list(n_files, size)
    need = (size - len(bad_left_list)) % size
    if need != 0:
        _img.extend(_img[-need:])
        _lab.extend(_lab[-need:])
    assert len(_img) % size == 0
    if rank == 0 and verbose:
        print("rank%d: bad list is %s, extended to %d" % (rank, str(bad_left_list), len(_img)))
    return _img, _lab


def get_rand3d(rand_crop, mode, rs=None):
    """Three uniforms in [0,1): (y-offset, x-offset, flip); 0.5/0.5/0 for val."""
    if not rand_crop or mode == "val":
        return np.float32([0.5, 0.5, 0])
    rs = rs or np.random
    return np.float32(rs.rand(3))


def draw_crops(n, in_hw, out_hw, mode, rand_crop=True, batch_crop_mirror=False, rs=None):
    """Per-image (y0, x0) offsets and flip flags; centre crop / no flip for val."""
    H, W = in_hw
    ch, cw = out_hw
    rs = rs or np.random
    if mode == "val" or not rand_crop:
        offs = np.tile(np.int32([[(H - ch) // 2, (W - cw) // 2]]), (n, 1))
        return offs, np.zeros(n, dtype=np.uint8)
    if batch_crop_mirror:
        r = get_rand3d(True, mode, rs)
        offs = np.tile(np.int32([[int(r[0] * (H - ch + 1)), int(r[1] * (W - cw + 1))]]), (n, 1))
        flips = np.full(n, int(r[2] > 0.5), dtype=np.uint8)
        return offs, flips
    oy = rs.randint(0, H - ch + 1, n)
    ox = rs.randint(0, W - cw + 1, n)
    flips = (rs.rand(n) > 0.5).astype(np.uint8)
    return np.stack([oy, ox], 1).astype(np.int32), flips


RRC_KEY = "random_resized_crop"
RRC_DEFAULTS = {"scale": (0.08, 1.0), "ratio": (3.0 / 4.0, 4.0 / 3.0), "seed": 0}
RRC_ATTEMPTS = 10


def _real(v):
    return not isinstance(v, bool) and isinstance(v, (int, float, np.integer, np.floating)) and math.isfinite(v)


def check_resized_crop(cfg):
    """The validated ``config['random_resized_crop']`` with every key filled in (``scale`` and ``ratio`` as float pairs), or None for
    None; anything else is a ValueError that names the key.  Lists and tuples are both accepted, so the value survives JSON."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError("%s must be a dict or None, not %r" % (RRC_KEY, cfg))
    unknown = sorted(str(k) for k in cfg if k not in RRC_DEFAULTS)
    if unknown:
        raise ValueError("%s: unknown key %r; the keys are %s" % (RRC_KEY, unknown[0], ", ".join(RRC_DEFAULTS)))
    out = {}
    for k in ("scale", "ratio"):
        v = cfg.get(k, RRC_DEFAULTS[k])
        if not (isinstance(v, (list, tuple)) and len(v) == 2 and all(_real(e) for e in v)):
            raise ValueError("%s[%r] must be two finite real numbers [lo, hi], not %r" % (RRC_KEY, k, v))
        lo, hi = float(v[0]), float(v[1])
        if not (0.0 < lo <= hi and (k == "ratio" or hi <= 1.0)):
            raise ValueError("%s[%r] must satisfy %s, not %r" % (RRC_KEY, k, "0 < lo <= hi <= 1" if k == "scale" else "0 < lo <= hi", v))
        out[k] = (lo, hi)
    seed = cfg.get("seed", 0)
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise ValueError("%s['seed'] must be an int, not %r" % (RRC_KEY, seed))
    out["seed"] = int(seed) & (2 ** 64 - 1)
    return out


def resized_crop_rng(cfg, rank):
    """The box / flip generator of one worker, keyed by (seed, rank); separate from the fixed-crop RandomState, so a run without the
    key draws what it always drew."""
    return np.random.default_rng([cfg["seed"], int(rank)])


def draw_resized_crops(n, in_hw, scale, ratio, rng):
    """Per-image boxes (y0, x0, h, w) (int32 [n, 4]) and flip flags (uint8 [n], p = ½), drawn as torchvision's
    ``RandomResizedCrop.get_params``: up to 10 attempts of area H·W·U(scale) and ratio exp(U(log ratio)), w = round(√(area·r)),
    h = round(√(area / r)) (round half to even); the first attempt that fits sits at a uniform position, an image without one
    takes the centred box with the ratio clamped to its bounds.  All attempts of the batch are drawn at once."""
    H, W = in_hw
    lr = np.log(ratio)
    area = (H * W) * rng.uniform(scale[0], scale[1], (n, RRC_ATTEMPTS))
    r = np.exp(rng.uniform(lr[0], lr[1], (n, RRC_ATTEMPTS)))
    w = np.rint(np.sqrt(area * r)).astype(np.int64)
    h = np.rint(np.sqrt(area / r)).astype(np.int64)
    fits = (w > 0) & (w <= W) & (h > 0) & (h <= H)
    first = np.argmax(fits, axis=1)
    ok = fits[np.arange(n), first]
    h, w = h[np.arange(n), first], w[np.arange(n), first]
    # the fallback, torchvision's centred box (at least one pixel: a ratio far outside the image's can round a side to 0)
    in_r = W / H
    if in_r < ratio[0]:
        fh, fw = max(1, int(round(W / ratio[0]))), W
    elif in_r > ratio[1]:
        fh, fw = H, max(1, int(round(H * ratio[1])))
    else:
        fh, fw = H, W
    h, w = np.where(ok, h, fh), np.where(ok, w, fw)
    y0 = np.where(ok, rng.integers(0, H - h + 1), (H - fh) // 2)
    x0 = np.where(ok, rng.integers(0, W - w + 1), (W - fw) // 2)
    flips = (rng.random(n) < 0.5).astype(np.uint8)
    return np.stack([y0, x0, h, w], 1).astype(np.int32), flips


def crop_and_mirror(data, mode, rand_crop, flag_batch, cropsize, rs=None):
    """Host reference: ``data`` is NHWC float/uint8; returns NHWC ``cropsize²`` crops."""
    n, H, W, C = data.shape
    offs, flips = draw_crops(n, (H, W), (cropsize, cropsize), mode, rand_crop, flag_batch, rs)
    out = np.empty((n, cropsize, cropsize, C), dtype=data.dtype)
    for i in range(n):
        y0, x0 = offs[i]
        patch = data[i, y0:y0 + cropsize, x0:x0 + cropsize, :]
        out[i] = patch[:, ::-1, :] if flips[i] else patch
    return np.ascontiguousarray(out)
