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


CJ_KEY = "color_jitter"
CJ_STRENGTHS = ("brightness", "contrast", "saturation", "lighting")
CJ_DEFAULTS = {"brightness": 0.0, "contrast": 0.0, "saturation": 0.0, "lighting": 0.0, "seed": 0}
CJ_GRAY = np.array([0.299, 0.587, 0.114])                      # fb.resnet.torch's grayscale weights
# the ImageNet RGB eigen-decomposition of fb.resnet.torch's Lighting (Krizhevsky et al. 2012): eigenvalues and eigenvectors (columns)
CJ_EIGVAL = np.array([0.2175, 0.0188, 0.0045])
CJ_EIGVEC = np.array([[-0.5675, 0.7192, 0.4009],
                      [-0.5808, -0.0045, -0.8140],
                      [-0.5836, -0.6948, 0.4203]])
CJ_RECORD_FLOATS = 24                                          # M (3×3), K (3×3), ℓ (3), 3 zeros: 96 bytes, six float4


def check_color_jitter(cfg):
    """The validated ``config['color_jitter']`` with every key filled in (the four strengths as floats in [0, 1], at least one of them
    positive, and an int seed), or None for None; anything else is a ValueError that names the key."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError("%s must be a dict or None, not %r" % (CJ_KEY, cfg))
    unknown = sorted(str(k) for k in cfg if k not in CJ_DEFAULTS)
    if unknown:
        raise ValueError("%s: unknown key %r; the keys are %s" % (CJ_KEY, unknown[0], ", ".join(CJ_DEFAULTS)))
    out = {}
    for k in CJ_STRENGTHS:
        v = cfg.get(k, CJ_DEFAULTS[k])
        if not _real(v):
            raise ValueError("%s[%r] must be a finite real number, not %r" % (CJ_KEY, k, v))
        if not 0.0 <= float(v) <= 1.0:
            raise ValueError("%s[%r] must lie in [0, 1], not %r" % (CJ_KEY, k, v))
        out[k] = float(v)
    if not any(out[k] > 0.0 for k in CJ_STRENGTHS):
        raise ValueError("%s: at least one of %s must be > 0" % (CJ_KEY, ", ".join(CJ_STRENGTHS)))
    seed = cfg.get("seed", 0)
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise ValueError("%s['seed'] must be an int, not %r" % (CJ_KEY, seed))
    out["seed"] = int(seed) & (2 ** 64 - 1)
    return out


def color_jitter_rng(cfg, rank):
    """The colour generator of one worker, keyed by (seed, rank, 1): apart from the random-resized-crop generator and the fixed-crop
    RandomState, so turning the key on or off changes neither the boxes nor the crops drawn."""
    return np.random.default_rng([cfg["seed"], int(rank), 1])


def color_jitter_records(n, cfg, rng):
    """Per-image colour maps of fb.resnet.torch's ``ColorJitter`` (brightness, saturation, contrast in a random order) then
    ``Lighting``, composed into the affine map v' = M·v + K·μ + ℓ of an output pixel's RGB v (0…255) and the crop's mean RGB μ.

    Each image draws, whatever the strengths: three uniforms for the factors (a, s, c) = 1 + U(−strength, strength), three uniforms
    whose argsort is the order of the three operations (0 brightness, 1 saturation, 2 contrast; first applied first), three normals for
    α = N(0, lighting).  All of the batch is drawn at once.  Starting from (M, K) = (I, 0), with G = 𝟙gᵀ the grayscale projection:
    brightness (a·M, a·K); saturation P = s·I + (1 − s)·G, (P·M, P·K); contrast (c·M, c·K + (1 − c)·G·(M + K)), since the crop mean
    of M·v + K·μ is (M + K)·μ.  ℓ = 255·E·(α ∘ λ).  Composed in float64, rounded once.  The three operations commute (g sums to 1),
    so the order moves the record only by rounding; it is drawn so the stream follows fb.resnet.torch's ``RandomOrder``.

    Returns (records float32 [n, 24]: M row-major, K row-major, ℓ, three zeros; factors float64 [n, 3] (a, s, c); order int64 [n, 3];
    alpha float64 [n, 3])."""
    u = rng.random((n, 6))
    alpha = rng.standard_normal((n, 3)) * cfg["lighting"]
    strength = np.array([cfg["brightness"], cfg["saturation"], cfg["contrast"]])
    factors = 1.0 + strength * (2.0 * u[:, :3] - 1.0)
    order = np.argsort(u[:, 3:], axis=1, kind="stable")
    M, K, ell = color_jitter_maps(factors, order, alpha)
    rec = np.zeros((n, CJ_RECORD_FLOATS), np.float32)
    rec[:, 0:9] = M.reshape(n, 9)
    rec[:, 9:18] = K.reshape(n, 9)
    rec[:, 18:21] = ell
    return rec, factors, order, alpha


def color_jitter_maps(factors, order, alpha):
    """The float64 (M [n, 3, 3], K [n, 3, 3], ℓ [n, 3]) of :func:`color_jitter_records` for given factors, orders and α."""
    n = len(factors)
    G = np.outer(np.ones(3), CJ_GRAY)
    M = np.broadcast_to(np.eye(3), (n, 3, 3)).copy()
    K = np.zeros((n, 3, 3))
    a, s, c = (np.asarray(factors, np.float64)[:, i][:, None, None] for i in range(3))
    P = s * np.eye(3) + (1.0 - s) * G
    for pos in range(3):
        op = np.asarray(order)[:, pos][:, None, None]
        M, K = (np.where(op == 0, a * M, np.where(op == 1, P @ M, c * M)),
                np.where(op == 0, a * K, np.where(op == 1, P @ K, c * K + (1.0 - c) * (G @ (M + K)))))
    return M, K, 255.0 * (np.asarray(alpha, np.float64) * CJ_EIGVAL) @ CJ_EIGVEC.T


AA_KEY = "auto_augment"
AA_DEFAULTS = {"policy": "trivial_wide", "num_ops": 2, "magnitude": 9, "num_magnitude_bins": 31, "seed": 0, "interpolation": None,
               "severity": 3, "mixture_width": 3, "chain_depth": -1, "alpha": 1.0, "all_ops": True}
AA_POLICIES = ("trivial_wide", "rand", "autoaugment", "augmix")
# the keys that belong to some policies only; "seed" and "interpolation" belong to all four
AA_POLICY_KEYS = {"num_ops": ("rand",), "magnitude": ("rand",), "num_magnitude_bins": ("trivial_wide", "rand"),
                  "severity": ("augmix",), "mixture_width": ("augmix",), "chain_depth": ("augmix",), "alpha": ("augmix",),
                  "all_ops": ("augmix",)}
AA_INTERPOLATIONS = ("nearest", "bilinear")
# torchvision's default interpolation of each policy
AA_DEFAULT_INTERPOLATION = {"trivial_wide": "nearest", "rand": "nearest", "autoaugment": "nearest", "augmix": "bilinear"}
# torchvision's op set of TrivialAugmentWide and RandAugment, in their order; the op id is the index
AA_OPS = ("Identity", "ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Brightness", "Color", "Contrast", "Sharpness",
          "Posterize", "Solarize", "AutoContrast", "Equalize")
AA_INVERT = 14                                                 # AutoAugment's Invert, 255 − v
AA_NONE = 15                                                   # an AugMix chain step past the chain's depth: nothing is done
AA_OP_IDS = dict({k: i for i, k in enumerate(AA_OPS)}, Invert=AA_INVERT)
AA_SIGNED = frozenset(AA_OPS[1:10])
AA_LUT_OPS = frozenset((6, 8, 10, 11, 12, 13, AA_INVERT))       # point ops applied through a per-image, per-channel 256-entry LUT
AA_RECORD_FLOATS = 12                     # op, scalar, 1 − factor, bilinear (0 / 1), inverse affine matrix (6), 0, 0: 48 bytes
AA_CHAIN_SLOTS = 3                                             # op slots per AugMix chain (the largest chain_depth)
AA_BINS = 10                                                   # magnitude bins of AutoAugment and AugMix (torchvision's _PARAMETER_MAX)
# torchvision.transforms.v2.AutoAugment's ImageNet policy: 25 sub-policies of two (op, probability, magnitude bin or None)
AA_IMAGENET_POLICY = (
    (("Posterize", 0.4, 8), ("Rotate", 0.6, 9)), (("Solarize", 0.6, 5), ("AutoContrast", 0.6, None)),
    (("Equalize", 0.8, None), ("Equalize", 0.6, None)), (("Posterize", 0.6, 7), ("Posterize", 0.6, 6)),
    (("Equalize", 0.4, None), ("Solarize", 0.2, 4)), (("Equalize", 0.4, None), ("Rotate", 0.8, 8)),
    (("Solarize", 0.6, 3), ("Equalize", 0.6, None)), (("Posterize", 0.8, 5), ("Equalize", 1.0, None)),
    (("Rotate", 0.2, 3), ("Solarize", 0.6, 8)), (("Equalize", 0.6, None), ("Posterize", 0.4, 6)),
    (("Rotate", 0.8, 8), ("Color", 0.4, 0)), (("Rotate", 0.4, 9), ("Equalize", 0.6, None)),
    (("Equalize", 0.0, None), ("Equalize", 0.8, None)), (("Invert", 0.6, None), ("Equalize", 1.0, None)),
    (("Color", 0.6, 4), ("Contrast", 1.0, 8)), (("Rotate", 0.8, 8), ("Color", 1.0, 2)),
    (("Color", 0.8, 8), ("Solarize", 0.8, 7)), (("Sharpness", 0.4, 7), ("Invert", 0.6, None)),
    (("ShearX", 0.6, 5), ("Equalize", 1.0, None)), (("Color", 0.4, 0), ("Equalize", 0.6, None)),
    (("Equalize", 0.4, None), ("Solarize", 0.2, 4)), (("Solarize", 0.6, 5), ("AutoContrast", 0.6, None)),
    (("Invert", 0.6, None), ("Equalize", 1.0, None)), (("Color", 0.6, 4), ("Contrast", 1.0, 8)),
    (("Equalize", 0.8, None), ("Equalize", 0.6, None)))
# torchvision's AugMix op spaces, in their order: _PARTIAL_AUGMENTATION_SPACE (all_ops False) and _AUGMENTATION_SPACE
AA_AUGMIX_OPS = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate", "Posterize", "Solarize", "AutoContrast", "Equalize",
                 "Brightness", "Color", "Contrast", "Sharpness")
AA_AUGMIX_PARTIAL = 9


def _aa_int(cfg, k):
    v = cfg.get(k, AA_DEFAULTS[k])
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
        raise ValueError("%s[%r] must be an int, not %r" % (AA_KEY, k, v))
    return int(v)


def check_auto_augment(cfg):
    """The validated ``config['auto_augment']`` with every key of its policy filled in, or None for None; anything else is a
    ValueError that names the key.  ``num_ops`` and ``magnitude`` belong to "rand", ``num_magnitude_bins`` to "trivial_wide" and
    "rand", ``severity``, ``mixture_width``, ``chain_depth``, ``alpha`` and ``all_ops`` to "augmix".  ``interpolation`` ("nearest"
    or "bilinear") is accepted by every policy; it is filled in for "autoaugment" and "augmix", and kept for "trivial_wide" and
    "rand" only when given, so their validated dicts are what they always were (:func:`aa_bilinear` reads it)."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError("%s must be a dict or None, not %r" % (AA_KEY, cfg))
    unknown = sorted(str(k) for k in cfg if k not in AA_DEFAULTS)
    if unknown:
        raise ValueError("%s: unknown key %r; the keys are %s" % (AA_KEY, unknown[0], ", ".join(AA_DEFAULTS)))
    policy = cfg.get("policy", AA_DEFAULTS["policy"])
    if policy not in AA_POLICIES:
        raise ValueError("%s['policy'] must be one of %s, not %r" % (AA_KEY, ", ".join(AA_POLICIES), policy))
    for k, owners in AA_POLICY_KEYS.items():
        if k in cfg and policy not in owners:
            raise ValueError("%s[%r] belongs to policy %s, not %r" % (AA_KEY, k, " / ".join(repr(p) for p in owners), policy))
    out = {"policy": policy}
    if policy in ("trivial_wide", "rand"):
        for k in ("num_magnitude_bins", "num_ops", "magnitude", "seed"):
            out[k] = _aa_int(cfg, k)
        if out["num_magnitude_bins"] < 2:
            raise ValueError("%s['num_magnitude_bins'] must be >= 2, not %r" % (AA_KEY, out["num_magnitude_bins"]))
        if not 1 <= out["num_ops"] <= 4:
            raise ValueError("%s['num_ops'] must lie in [1, 4], not %r" % (AA_KEY, out["num_ops"]))
        if not 0 <= out["magnitude"] <= out["num_magnitude_bins"] - 1:
            raise ValueError("%s['magnitude'] must lie in [0, num_magnitude_bins - 1], not %r" % (AA_KEY, out["magnitude"]))
        if policy == "trivial_wide":
            del out["num_ops"], out["magnitude"]
    elif policy == "augmix":
        for k, lo, hi in (("severity", 1, 10), ("mixture_width", 1, 4), ("chain_depth", -1, 3)):
            out[k] = _aa_int(cfg, k)
            if not lo <= out[k] <= hi or (k == "chain_depth" and out[k] == 0):
                raise ValueError("%s[%r] must lie in [%d, %d]%s, not %r" % (AA_KEY, k, lo, hi, " and not be 0" if k == "chain_depth"
                                                                            else "", cfg.get(k)))
        alpha = cfg.get("alpha", AA_DEFAULTS["alpha"])
        if not _real(alpha) or not 0.0 < float(alpha) <= 16.0:
            raise ValueError("%s['alpha'] must be a finite real number in (0, 16], not %r" % (AA_KEY, alpha))
        out["alpha"] = float(alpha)
        all_ops = cfg.get("all_ops", AA_DEFAULTS["all_ops"])
        if not isinstance(all_ops, (bool, np.bool_)):
            raise ValueError("%s['all_ops'] must be a bool, not %r" % (AA_KEY, all_ops))
        out["all_ops"] = bool(all_ops)
    if policy in ("autoaugment", "augmix") or "interpolation" in cfg:
        interp = cfg.get("interpolation", AA_DEFAULT_INTERPOLATION[policy])
        if interp not in AA_INTERPOLATIONS:
            raise ValueError("%s['interpolation'] must be one of %s, not %r" % (AA_KEY, ", ".join(AA_INTERPOLATIONS), interp))
        out["interpolation"] = interp
    out["seed"] = _aa_int(cfg, "seed") & (2 ** 64 - 1)
    return out


def aa_bilinear(cfg):
    """Whether a validated ``auto_augment`` config resamples its geometric ops bilinearly (torchvision's default per policy)."""
    return cfg.get("interpolation", AA_DEFAULT_INTERPOLATION[cfg["policy"]]) == "bilinear"


def aa_slots(cfg):
    """Op slots per image of a validated ``auto_augment`` config: 1 ("trivial_wide"), ``num_ops`` ("rand"), 2 ("autoaugment") or
    3 per chain ("augmix")."""
    return {"trivial_wide": 1, "autoaugment": 2}.get(cfg["policy"]) or (
        cfg["num_ops"] if cfg["policy"] == "rand" else AA_CHAIN_SLOTS * cfg["mixture_width"])


def auto_augment_rng(cfg, rank):
    """The policy generator of one worker, keyed by (seed, rank, 2): apart from the crop, colour and erasing generators."""
    return np.random.default_rng([cfg["seed"], int(rank), 2])


def auto_augment_space(policy, num_bins, out_hw, all_ops=True):
    """{op name: (magnitudes float64 [num_bins] or None, signed)}: torchvision's ``_AUGMENTATION_SPACE`` of ``TrivialAugmentWide``
    ("trivial_wide"), ``RandAugment`` ("rand"), ``AutoAugment`` ("autoaugment": RandAugment's without Identity, with Invert) or
    ``AugMix`` ("augmix"; its ``_PARTIAL_AUGMENTATION_SPACE`` when not ``all_ops``) for an image of ``out_hw``, in torchvision's
    order, computed as torchvision computes it (fp32 linspace)."""
    import torch
    h, w = out_hw
    lin = lambda hi, lo=0.0: torch.linspace(lo, hi, num_bins).double().numpy()  # noqa: E731
    bits = lambda top, post: (top - (torch.arange(num_bins) / ((num_bins - 1) / post))).round().int().double().numpy()  # noqa: E731
    if policy == "trivial_wide":
        geo, shear, rot, col, post = (lin(32.0), lin(32.0)), lin(0.99), lin(135.0), lin(0.99), bits(8, 6)
    elif policy == "augmix":
        geo, shear, rot, col, post = (lin(w / 3.0), lin(h / 3.0)), lin(0.3), lin(30.0), lin(0.9), bits(4, 4)
    else:
        geo, shear, rot, col, post = (lin(150.0 / 331.0 * w), lin(150.0 / 331.0 * h)), lin(0.3), lin(30.0), lin(0.9), bits(8, 4)
    mags = {"Identity": None, "ShearX": shear, "ShearY": shear, "TranslateX": geo[0], "TranslateY": geo[1], "Rotate": rot,
            "Brightness": col, "Color": col, "Contrast": col, "Sharpness": col, "Posterize": post, "Solarize": lin(0.0, 1.0),
            "AutoContrast": None, "Equalize": None, "Invert": None}
    names = {"autoaugment": AA_OPS[1:] + ("Invert",), "augmix": AA_AUGMIX_OPS if all_ops else AA_AUGMIX_OPS[:AA_AUGMIX_PARTIAL]}
    return {k: (mags[k], k in AA_SIGNED) for k in names.get(policy, AA_OPS)}


def inverse_affine_matrix(center, angle, translate, shear):
    """torchvision's ``_get_inverse_affine_matrix`` (scale 1) in float64, vectorised: arrays of the centre (cx, cy), the angle and the
    translation (tx, ty), and shear (sx, sy), both angles in degrees.  Returns float64 [n, 6]."""
    rot, sx, sy = np.radians(angle), np.radians(shear[0]), np.radians(shear[1])
    (cx, cy), (tx, ty) = center, translate
    a = np.cos(rot - sy) / np.cos(sy)
    b = -np.cos(rot - sy) * np.tan(sx) / np.cos(sy) - np.sin(rot)
    c = np.sin(rot - sy) / np.cos(sy)
    d = -np.sin(rot - sy) * np.tan(sx) / np.cos(sy) + np.cos(rot)
    m = [d, -b, np.zeros_like(a), -c, a, np.zeros_like(a)]
    m[2] = m[2] + m[0] * (-cx - tx) + m[1] * (-cy - ty)
    m[5] = m[5] + m[3] * (-cx - tx) + m[4] * (-cy - ty)
    m[2] = m[2] + cx
    m[5] = m[5] + cy
    return np.stack(m, -1)


def auto_augment_records(n, cfg, rng, out_hw):
    """The per-image op records of one batch: for every image and op slot (one slot for "trivial_wide", ``num_ops`` for "rand") the
    op (uniform over the 14), the magnitude bin (uniform, or ``magnitude`` for "rand") and the sign (negative with p = ½, signed ops
    only), drawn for the whole batch at once whatever the op.  Each record is composed in float64 as torchvision's op computes its
    parameters and rounded once: op id; the scalar (factor 1 + m, Solarize's threshold 255·m, or Posterize's bits); 1 − factor for
    the blends; the fp32 inverse affine matrix of ShearX / ShearY (shear degrees(atan m) about (0, 0)), TranslateX / TranslateY
    (int(m) pixels) and Rotate (about the centre).

    "autoaugment" draws a sub-policy of :data:`AA_IMAGENET_POLICY` per image (uniform over the 25); each of its two ops applies iff
    U ≤ p (torchvision's ``torch.rand(()) <= probability``) and is an Identity record otherwise; signed ops are negated with p = ½.
    "augmix" is :func:`augmix_records`, whose weights this function drops.  Geometric records of a bilinear config carry 1 in
    field 3.

    Returns (records float32 [n, slots, 12], op int64 [n, slots], magnitude float64 [n, slots], the signed magnitude each op uses)."""
    if cfg["policy"] == "augmix":
        rec, _, op, mag = augmix_records(n, cfg, rng, out_hw)
        return rec, op, mag
    if cfg["policy"] == "autoaugment":
        space = auto_augment_space("autoaugment", AA_BINS, out_hw)
        names = [[AA_OP_IDS[o] for o, _, _ in sub] for sub in AA_IMAGENET_POLICY]
        prob = np.array([[p for _, p, _ in sub] for sub in AA_IMAGENET_POLICY])
        mags = np.array([[space[o][0][b] if b is not None else 0.0 for o, _, b in sub] for sub in AA_IMAGENET_POLICY])
        signed = np.array([[space[o][1] for o, _, _ in sub] for sub in AA_IMAGENET_POLICY])
        sub = rng.integers(0, len(AA_IMAGENET_POLICY), n)
        applies = rng.random((n, 2)) <= prob[sub]
        neg = rng.random((n, 2)) <= 0.5
        op = np.where(applies, np.array(names)[sub], 0)
        mag = np.where(applies, np.where(signed[sub] & neg, -mags[sub], mags[sub]), 0.0)
        return aa_compose_records(op, mag, out_hw, aa_bilinear(cfg)), op, mag
    space = auto_augment_space(cfg["policy"], cfg["num_magnitude_bins"], out_hw)
    slots = 1 if cfg["policy"] == "trivial_wide" else cfg["num_ops"]
    op = rng.integers(0, len(AA_OPS), (n, slots))
    if cfg["policy"] == "trivial_wide":
        bins = rng.integers(0, cfg["num_magnitude_bins"], (n, slots))
    else:
        bins = np.full((n, slots), cfg["magnitude"])
    neg = rng.random((n, slots)) <= 0.5
    table = np.stack([space[k][0] if space[k][0] is not None else np.zeros(cfg["num_magnitude_bins"]) for k in AA_OPS])
    signed = np.array([space[k][1] for k in AA_OPS])
    mag = table[op, bins]
    mag = np.where(signed[op] & neg, -mag, mag)
    return aa_compose_records(op, mag, out_hw, aa_bilinear(cfg)), op, mag


def augmix_records(n, cfg, rng, out_hw):
    """The AugMix draw of one batch ("augmix" configs), all at once: per image m = Dirichlet(α, α) and d = Dirichlet(α·1_width);
    per chain a depth (``chain_depth``, or uniform over {1, 2, 3} for −1); per chain step an op uniform over the space
    (:func:`auto_augment_space`, 13 or 9 ops), a magnitude bin uniform over [0, severity) and a sign (negative with p = ½, signed ops
    only).  Chain i's steps are slots 3i … 3i + 2; a step past its chain's depth is :data:`AA_NONE`.  The weights are computed in fp32
    as torchvision's ``AugMix.forward`` computes them: m₀ = fl32(m₀) and w_i = fl32(d_i)·fl32(m₁).

    Returns (records float32 [n, 3·width, 12], weights float32 [n, 1 + width] = (m₀, w_0 … w_{width−1}), op int64 [n, 3·width],
    magnitude float64 [n, 3·width])."""
    width, alpha = cfg["mixture_width"], cfg["alpha"]
    space = auto_augment_space("augmix", AA_BINS, out_hw, cfg["all_ops"])
    names = list(space)
    m = rng.dirichlet([alpha, alpha], n).astype(np.float32)
    d = rng.dirichlet([alpha] * width, n).astype(np.float32)
    if cfg["chain_depth"] > 0:
        depth = np.full((n, width), cfg["chain_depth"])
    else:
        depth = rng.integers(1, AA_CHAIN_SLOTS + 1, (n, width))
    k = rng.integers(0, len(names), (n, width, AA_CHAIN_SLOTS))
    bins = rng.integers(0, cfg["severity"], (n, width, AA_CHAIN_SLOTS))
    neg = rng.random((n, width, AA_CHAIN_SLOTS)) <= 0.5
    table = np.stack([space[o][0] if space[o][0] is not None else np.zeros(AA_BINS) for o in names])
    signed = np.array([space[o][1] for o in names])
    live = np.arange(AA_CHAIN_SLOTS) < depth[..., None]
    op = np.where(live, np.array([AA_OP_IDS[o] for o in names])[k], AA_NONE).reshape(n, -1)
    mag = np.where(live, np.where(signed[k] & neg, -table[k, bins], table[k, bins]), 0.0).reshape(n, -1)
    weights = np.concatenate([m[:, :1], d * m[:, 1:]], 1)
    return aa_compose_records(op, mag, out_hw, aa_bilinear(cfg)), weights, op, mag


def aa_compose_records(op, mag, out_hw, bilinear=False):
    """The float32 [..., 12] records of op ids ``op`` at signed magnitudes ``mag`` (see :func:`auto_augment_records`), composed in
    float64 and rounded once; field 3 is 1 for a geometric op when ``bilinear``."""
    h, w = out_hw
    rec = np.zeros(op.shape + (AA_RECORD_FLOATS,), np.float64)
    rec[..., 0] = op
    factor = 1.0 + mag
    blend = (op >= 6) & (op <= 9)
    rec[..., 1] = np.where(blend, factor, np.where(op == 10, np.trunc(mag), np.where(op == 11, 255.0 * mag, 0.0)))
    rec[..., 2] = np.where(blend, 1.0 - factor, 0.0)
    deg = np.degrees(np.arctan(mag))
    centre = (np.where(op <= 2, -0.5 * w, 0.0), np.where(op <= 2, -0.5 * h, 0.0))
    mats = inverse_affine_matrix(centre, np.where(op == 5, -mag, 0.0),
                                 (np.where(op == 3, np.trunc(mag), 0.0), np.where(op == 4, np.trunc(mag), 0.0)),
                                 (np.where(op == 1, deg, 0.0), np.where(op == 2, deg, 0.0)))
    geo = (op >= 1) & (op <= 5)
    rec[..., 3] = np.where(geo & bool(bilinear), 1.0, 0.0)
    rec[..., 4:10] = np.where(geo[..., None], mats, 0.0)
    return rec.astype(np.float32)


VC_KEY = "val_crops"


def check_val_crops(v):
    """The validated ``config['val_crops']``: the int 1 (one centre crop, the default), 2 (the centre crop and its mirror) or 10 (the
    four corners and the centre, each with its mirror); a bool, a float, a string or any other int is a ValueError that names the
    key."""
    from ...ops.reference import MULTI_CROP_VIEWS
    if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or int(v) not in MULTI_CROP_VIEWS:
        raise ValueError("%s must be one of the ints %s, not %r" % (VC_KEY, ", ".join(map(str, MULTI_CROP_VIEWS)), v))
    return int(v)


RE_KEY = "random_erasing"
RE_DEFAULTS = {"p": 0.5, "scale": (0.02, 0.33), "ratio": (0.3, 3.3), "seed": 0}
RE_ATTEMPTS = 10


def check_random_erasing(cfg):
    """The validated ``config['random_erasing']`` with every key filled in (``p`` a float in [0, 1], ``scale`` and ``ratio`` float pairs
    checked as :func:`check_resized_crop` checks them, an int seed), or None for None; anything else is a ValueError that names the
    key.  There is no ``value`` key: the box is set to 0 in the normalised output, torchvision's ``RandomErasing(value=0)``."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError("%s must be a dict or None, not %r" % (RE_KEY, cfg))
    unknown = sorted(str(k) for k in cfg if k not in RE_DEFAULTS)
    if unknown:
        raise ValueError("%s: unknown key %r; the keys are %s" % (RE_KEY, unknown[0], ", ".join(RE_DEFAULTS)))
    p = cfg.get("p", RE_DEFAULTS["p"])
    if not _real(p):
        raise ValueError("%s['p'] must be a finite real number, not %r" % (RE_KEY, p))
    if not 0.0 <= float(p) <= 1.0:
        raise ValueError("%s['p'] must lie in [0, 1], not %r" % (RE_KEY, p))
    out = {"p": float(p)}
    for k in ("scale", "ratio"):
        v = cfg.get(k, RE_DEFAULTS[k])
        if not (isinstance(v, (list, tuple)) and len(v) == 2 and all(_real(e) for e in v)):
            raise ValueError("%s[%r] must be two finite real numbers [lo, hi], not %r" % (RE_KEY, k, v))
        lo, hi = float(v[0]), float(v[1])
        if not (0.0 < lo <= hi and (k == "ratio" or hi <= 1.0)):
            raise ValueError("%s[%r] must satisfy %s, not %r" % (RE_KEY, k, "0 < lo <= hi <= 1" if k == "scale" else "0 < lo <= hi", v))
        out[k] = (lo, hi)
    seed = cfg.get("seed", 0)
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise ValueError("%s['seed'] must be an int, not %r" % (RE_KEY, seed))
    out["seed"] = int(seed) & (2 ** 64 - 1)
    return out


def random_erasing_rng(cfg, rank):
    """The erase-box generator of one worker, keyed by (seed, rank, 3): apart from the crop and colour generators, so turning the key
    on or off changes neither the boxes, nor the fixed crops, nor the colour records drawn."""
    return np.random.default_rng([cfg["seed"], int(rank), 3])


def draw_erase_boxes(n, out_hw, cfg, rng):
    """Per-image erase boxes (i, j, h, w) (int32 [n, 4]) in output coordinates, drawn as torchvision's ``RandomErasing``: the image
    is erased when U < p; then up to 10 attempts of area H·W·U(scale) and ratio exp(U(log ratio)), h = round(√(area·r)),
    w = round(√(area / r)) (round half to even), and the first attempt with h < H and w < W sits at a uniform position.  An image that
    is not erased, or has no fitting attempt, gets (0, 0, 0, 0).  Every image draws the same count of numbers whatever p, all of the
    batch at once."""
    H, W = out_hw
    lr = np.log(cfg["ratio"])
    u = rng.random(n)
    area = (H * W) * rng.uniform(cfg["scale"][0], cfg["scale"][1], (n, RE_ATTEMPTS))
    r = np.exp(rng.uniform(lr[0], lr[1], (n, RE_ATTEMPTS)))
    h = np.rint(np.sqrt(area * r)).astype(np.int64)
    w = np.rint(np.sqrt(area / r)).astype(np.int64)
    fits = (h < H) & (w < W)
    first = np.argmax(fits, axis=1)
    ok = fits[np.arange(n), first] & (u < cfg["p"])
    h = np.where(ok, h[np.arange(n), first], 0)
    w = np.where(ok, w[np.arange(n), first], 0)
    i = np.where(ok, rng.integers(0, H - h + 1), 0)
    j = np.where(ok, rng.integers(0, W - w + 1), 0)
    return np.stack([i, j, h, w], 1).astype(np.int32)


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
