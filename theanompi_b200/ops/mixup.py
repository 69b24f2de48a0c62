"""Mixup and CutMix (``config['mixup']``): the record of one step's draw, the validation of the config dict, and the buffer that
holds the record on the training device.

The layout of :data:`RECORD` is ``csrc/api.h: MixRecord``, byte for byte; nothing else hard-codes its offsets.  On CUDA the record is
written by ``mix_draw_kernel`` inside the captured step, keyed by the device step counter, and read there by ``mix_batch_kernel`` and
``softmax_xent_mix_kernel``.  On the CPU :func:`reference.mix_draw` computes the same draw and the record is a host tensor of the
same 64 bytes.
"""
from __future__ import annotations

import math

import numpy as np
import torch

MIX_NONE, MIX_MIXUP, MIX_CUTMIX = 0, 1, 2
RECORD = np.dtype([("mode", "<i4"), ("lam", "<f4"), ("lam_raw", "<f8"), ("cy", "<i4"), ("cx", "<i4"), ("y0", "<i4"), ("y1", "<i4"),
                   ("x0", "<i4"), ("x1", "<i4"), ("H", "<i4"), ("W", "<i4"), ("pad", "<i4", (4,))])
assert RECORD.itemsize == 64
RECORD_BYTES = RECORD.itemsize

KEYS = ("alpha", "cutmix_alpha", "switch_prob", "prob", "seed")
DEFAULTS = {"alpha": 0.0, "cutmix_alpha": 0.0, "switch_prob": 0.5, "prob": 1.0, "seed": 0}
MAX_ALPHA = 16.0          # the range the Gamma sampler is tested over


def check_config(cfg):
    """The validated ``config['mixup']`` with every key filled in, or None for None; anything else is a ValueError that names the
    offending key."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError("mixup must be a dict or None, not %r" % (cfg,))
    unknown = sorted(str(k) for k in cfg if k not in KEYS)
    if unknown:
        raise ValueError("mixup: unknown key %r; the keys are %s" % (unknown[0], ", ".join(KEYS)))
    out = dict(DEFAULTS)
    for k in ("alpha", "cutmix_alpha", "switch_prob", "prob"):
        v = cfg.get(k, DEFAULTS[k])
        if isinstance(v, bool) or not isinstance(v, (int, float, np.integer, np.floating)) or not math.isfinite(v):
            raise ValueError("mixup[%r] must be a finite real number, not %r" % (k, v))
        out[k] = float(v)
    for k in ("alpha", "cutmix_alpha"):
        if not 0.0 <= out[k] <= MAX_ALPHA:
            raise ValueError("mixup[%r] must be in [0, %g], not %r" % (k, MAX_ALPHA, out[k]))
    if out["alpha"] == 0.0 and out["cutmix_alpha"] == 0.0:
        raise ValueError("mixup['alpha'] and mixup['cutmix_alpha'] are both 0: set one of them > 0, or mixup = None")
    for k in ("switch_prob", "prob"):
        if not 0.0 <= out[k] <= 1.0:
            raise ValueError("mixup[%r] must be a probability in [0, 1], not %r" % (k, out[k]))
    seed = cfg.get("seed", 0)
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)):
        raise ValueError("mixup['seed'] must be an int, not %r" % (seed,))
    out["seed"] = int(seed) & (2 ** 64 - 1)
    return out


def decode(rec):
    """The record(s) of a 64·n-byte uint8 tensor (any device) or of a :data:`RECORD` array, as a numpy structured array (one
    record: a 0-d one, whose fields read as scalars)."""
    if isinstance(rec, (np.ndarray, np.void)) and rec.dtype == RECORD:
        return rec
    buf = rec.detach().cpu().contiguous().numpy().tobytes()
    arr = np.frombuffer(buf, dtype=RECORD)
    return arr[0] if arr.shape[0] == 1 else arr


def encode(arr):
    """A :data:`RECORD` array (or one record) as a uint8 host tensor."""
    return torch.from_numpy(np.ascontiguousarray(np.asarray(arr, dtype=RECORD).reshape(-1)).view(np.uint8).copy())


class Mixer(object):
    """One model's Mixup / CutMix: the validated config, the worker's rank, the image size (H, W) of the mix point, and the record
    buffer of the training step.  :meth:`draw` is the step's first mixing launch; it returns the record the mix and the loss read."""

    def __init__(self, cfg, rank, hw, device):
        self.cfg = check_config(cfg)
        self.rank = int(rank)
        self.H, self.W = (int(v) for v in hw)
        self.device = torch.device(device)
        self.rec = torch.zeros(RECORD_BYTES, dtype=torch.uint8, device=self.device)

    def draw(self):
        """The draw of this step into :attr:`rec`: on CUDA one single-thread launch that reads the device step counter (so every
        replay of a captured step draws anew), on the CPU :func:`reference.mix_draw` at the host step counter."""
        from .functional import mix_draw
        return mix_draw(self.cfg, self.rank, (self.H, self.W), self.rec)
