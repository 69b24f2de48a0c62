"""CIFAR augmentation (``config['cifar_augment']``): fb.resnet.torch's zero-padded ``RandomCrop(32, pad)`` and horizontal flip, then
DeVries & Taylor's Cutout, drawn per image on the device inside the captured training step.  This module owns the validated config,
the Philox counter tag, the layout of one step's three buffers and the buffers themselves.

Image n of a step (B images of SIZE × SIZE) draws oy, ox ∈ [0, 2·pad], a flip and a Cutout centre (cy, cx) ∈ [0, SIZE)².  Philox4x32-10,
key (seed_lo, seed_hi ^ rank); block 0 has counter (n, TAG, step_lo, step_hi), block 1 (n, TAG + 1, step_lo, step_hi).  Each value is
⌊w·k / 2^32⌋: oy and ox are block 0 words 0 and 1 with k = 2·pad + 1, the flip is word 2 >> 31, cy word 3 and cx block 1 word 0 with
k = SIZE.  The buffers:

- ``offs``  int32 [B, 2]: (oy − pad, ox − pad), the crop offsets of the zero-filled ``crop_mirror_normalize``;
- ``flips`` uint8 [B]:    1 where the crop is mirrored;
- ``boxes`` int32 [B, 4]: the Cutout box (y1, x1, y2 − y1, x2 − x1) of ``random_erase``, y1 = clamp(cy − L//2, 0, SIZE),
  y2 = clamp(cy + L//2, 0, SIZE) and the same for x (an odd L cuts an (L − 1)-wide hole, as DeVries & Taylor's code does).

On CUDA ``cifar_augment_draw_kernel`` (``csrc/nn_kernels.cu``) writes them from the device step counter; on the CPU
:func:`reference.cifar_augment_draw` computes the same values bit for bit.
"""
from __future__ import annotations

import numpy as np
import torch

KEY = "cifar_augment"
KEYS = ("pad", "cutout", "seed")
DEFAULTS = {"pad": 4, "cutout": 0, "seed": 0}
SIZE = 32                  # CIFAR image side: the crop is SIZE × SIZE and the Cutout centre ranges over it
TAG = 0xA0000000           # second Philox counter word of block 0; block 1 uses TAG + 1 (csrc/nn_kernels.cu: kCifarAugTag)
RANGES = {"pad": (0, SIZE - 1), "cutout": (0, SIZE)}


def check_config(cfg):
    """The validated ``config['cifar_augment']`` with every key filled in, or None for None; a non-dict, an unknown key, a bool, a
    non-integer or an out-of-range value is a ValueError that names the key."""
    if cfg is None:
        return None
    if not isinstance(cfg, dict):
        raise ValueError("%s must be a dict or None, not %r" % (KEY, cfg))
    unknown = sorted(str(k) for k in cfg if k not in KEYS)
    if unknown:
        raise ValueError("%s: unknown key %r; the keys are %s" % (KEY, unknown[0], ", ".join(KEYS)))
    out = dict(DEFAULTS)
    for k in KEYS:
        v = cfg.get(k, DEFAULTS[k])
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError("%s[%r] must be an int, not %r" % (KEY, k, v))
        v = int(v)
        if k in RANGES and not RANGES[k][0] <= v <= RANGES[k][1]:
            raise ValueError("%s[%r] must be in [%d, %d], not %r" % (KEY, k, RANGES[k][0], RANGES[k][1], v))
        out[k] = v
    out["seed"] &= 2 ** 64 - 1
    return out


def cutout_boxes(cy, cx, L):
    """DeVries & Taylor's Cutout hole of side ``L`` centred on (cy, cx) (int arrays), as int32 [..., 4] boxes (y1, x1, y2 − y1, x2 − x1):
    y1 = clamp(cy − L//2, 0, SIZE), y2 = clamp(cy + L//2, 0, SIZE), the same for x."""
    cy, cx = np.asarray(cy, dtype=np.int64), np.asarray(cx, dtype=np.int64)
    y1, y2 = np.clip(cy - L // 2, 0, SIZE), np.clip(cy + L // 2, 0, SIZE)
    x1, x2 = np.clip(cx - L // 2, 0, SIZE), np.clip(cx + L // 2, 0, SIZE)
    return np.stack([y1, x1, y2 - y1, x2 - x1], axis=-1).astype(np.int32)


class CifarAugment(object):
    """One model's CIFAR augmentation: the validated config, the worker's rank and the three buffers of the training step's
    B images.  :meth:`draw` is one launch per training step."""

    def __init__(self, cfg, rank, B, device):
        self.cfg = check_config(cfg)
        self.rank, self.B = int(rank), int(B)
        self.device = torch.device(device)
        self.offs = torch.zeros((self.B, 2), dtype=torch.int32, device=self.device)
        self.flips = torch.zeros((self.B,), dtype=torch.uint8, device=self.device)
        self.boxes = torch.zeros((self.B, 4), dtype=torch.int32, device=self.device)

    @property
    def cutout(self):
        return self.cfg["cutout"] > 0

    def draw(self):
        """This step's offsets, flips and boxes into the buffers: on CUDA one launch that reads the device step counter (so every
        replay of a captured step draws anew), on the CPU :func:`reference.cifar_augment_draw` at the host step counter."""
        from .functional import cifar_augment_draw
        return cifar_augment_draw(self)
