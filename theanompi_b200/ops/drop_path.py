"""Stochastic depth (``config['drop_path_rate']``, Huang et al. 2016, as timm's ``drop_path`` with ``scale_by_keep=True``): the
per-block drop probabilities, the layout of one training step's drop table, and the buffers that hold it on the training device.

Blocks are numbered l = 0 … L − 1 in forward order; block l drops with p_l = p·l / (L − 1) (0 when L = 1), the linear rule of
``torch.linspace(0, p, L)``.  The table of a step is fp32 ``[L, B]``: entry (l, n) is 0 when block l drops sample n, else
fp32(1 / (1 − p_l)), computed in fp64 and rounded once.  Row l (``table[l]``, B contiguous floats) is what block l's residual merge
reads.  Sample n of block l drops when u = (w >> 8)·2^-24 < p_l, w the first word of Philox4x32-10 with key (seed_lo, seed_hi ^ rank)
and counter (n, l ^ :data:`TAG`, step_lo, step_hi); the comparison is done exactly as (w >> 8) < ⌈p_l·2^24⌉.  On CUDA the table is
written by ``drop_path_draw_kernel`` (``csrc/nn_kernels.cu``) from the device step counter inside the captured step; on the CPU
:func:`reference.drop_path_draw` computes the same table bit for bit.  Nothing else hard-codes this layout or the p_l rule.
"""
from __future__ import annotations

import math

import numpy as np
import torch

KEY = "drop_path_rate"
TAG = 0xC0000000           # second Philox counter word is l ^ TAG (csrc/nn_kernels.cu: kDropPathTag)
MAX_BLOCKS = 65535         # l ^ TAG stays in [0xC0000000, 0xC000FFFF]


def check_rate(p):
    """``config['drop_path_rate']`` as a float in [0, 1); anything else (a bool, NaN, a string, a negative value, 1.0) is a
    ValueError that names the key."""
    ok = not isinstance(p, bool) and isinstance(p, (int, float, np.integer, np.floating))
    if not (ok and math.isfinite(p) and 0.0 <= p < 1.0):
        raise ValueError("%s must be a real number in [0, 1), not %r" % (KEY, p))
    return float(p)


def block_rates(p, L):
    """p_l = p·l / (L − 1) for l < L in fp64 (all 0 when L = 1)."""
    if not 1 <= int(L) <= MAX_BLOCKS:
        raise ValueError("drop-path needs 1 <= L <= %d residual blocks, not %r" % (MAX_BLOCKS, L))
    L = int(L)
    if L == 1:
        return np.zeros(1, dtype=np.float64)
    return float(p) * np.arange(L, dtype=np.float64) / float(L - 1)


def thresholds(rates):
    """⌈p_l·2^24⌉ per block (int64): the sample drops when (w >> 8) is below it.  p_l·2^24 is exact in fp64."""
    return np.ceil(np.asarray(rates, dtype=np.float64) * 16777216.0).astype(np.int64)


def keep_scales(rates):
    """fp32(1 / (1 − p_l)) per block, the scale of a kept sample, computed in fp64 and rounded once."""
    return (1.0 / (1.0 - np.asarray(rates, dtype=np.float64))).astype(np.float32)


class DropPath(object):
    """One model's drop-path: the block rates, the per-block threshold and keep-scale buffers the draw kernel reads, and the
    ``[L, B]`` table of the training step.  :meth:`draw` is one launch per training step; :meth:`row` is block l's row of it, or
    None where p_l = 0 (such a block runs the kernels without a row)."""

    def __init__(self, p, L, B, rank, device):
        self.p = check_rate(p)
        self.rates = block_rates(self.p, L)
        self.L, self.B, self.rank = int(L), int(B), int(rank)
        self.device = torch.device(device)
        self.thresh = torch.from_numpy(thresholds(self.rates).astype(np.int32)).to(self.device)
        self.keep = torch.from_numpy(keep_scales(self.rates)).to(self.device)
        self.table = torch.ones((self.L, self.B), dtype=torch.float32, device=self.device)

    def draw(self):
        """This step's table into :attr:`table`: on CUDA one launch that reads the device step counter (so every replay of a
        captured step draws anew), on the CPU :func:`reference.drop_path_draw` at the host step counter."""
        from .functional import drop_path_draw
        return drop_path_draw(self, self.table)

    def row(self, l):
        return None if self.rates[l] == 0.0 else self.table[l]
