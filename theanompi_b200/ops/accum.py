"""Gradient-accumulation switch of the backward pass.

A model that accumulates the gradient of n micro-batches before one optimizer step (``config['grad_accum'] = n``, see
:class:`theanompi_b200.models.base.ModelBase`) sets this switch around the forward + backward of every micro-step:

* ``accumulate``: the parameter-gradient kernels add into the arena's G views instead of overwriting them (the ``mid`` and
  ``last`` micro-steps of a window; the ``first`` one stores, so G needs no clearing);
* ``grad_scale``: the factor 1/n of the softmax / NLL gradient (every Softmax head of the step), applied in fp32 inside the kernel's
  dlogits scale, so that G holds the mean gradient over the n micro-batches after the last one.  The reported loss is unscaled.

The switch is read on the host when the kernels are launched, so a CUDA graph captured under it keeps the mode it was captured
with: a model captures one graph per micro-step kind.
"""
from __future__ import annotations

import contextlib

_STATE = {"accumulate": False, "grad_scale": 1.0}


def accumulating():
    """True while the backward kernels add into the parameter gradients."""
    return _STATE["accumulate"]


def grad_scale():
    """The factor of the softmax / NLL gradient (1/n during a window of n micro-batches, else 1)."""
    return _STATE["grad_scale"]


@contextlib.contextmanager
def mode(accumulate, grad_scale=1.0):
    """Run the enclosed forward + backward with parameter gradients added into G (``accumulate``) and the loss gradient scaled by
    ``grad_scale``; restores the previous mode on exit."""
    old = dict(_STATE)
    _STATE["accumulate"], _STATE["grad_scale"] = bool(accumulate), float(grad_scale)
    try:
        yield
    finally:
        _STATE.update(old)
