"""Bit identity of the five flat arena optimizers: five steps on a seeded multi-group arena, in bf16 with a shadow and in tf32
without, must reproduce the SHA-256 digests of W, U, the extra flat buffers and H stored in ``golden/flat_update_sm90a.json``.

The arena has weight decay, a bias lr multiplier, tensors whose sizes are not multiples of the 1024-element block, a
non-exchanged (batch-norm gamma) group and more blocks than the kernels' grid, so the block loop runs more than once.  The flat
kernels have no atomics, so the digests do not depend on the grid size.

    python tests/test_gpu_flat_update.py OUT.json      # (re)write the digests
"""
import hashlib
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "flat_update_sm90a.json")
STEPS = 5


def _sgd(mu, nesterov, use_momentum=True, k=1, **kw):
    def make(a):
        from theanompi_b200.utils.opt import FlatSGD
        o = FlatSGD(a, mu, nesterov, use_momentum)
        return o, lambda: o.step(0.01, k, **kw)
    return make


def _opt(cls_name, **kw):
    def make(a):
        from theanompi_b200.utils import opt
        o = getattr(opt, cls_name)(a, **kw)
        return o, o.step
    return make


# name -> (lr, optimizer factory)
CONFIGS = {
    "sgd_momentum": (0.01, _sgd(0.9, False)),
    "sgd_nesterov": (0.01, _sgd(0.9, True)),
    "sgd_no_momentum": (0.01, _sgd(0.9, False, use_momentum=False)),
    "sgd_inv_k_0.5": (0.01, _sgd(0.9, False, k=2)),
    "sgd_only_local": (0.01, _sgd(0.9, False, only_local=True)),
    "sgd_only_exchanged": (0.01, _sgd(0.9, False, only_exchanged=True)),
    "rmsprop": (1e-3, _opt("FlatRMSProp")),
    "rmsprop_clip": (1e-3, _opt("FlatRMSProp", clip=0.05)),
    "adam": (1e-3, _opt("FlatAdam")),
    "adadelta": (1.0, _opt("FlatAdadelta")),
    "rmsprop_centered": (1e-3, _opt("FlatCenteredRMSProp")),
}


def _arena(shadow):
    from theanompi_b200.parallel.arena import FlatArena
    g = torch.Generator().manual_seed(2024)
    shapes = [("W", (300, 70)), ("b", (300,)), ("gamma", (96,)), ("W", (64, 3, 3, 16)), ("b", (17,)), ("W", (1100, 1024))]
    params = []
    for name, shape in shapes:
        p = torch.nn.Parameter(torch.randn(*shape, generator=g) * 0.05)
        p.pname = name
        params.append(p)
    wt = ["W" if n == "W" else "b" for n, _ in shapes]
    return FlatArena(params, wt, "cuda:0", weight_decay=5e-4, shadow=shadow), g


def _sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def digests(prec, name):
    lr, make = CONFIGS[name]
    a, g = _arena(prec == "bf16")
    a.hyper[0] = lr
    opt, step = make(a)
    for _ in range(STEPS):
        a.G.copy_((torch.randn(a.numel, generator=g) * 0.1).cuda())
        step()
    torch.cuda.synchronize()
    out = {"W": _sha(a.W), "U": _sha(a.U)}
    for buf in ("V", "R", "S"):
        if isinstance(getattr(opt, buf, None), torch.Tensor):
            out[buf] = _sha(getattr(opt, buf))
    if a.H is not None:
        out["H"] = _sha(a.H)
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("prec", ["bf16", "tf32"])
@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_flat_update_bits(prec, name):
    with open(GOLDEN) as f:
        want = json.load(f)["%s/%s" % (prec, name)]
    assert digests(prec, name) == want


if __name__ == "__main__":
    res = {"%s/%s" % (p, n): digests(p, n) for p in ("bf16", "tf32") for n in sorted(CONFIGS)}
    with open(sys.argv[1], "w") as f:
        json.dump(res, f, indent=1, sort_keys=True)
