"""Independent oracle for the "autoaugment" and "augmix" policies: torchvision's own ``AutoAugment.forward`` and ``AugMix.forward``
(torchvision.transforms.v2) run on one uint8 CHW image with their random draws replaced by a given draw.  ``torch.randint``,
``torch.rand``, ``_get_random_item`` and ``_sample_dirichlet`` are patched inside ``torchvision.transforms.v2._auto_augment`` only, so
the ops themselves run as torchvision runs them.  Needs torchvision, which is not a dependency of the package."""
import contextlib
import types

import pytest
import torch


def _module():
    return pytest.importorskip("torchvision.transforms.v2._auto_augment")


@contextlib.contextmanager
def _replay(randint=(), rand=(), items=(), dirichlet=()):
    """Inside the block, torchvision's auto-augment module draws the given values in order: ``randint`` ints, ``rand`` floats,
    ``items`` op names and ``dirichlet`` fp32 rows.  Every queue must be used up."""
    A = _module()
    queues = {"randint": list(randint), "rand": list(rand), "items": list(items), "dirichlet": list(dirichlet)}

    def pop(k):
        assert queues[k], "torchvision drew more %s values than the record holds" % k
        return queues[k].pop(0)

    def randint(*args, size=None, **kw):
        v = pop("randint")
        return torch.tensor(v if size is None or size == () else [v] * int(torch.Size(size).numel()), dtype=torch.int64)

    class _Torch(types.SimpleNamespace):                        # torch, with the two draws replaced
        def __getattr__(self, k):
            return getattr(torch, k)

    proxy = _Torch(randint=randint, rand=lambda *a, **kw: torch.tensor(float(pop("rand"))))
    saved = A.torch, A._AutoAugmentBase._get_random_item, A.AugMix._sample_dirichlet
    A.torch = proxy
    A._AutoAugmentBase._get_random_item = lambda self, dct: (lambda k: (k, dct[k]))(pop("items"))
    A.AugMix._sample_dirichlet = lambda self, params: torch.as_tensor(pop("dirichlet"), dtype=torch.float32).reshape(1, -1)
    try:
        yield
    finally:
        A.torch, A._AutoAugmentBase._get_random_item, A.AugMix._sample_dirichlet = saved
    assert not any(queues.values()), "torchvision drew fewer values than the record holds: %r" % queues


def interpolation(name):
    from torchvision.transforms import InterpolationMode
    return {"nearest": InterpolationMode.NEAREST, "bilinear": InterpolationMode.BILINEAR}[name]


def autoaugment(img, sub, apply_u, sign_u, interp="nearest"):
    """torchvision's ``AutoAugment(IMAGENET)`` on ``img`` with sub-policy ``sub``, the two application uniforms ``apply_u`` and the
    two sign uniforms ``sign_u`` (each used only where torchvision draws it: a sign for an applied, signed op with a magnitude)."""
    A = _module()
    t = A.AutoAugment(interpolation=interpolation(interp))
    rand = []
    for j, (name, p, b) in enumerate(t._policies[sub]):
        rand.append(float(apply_u[j]))
        if apply_u[j] <= p and b is not None and t._AUGMENTATION_SPACE[name][1]:
            rand.append(float(sign_u[j]))
    with _replay(randint=[int(sub)], rand=rand):
        return t(img)


def augmix(img, m, d, depths, names, bins, sign_u, severity=3, chain_depth=-1, all_ops=True, interp="bilinear"):
    """torchvision's ``AugMix`` on ``img`` with the Dirichlet rows ``m`` (2) and ``d`` (width), the chain depths, and per chain step
    the op name, the magnitude bin and the sign uniform (``names``, ``bins``, ``sign_u``: [width][3], steps past the depth unused)."""
    A = _module()
    width = len(d)
    t = A.AugMix(severity=severity, mixture_width=width, chain_depth=chain_depth, all_ops=all_ops, interpolation=interpolation(interp))
    space = t._AUGMENTATION_SPACE if all_ops else t._PARTIAL_AUGMENTATION_SPACE
    randint, rand, items = [], [], []
    for i in range(width):
        if chain_depth <= 0:
            randint.append(int(depths[i]))
        for s in range(int(depths[i])):
            items.append(names[i][s])
            fn, signed = space[names[i][s]]
            if fn(10, 1, 1) is not None:
                randint.append(int(bins[i][s]))
                if signed:
                    rand.append(float(sign_u[i][s]))
    with _replay(randint=randint, rand=rand, items=items, dirichlet=[m, d]):
        return t(img)
