"""Independent oracle for auto_augment: torchvision's own TrivialAugmentWide / RandAugment op code
(``_AutoAugmentBase._apply_image_or_video_transform``, nearest interpolation, fill 0) applied with the drawn magnitudes, and the tie rule
the kernels are held to.  Needs torchvision, which is not a dependency of the package."""
import numpy as np
import pytest
import torch


def torchvision_op(img, name, magnitude):
    """torchvision's op ``name`` with signed ``magnitude`` on a uint8 CHW image."""
    A = pytest.importorskip("torchvision.transforms.v2._auto_augment")
    from torchvision import tv_tensors
    from torchvision.transforms import InterpolationMode
    fill = {torch.Tensor: None, tv_tensors.Image: None}
    return A.TrivialAugmentWide()._apply_image_or_video_transform(img, name, float(magnitude), interpolation=InterpolationMode.NEAREST,
                                                                 fill=fill)


def torchvision_space(policy, num_bins, out_hw):
    """{name: (magnitudes float64 or None, signed)} from torchvision's ``_AUGMENTATION_SPACE``."""
    A = pytest.importorskip("torchvision.transforms.v2._auto_augment")
    cls = A.TrivialAugmentWide if policy == "trivial_wide" else A.RandAugment
    out = {}
    for k, (fn, signed) in cls._AUGMENTATION_SPACE.items():
        m = fn(num_bins, out_hw[0], out_hw[1])
        out[k] = (None if m is None else m.double().numpy(), signed)
    return out


def assert_tie_rule(got, want, what, level=1, limit=1e-3):
    """The tie rule: equal except at elements whose float64 value lies next to a rounding, truncation or nearest-index boundary,
    where the fp32 evaluation may land one level (or, for a nearest-index tie, one neighbour) away.  Such elements must be fewer than
    ``limit`` of the total, and a value op may miss by at most ``level`` (None: a geometric op, where the neighbour's value is
    arbitrary), so a wrong formula cannot hide behind the rule."""
    got, want = np.asarray(got).astype(np.int64), np.asarray(want).astype(np.int64)
    diff = got != want
    assert diff.mean() < limit, "%s: %d of %d elements differ" % (what, diff.sum(), diff.size)
    if level is not None and diff.any():
        assert np.abs(got - want).max() <= level, "%s: a difference of %d levels" % (what, np.abs(got - want).max())
