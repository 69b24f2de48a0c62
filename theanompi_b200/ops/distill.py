"""Knowledge distillation of the native ImageNet classifiers (``config['distill']``, a dict; None = off): the student trains against a
frozen teacher's softened predictions on exactly the batch it sees (Hinton et al. 2015; Beyer et al. 2022, "a good teacher is patient and
consistent").  Every training step, after the step's draws and the in-place Mixup / CutMix, the teacher runs an eval-mode forward on the
student's x_in inside the same captured step, and the loss becomes

    L = (1 − α)·CE_q(z) + α·T²·KL(softmax(t/T) ‖ softmax(z/T))

per row, averaged over the batch: z the student's main-head logits, t the teacher's, q the hard target the step would use without the key
(one-hot, label-smoothed or mixed; the teacher's distribution is never smoothed).  One fused launch computes it with its gradient
(``softmax_xent_kd``), so the loss stays two launches.

Keys: ``teacher`` ("module.path:ClassName", one of :data:`TEACHERS`), ``checkpoint`` (a ``ckpt_<epoch>.pt`` of
``utils/helper_funcs.save_checkpoint``: the teacher takes its weights from ``arena`` and its batch-norm statistics from
``extra_state['bn']``), ``alpha`` α in (0, 1] (0.5), ``temperature`` T > 0 (1.0), ``config`` (teacher constructor keys, only ``blocks``).
Every other teacher constructor key comes from the student.  The teacher is never trained, saved or exchanged: its weights, bf16 shadow
and running statistics stay as loaded, and a resumed run loads it again from ``checkpoint``."""
from __future__ import annotations

import importlib
import math
import os

import numpy as np
import torch

KEY = "distill"
KEYS = ("teacher", "checkpoint", "alpha", "temperature", "config")
CONFIG_KEYS = ("blocks",)
# the native ImageNet classifiers a teacher may be (module, class); the students are the same five (ModelBase.supports_distill)
TEACHERS = (("theanompi_b200.models.alex_net", "AlexNet"), ("theanompi_b200.models.googlenet", "GoogLeNet"),
            ("theanompi_b200.models.lasagne_model_zoo.vgg16", "VGG16"), ("theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50"),
            ("theanompi_b200.models.lasagne_model_zoo.resnet152_outdated", "ResNet152"))


def _real(v):
    return not isinstance(v, (bool, np.bool_)) and isinstance(v, (int, float, np.integer, np.floating)) and math.isfinite(v)


def check_config(cfg):
    """The validated dict {teacher, checkpoint, alpha, temperature, config}; anything malformed is a ValueError that names ``distill``.
    Whether the teacher imports and the checkpoint fits it is checked when :class:`Distill` builds it."""
    k = KEY
    if not isinstance(cfg, dict):
        raise ValueError("%s must be a dict or None, not %r" % (k, cfg))
    unknown = sorted(set(cfg) - set(KEYS))
    if unknown:
        raise ValueError("%s: unknown key %r; the keys are %s" % (k, unknown[0], ", ".join(KEYS)))
    teacher = cfg.get("teacher")
    parts = teacher.split(":") if isinstance(teacher, str) else []
    if len(parts) != 2 or not all(parts):
        raise ValueError("%s['teacher'] must be 'module.path:ClassName', not %r" % (k, teacher))
    ckpt = cfg.get("checkpoint")
    if not isinstance(ckpt, str) or not ckpt:
        raise ValueError("%s['checkpoint'] must be the path of a checkpoint of the teacher, not %r" % (k, ckpt))
    alpha = cfg.get("alpha", 0.5)
    if not (_real(alpha) and 0.0 < alpha <= 1.0):
        raise ValueError("%s['alpha'] must be a real number in (0, 1], not %r" % (k, alpha))
    temp = cfg.get("temperature", 1.0)
    if not (_real(temp) and temp > 0.0):
        raise ValueError("%s['temperature'] must be a finite real number > 0, not %r" % (k, temp))
    tc = cfg.get("config", {})
    if not isinstance(tc, dict):
        raise ValueError("%s['config'] must be a dict of teacher constructor keys, not %r" % (k, tc))
    bad = sorted(set(tc) - set(CONFIG_KEYS))
    if bad:
        raise ValueError("%s['config']: key %r is not accepted; the teacher takes every other constructor key from the student, and "
                         "only %s may be set" % (k, bad[0], ", ".join(CONFIG_KEYS)))
    out_tc = {}
    if "blocks" in tc:
        b = tc["blocks"]
        if not (isinstance(b, (list, tuple)) and b and all(not isinstance(n, bool) and isinstance(n, (int, np.integer)) and n >= 1
                                                           for n in b)):
            raise ValueError("%s['config']['blocks'] must be a list of ints >= 1, not %r" % (k, b))
        out_tc["blocks"] = tuple(int(n) for n in b)
    return {"teacher": teacher, "checkpoint": ckpt, "alpha": float(alpha), "temperature": float(temp), "config": out_tc}


def teacher_class(spec):
    """The class named by ``spec`` ("module.path:ClassName"); a ValueError names ``distill`` when it cannot be imported or is not one of
    :data:`TEACHERS`."""
    mod, name = spec.split(":")
    try:
        cls = getattr(importlib.import_module(mod), name)
    except (ImportError, AttributeError) as e:
        raise ValueError("%s['teacher'] = %r cannot be imported: %s" % (KEY, spec, e)) from None
    allowed = [getattr(importlib.import_module(m), c) for m, c in TEACHERS]
    if not any(cls is a for a in allowed):
        raise ValueError("%s['teacher'] = %r is not supported; the teacher is one of %s" % (KEY, spec, ", ".join(c for _, c in TEACHERS)))
    return cls


class KdTarget(object):
    """One step's distillation target for the loss (models/layers2.py: Softmax): the teacher's logits with α and T."""

    __slots__ = ("logits", "alpha", "temperature")

    def __init__(self, logits, alpha, temperature):
        self.logits, self.alpha, self.temperature = logits, alpha, temperature


class Distill(object):
    """The frozen teacher of a student model and its eval-mode forward (``config['distill']``, see the module docstring)."""

    def __init__(self, student, cfg):
        from ..models import layers2
        from ..models.layers2 import BatchNormal, Crop, Dropout
        cfg = check_config(cfg)
        self.alpha, self.temperature = cfg["alpha"], cfg["temperature"]
        cls = teacher_class(cfg["teacher"])
        path = cfg["checkpoint"]
        if not os.path.isfile(path):
            raise ValueError("%s['checkpoint']: no checkpoint at %r" % (KEY, path))
        B = student.batch_size
        tcfg = dict(verbose=False, rank=0, size=1, device=str(student.device), dtype=student.precision, batch_size=B, file_batch_size=B,
                    n_class=student.n_softmax_out, no_paraload=True, cuda_graph=False,
                    data_kwargs=dict(n_train_files=1, n_val_files=1, synthetic=True), **cfg["config"])
        # the layer classes keep class-wide lists (the train / eval switches, the dropout layer ids) and layers2 one weight generator: the
        # teacher's layers leave the lists and the generator is put back as it was, so the student and any model built after it draw,
        # number and switch exactly as without the teacher
        rng, rng_state = layers2.rng, layers2.rng.get_state()
        n_drop, n_bn, n_crop = len(Dropout.layers), len(BatchNormal.layers), len(Crop.layers)
        try:
            self.teacher = t = cls(tcfg)
        finally:
            self._dropouts = Dropout.layers[n_drop:]
            self._bns = BatchNormal.layers[n_bn:]
            self._crops = Crop.layers[n_crop:]
            del Dropout.layers[n_drop:], BatchNormal.layers[n_bn:], Crop.layers[n_crop:]
            rng.set_state(rng_state)
            layers2.rng = rng
        name = type(student).__name__
        if tuple(t.input_shape[1:]) != tuple(student.input_shape[1:]):
            raise ValueError("%s: the teacher %s takes (H, W, C) = %s, the student %s %s" % (
                KEY, cls.__name__, tuple(t.input_shape[1:]), name, tuple(student.input_shape[1:])))
        if t.n_softmax_out != student.n_softmax_out:
            raise ValueError("%s: the teacher %s has %d classes, the student %s %d" % (KEY, cls.__name__, t.n_softmax_out, name,
                                                                                     student.n_softmax_out))
        self._load(path)

    def _load(self, path):
        t = self.teacher
        try:
            sd = torch.load(path, map_location="cpu", weights_only=False)
        except Exception as e:  # noqa: BLE001
            raise ValueError("%s['checkpoint']: %r cannot be read: %s" % (KEY, path, e)) from None
        a = t.arena
        arena = sd.get("arena") if isinstance(sd, dict) else None
        if arena is None or list(arena.get("sizes", ())) != list(a.sizes) or list(arena.get("offsets", ())) != list(a.offsets):
            raise ValueError("%s['checkpoint']: the arena of %r does not match the layout of the teacher %s%s" % (
                KEY, path, type(t).__name__, "" if arena is None else " (%d tensors, %d in the checkpoint)" % (len(a.sizes),
                                                                                                               len(arena.get("sizes", ())))))
        bns = t._bn_layers()
        bn = (sd.get("extra_state") or {}).get("bn", [])
        if len(bn) != len(bns) or any(tuple(m.shape) != tuple(l.running_mean.shape) for l, (m, _) in zip(bns, bn)):
            raise ValueError("%s['checkpoint']: the batch-norm statistics of %r do not match the teacher %s (%d layers, %d in the "
                             "checkpoint)" % (KEY, path, type(t).__name__, len(bns), len(bn)))
        a.load_state_dict(arena)
        for l, (m, v) in zip(bns, bn):
            l.running_mean = m.to(t.device, torch.float32).clone()
            l.running_var = v.to(t.device, torch.float32).clone()

    def target(self, x):
        """This step's :class:`KdTarget`: the teacher's logits of its eval-mode forward on ``x`` (no gradient, no statistics update,
        no dropout, whatever the class-wide switches say)."""
        for l in self._dropouts:
            l.flag_on = False
        for l in self._bns:
            l.training = False
        for l in self._crops:
            l.flag_rand = False
        with torch.no_grad():
            self.teacher.forward(x)
        return KdTarget(self.teacher.output_layer.logits, self.alpha, self.temperature)
