"""Optimizer split for BSP ("cdd" mode) and the flat fused SGD.

Reference: ``theanompi/lib/opt.py`` builds two Theano functions per model,
``get_vel`` (fwd + bwd + *pre* update into the send buffers ``vels``) and
``descent_vel`` (*post* update from the receive buffers ``vels2``), with one
elementwise kernel per tensor per buffer (``opt.py:2-52,181-330``).

Here the three reference optimizers keep their names and algebra but act on the
flat arena (one launch each):

``BSP_MSGD``   aggregate *momentum*  (``opt.py:181-268``)
               pre : U ← μU + (G + ηW)            send = U
               post: W ← W − lr·m · R / k          (R = Σ_ranks U)
``_BSP_MSGD``  aggregate *gradient*  (``opt.py:78-177``)
               pre : G ← (G + ηW) / k              send = G
               post: U ← μU + R ;  W ← W − lr·m · U
``BSP_SGD``    no momentum           (``opt.py:271-330``)
               pre : G ← lr·m · (G + ηW) / k       send = G
               post: W ← W − R
``BSP_LARS``   :class:`FlatLARS`, aggregate gradient (``config['optimizer'] = 'lars'``; no counterpart in the reference)
               pre : batch-norm groups             send = G
               post: LARS step from R / k
``BSP_LAMB``   :class:`FlatLAMB`, aggregate gradient (``config['optimizer'] = 'lamb'``; no counterpart in the reference)
               pre : batch-norm groups             send = G
               post: LAMB step from R / k

(m = per-group lr multiplier: 1 for 'W', 2 for 'b'; η only on 'W'; BN gamma/beta
are updated locally in the pre step and never exchanged, ``opt.py:207-226``.)

The H100 fast path does not use the split at all: the fused exchanger kernels
(``csrc/comm_kernels.cu``) read every peer's G over NVLink, average, and apply
the momentum/weight-decay/lr update in the same pass — :class:`FlatSGD` is the
k = 1 (single GPU) instance of that kernel.

Reference bug fixed (SURVEY §2.9 #8): ``cdd_iter_fn`` applied ``descent_vel()``
*before* the next ``get_vel()``; here the post step runs right after the exchange,
so validation and checkpoints always see fully-updated weights.  The reference's
Nesterov expression (``mu**2*u - (1+mu)*g`` followed by ``w - lr*u``) has the
wrong sign; we implement the standard form  ``w ← w − lr (g_eff + μ u_new)``.
"""
from __future__ import annotations

import numpy as np
import torch

from ..ops import reference as ref
from ..parallel.arena import BLOCK


class SharedScalar(object):
    """``theano.shared`` look-alike backed by one element of a device tensor so
    CUDA graphs pick up new values without re-capture (``model.shared_lr``)."""

    def __init__(self, buf, index, value=0.0):
        self._buf, self._i = buf, index
        self._host = float(value)
        self.set_value(value)

    def get_value(self):
        return self._host

    def set_value(self, v):
        self._host = float(v)
        self._buf[self._i] = float(v)

    def mirror(self, v):
        """Set the host copy only: the device element already holds ``v`` (a per-update :class:`LrSchedule` wrote it)."""
        self._host = float(v)


class LrSchedule(object):
    """Per-update learning-rate schedule (``config['lr_schedule']``, a dict), the lr of update u = 0, 1, 2, ... written to
    ``arena.hyper[0]`` by one single-thread launch at the start of each update's step (``cuda_impl.lr_schedule_step``), inside
    the captured CUDA graph: replays follow the schedule with no host work.  The CPU applies ``reference.lr_at`` instead.

    Keys (``peak`` is the model's learning_rate):
      ``warmup_steps`` W >= 0 (0), ``warmup_start`` s in [0, 1] (0): for u < W, lr = peak·(s + (1 − s)·u / W);
      ``decay``: 'constant' (default), 'cosine', 'poly' (``power`` >= 0, default 1) or 'multistep' (``milestones``: at most 8
      strictly increasing update indices >= W; ``gamma``, default 0.1);
      ``total_steps`` T > W (default: the model's n_epochs × updates_per_epoch), ``final_lr`` (0): the end of cosine and poly.

    The update index ``u`` (int64 [1], on the arena's device) is checkpointed by :meth:`state_dict`."""

    KEYS = ("warmup_steps", "warmup_start", "decay", "total_steps", "final_lr", "power", "gamma", "milestones")
    DECAYS = ("constant", "cosine", "poly", "multistep")
    MAX_MILESTONES = 8

    def __init__(self, arena, cfg, peak, total_steps):
        if not isinstance(cfg, dict):
            raise ValueError("lr_schedule must be a dict or None, not %r" % (cfg,))
        unknown = sorted(set(cfg) - set(self.KEYS))
        if unknown:
            raise ValueError("lr_schedule: unknown key %r; the keys are %s" % (unknown[0], ", ".join(self.KEYS)))
        self.arena = arena
        self.peak = float(peak)
        self.decay = cfg.get("decay", "constant")
        if self.decay not in self.DECAYS:
            raise ValueError("lr_schedule['decay'] must be one of %s, not %r" % (", ".join(self.DECAYS), self.decay))
        self.warmup_steps = self._int(cfg, "warmup_steps", 0)
        if self.warmup_steps < 0:
            raise ValueError("lr_schedule['warmup_steps'] must be >= 0, not %d" % self.warmup_steps)
        self.total_steps = self._int(cfg, "total_steps", total_steps)
        if not self.warmup_steps < self.total_steps:
            raise ValueError("lr_schedule['total_steps'] (%d) must be greater than warmup_steps (%d)"
                             % (self.total_steps, self.warmup_steps))
        self.warmup_start = self._float(cfg, "warmup_start", 0.0)
        if not 0.0 <= self.warmup_start <= 1.0:
            raise ValueError("lr_schedule['warmup_start'] must be in [0, 1], not %r" % self.warmup_start)
        self.final_lr = self._float(cfg, "final_lr", 0.0)
        self.power = self._float(cfg, "power", 1.0)
        if not self.power >= 0.0:
            raise ValueError("lr_schedule['power'] must be >= 0, not %r" % self.power)
        self.gamma = self._float(cfg, "gamma", 0.1)
        ms = cfg.get("milestones", ())
        if not isinstance(ms, (list, tuple)) or any(isinstance(m, bool) or not isinstance(m, (int, np.integer)) for m in ms):
            raise ValueError("lr_schedule['milestones'] must be a list of update indices, not %r" % (ms,))
        self.milestones = tuple(int(m) for m in ms)
        if len(self.milestones) > self.MAX_MILESTONES:
            raise ValueError("lr_schedule['milestones'] holds at most %d update indices, not %d" % (self.MAX_MILESTONES, len(ms)))
        if any(b <= a for a, b in zip(self.milestones, self.milestones[1:])):
            raise ValueError("lr_schedule['milestones'] must be strictly increasing: %r" % (self.milestones,))
        if self.milestones and self.milestones[0] < self.warmup_steps:
            raise ValueError("lr_schedule['milestones'] must be >= warmup_steps (%d): %r" % (self.warmup_steps, self.milestones))
        self.u = torch.zeros(1, dtype=torch.int64, device=arena.hyper.device)

    @staticmethod
    def _int(cfg, key, default):
        v = cfg.get(key, default)
        if isinstance(v, bool) or not isinstance(v, (int, np.integer)):
            raise ValueError("lr_schedule[%r] must be an int, not %r" % (key, v))
        return int(v)

    @staticmethod
    def _float(cfg, key, default):
        v = cfg.get(key, default)
        if isinstance(v, bool) or not isinstance(v, (int, float, np.number)) or not np.isfinite(v):
            raise ValueError("lr_schedule[%r] must be a finite number, not %r" % (key, v))
        return float(v)

    def lr_at(self, u):
        """The schedule's lr of update ``u`` (``reference.lr_at``, an np.float32)."""
        return ref.lr_at(u, self.peak, self.decay, self.warmup_steps, self.warmup_start, self.total_steps, self.final_lr, self.power,
                         self.gamma, self.milestones)

    def step(self):
        """Start an update: lr(u) into ``arena.hyper[0]``, u += 1 (on CUDA one launch that reads only device memory)."""
        a = self.arena
        if a.hyper.is_cuda:
            from ..ops import cuda_impl
            cuda_impl.lr_schedule_step(a, self, self.u)
            return
        a.hyper[0] = float(self.lr_at(int(self.u)))
        self.u += 1

    def give_back(self):
        """Return the index of an update that was started but dropped (an open gradient-accumulation window at the end of an
        epoch): one device decrement, outside any graph.  The next update recomputes the same lr."""
        self.u -= 1

    def value(self):
        """The lr the last :meth:`step` wrote (reads ``arena.hyper[0]``: a device read)."""
        return float(self.arena.hyper[0])

    def state_dict(self):
        return {"u": int(self.u)}

    def load_state_dict(self, sd):
        self.u.fill_(int(sd["u"]))


class ModelEma(object):
    """Exponential moving average of the model (``config['model_ema']``, a dict): torchvision's ``ExponentialMovingAverage``, i.e.
    ``torch.optim.swa_utils.AveragedModel`` with ``avg_fn = d·e + (1 − d)·w`` and ``use_buffers=True``.  E holds an fp32 copy of the
    arena's W region and of the running mean and variance of every batch-norm layer, taken when the model is compiled.

    Keys: ``decay`` d in [0, 1] (0.9999), ``every`` >= 1 (1; torchvision's ``--model-ema-steps``), ``warmup`` >= 0 (0).  After
    optimizer update u = 1, 2, ... the average moves iff u is a multiple of ``every``: it copies E ← W when nothing has been averaged
    yet or u <= ``warmup``, else E ← fp32(d)·E + fp32(1 − d)·W (``reference.ema_update``).

    On CUDA :meth:`update` is two launches after the step's update (``cuda_impl.ema_advance``, ``cuda_impl.ema_update``) that read
    only device memory: the counters {u, n_averaged} and the step's mode live in :attr:`state`, so a captured CUDA graph keeps
    counting.  The batch-norm statistics are reached through a device table of {dst, src, n} segments, built at the first
    :meth:`update` or :meth:`swap` and rebuilt when a layer's statistics tensors have been replaced (``BatchNormal.forward`` moves
    them to the device lazily, ``load_extra_state`` replaces them).  :meth:`swap` exchanges the model's weights and statistics with
    E in one pass, the bf16 shadow following W."""

    KEY = "model_ema"
    KEYS = ("decay", "every", "warmup")

    def __init__(self, arena, bn_layers, cfg):
        """``bn_layers``: a callable returning the model's batch-norm layers; ``cfg``: a dict that :meth:`check_config` accepts."""
        cfg = self.check_config(cfg)
        self.decay, self.every, self.warmup = cfg["decay"], cfg["every"], cfg["warmup"]
        self.one_minus_decay = float(np.float32(1.0 - self.decay))          # 1 − d in float64, rounded once to fp32
        self.arena, self.bn_layers = arena, bn_layers
        dev = arena.W.device
        stats = self._stats()
        self.sizes = [int(s.numel()) for s in stats]
        with torch.no_grad():
            self.E = arena.W.detach().clone()
            self.E_bn = (torch.cat([s.detach().reshape(-1).to(dev, torch.float32) for s in stats]) if stats
                         else torch.zeros(0, dtype=torch.float32, device=dev))
        self.state = torch.zeros(3, dtype=torch.int64, device=dev)          # u, n_averaged, mode of the last update
        self._table, self._src = None, None

    @classmethod
    def check_config(cls, cfg):
        """The validated dict {decay, every, warmup}; anything else is a ValueError that names ``model_ema``."""
        k = cls.KEY
        if not isinstance(cfg, dict):
            raise ValueError("%s must be a dict or None, not %r" % (k, cfg))
        unknown = sorted(set(cfg) - set(cls.KEYS))
        if unknown:
            raise ValueError("%s: unknown key %r; the keys are %s" % (k, unknown[0], ", ".join(cls.KEYS)))
        d = cfg.get("decay", 0.9999)
        if isinstance(d, bool) or not isinstance(d, (int, float, np.integer, np.floating)) or not np.isfinite(d) or not 0.0 <= d <= 1.0:
            raise ValueError("%s['decay'] must be a real number in [0, 1], not %r" % (k, d))
        out = {"decay": float(d)}
        for key, default, lo in (("every", 1, 1), ("warmup", 0, 0)):
            v = cfg.get(key, default)
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < lo:
                raise ValueError("%s[%r] must be an int >= %d, not %r" % (k, key, lo, v))
            out[key] = int(v)
        return out

    def _stats(self):
        return [t for l in self.bn_layers() for t in (l.running_mean, l.running_var)]

    def _pairs(self):
        """(E part, model tensor) for W and every statistics tensor (the CPU path)."""
        out, o = [(self.E, self.arena.W)], 0
        for s, n in zip(self._stats(), self.sizes):
            out.append((self.E_bn[o:o + n], s))
            o += n
        return out

    def _ensure_table(self):
        """The device segment table of the statistics ({E_bn + offset, statistics tensor, n} per tensor, int64 [n, 3]), built again in
        place when a layer holds other tensors than the ones it points at, first moving statistics still on the host to the device
        (as the layer's first forward would)."""
        dev = self.arena.W.device
        for l in self.bn_layers():
            if l.running_mean.device != dev:
                l.running_mean = l.running_mean.to(dev)
                l.running_var = l.running_var.to(dev)
        stats = self._stats()
        if self._src is not None and all(a is b for a, b in zip(self._src, stats)):
            return
        rows, o = [], 0
        for s, n in zip(stats, self.sizes):
            assert s.dtype == torch.float32 and s.is_contiguous() and s.numel() == n, (s.dtype, tuple(s.shape), n)
            rows.append((self.E_bn.data_ptr() + 4 * o, s.data_ptr(), n))
            o += n
        host = torch.tensor(rows, dtype=torch.int64).view(-1, 3)
        if self._table is None:
            self._table = torch.zeros_like(host, device=dev)
        self._table.copy_(host)
        self._src = stats

    def update(self):
        """The averaging step after an optimizer update (on CUDA two launches, inside a captured step)."""
        if self.arena.W.is_cuda:
            from ..ops import cuda_impl
            self._ensure_table()
            cuda_impl.ema_advance(self.state, self.every, self.warmup)
            cuda_impl.ema_update(self.arena, self.E, self.state, self._table, self.decay, self.one_minus_decay)
            return
        u, n, mode = ref.ema_advance(int(self.state[0]), int(self.state[1]), self.every, self.warmup)
        self.state.copy_(torch.tensor([u, n, mode]))
        ref.ema_update(self._pairs(), mode, self.decay, self.one_minus_decay)

    def swap(self):
        """Exchange the model's W and batch-norm statistics with E (the bf16 shadow takes bf16-RN of the new W); twice is the
        identity."""
        a = self.arena
        if a.W.is_cuda:
            from ..ops import cuda_impl
            self._ensure_table()
            cuda_impl.ema_swap(a, self.E, self._table)
            return
        ref.ema_swap([(a.W, self.E)] + [(s, e) for e, s in self._pairs()[1:]], w_half=a.H)

    @property
    def n_averaged(self):
        return int(self.state[1])

    def state_dict(self):
        return {"E": self.E.detach().cpu().clone(), "bn": self.E_bn.detach().cpu().clone(), "u": int(self.state[0]),
                "n_averaged": int(self.state[1])}

    def load_state_dict(self, sd):
        if tuple(sd["E"].shape) != tuple(self.E.shape) or tuple(sd["bn"].shape) != tuple(self.E_bn.shape):
            raise ValueError("model_ema: the checkpoint's average does not match this model's arena and batch-norm layers")
        with torch.no_grad():
            self.E.copy_(sd["E"].to(self.E.device))
            self.E_bn.copy_(sd["bn"].to(self.E_bn.device))
        self.state.copy_(torch.tensor([int(sd["u"]), int(sd["n_averaged"]), 0]))


class Sam(object):
    """Sharpness-aware minimization (``config['sam']``, a dict; Foret et al., 2021) and its adaptive variant ASAM (Kwon et al., 2021),
    with the semantics of the standard PyTorch SAM wrapper (davda54/sam, the version that keeps ``old_p``).  After the step's first
    forward and backward at w, :meth:`perturb` computes n = ‖g‖₂ (ASAM: ‖|w|⊙g‖₂) over the real elements of every arena tensor and
    s = ρ / (n + 1e-12), saves w into P and moves the weights to w + e, e = g·s (ASAM: w²·g·s); the model then runs the second forward
    and backward there, and :meth:`restore` puts w back before the optimizer steps on the second gradient.

    Keys: ``rho`` ρ > 0 (0.05; ASAM's papers use about 0.5 to 2), ``adaptive`` (False).

    On CUDA :meth:`perturb` is three launches and :meth:`restore` one (``cuda_impl.sam_norm``, ``sam_perturb``, ``sam_restore``), all
    reading only device memory: they run inside the captured step.  The record {n, s, finite} (``csrc/api.h: ClipRecord``) stays on the
    device.  When n is NaN or Inf the weights are not moved, so the second pass runs at w; the wrapper would write NaN into every
    weight instead.  P costs 4 bytes per arena element and exists only with the key."""

    KEY = "sam"
    KEYS = ("rho", "adaptive")

    def __init__(self, arena, cfg):
        cfg = self.check_config(cfg)
        self.rho, self.adaptive = cfg["rho"], cfg["adaptive"]
        self.arena = arena
        dev = arena.W.device
        self.P = torch.zeros_like(arena.W)
        self.rec = torch.zeros(4, dtype=torch.float32, device=dev)          # csrc/api.h: ClipRecord {n, s, finite, pad}
        self._partial = torch.zeros(arena.n_blocks, dtype=torch.float32, device=dev) if arena.W.is_cuda else None

    @classmethod
    def check_config(cls, cfg):
        """The validated dict {rho, adaptive}; anything else is a ValueError that names ``sam``."""
        k = cls.KEY
        if not isinstance(cfg, dict):
            raise ValueError("%s must be a dict or None, not %r" % (k, cfg))
        unknown = sorted(set(cfg) - set(cls.KEYS))
        if unknown:
            raise ValueError("%s: unknown key %r; the keys are %s" % (k, unknown[0], ", ".join(cls.KEYS)))
        rho = cfg.get("rho", 0.05)
        if isinstance(rho, bool) or not isinstance(rho, (int, float, np.integer, np.floating)) or not np.isfinite(rho) or not rho > 0:
            raise ValueError("%s['rho'] must be a finite real number > 0, not %r" % (k, rho))
        adaptive = cfg.get("adaptive", False)
        if not isinstance(adaptive, (bool, np.bool_)):
            raise ValueError("%s['adaptive'] must be a bool, not %r" % (k, adaptive))
        return {"rho": float(rho), "adaptive": bool(adaptive)}

    @property
    def norm(self):
        """n of the last :meth:`perturb` (a device scalar): NaN or Inf when the weights were not moved."""
        return self.rec[0]

    def perturb(self):
        """P ← W, then W ← W + e and the bf16 shadow ← bf16(W), from the gradient of the first pass in the arena's G region."""
        a = self.arena
        if a.W.is_cuda:
            from ..ops import cuda_impl
            cuda_impl.sam_norm(a, self.rho, self.adaptive, self._partial, self.rec)
            cuda_impl.sam_perturb(a, self.P, self.rec, self.adaptive)
            return
        n = ref.sam_norm(a.W, a.G, a.offsets, a.sizes, self.adaptive)
        s, finite = ref.sam_scale(n, self.rho)
        self.rec[0], self.rec[1] = float(n), s
        self.rec[2:3].view(torch.int32).fill_(int(finite))
        ref.sam_perturb(a.W, a.G, self.P, s, finite, a.offsets, a.sizes, self.adaptive, w_half=a.H)

    def restore(self):
        """W ← P and the bf16 shadow ← bf16(P): the weights before :meth:`perturb`, bit for bit."""
        a = self.arena
        if a.W.is_cuda:
            from ..ops import cuda_impl
            cuda_impl.sam_restore(a, self.P)
            return
        ref.sam_restore(a.W, self.P, w_half=a.H)


def _fc_fusable(p, block):
    """Can ``p``'s weight gradient be consumed by the SGD epilogue of its wgrad GEMM?  It must come from ONE fp32 GEMM straight
    into ``gbuf`` (native FC / Softmax weights, ``rs_ok``), not be accumulated over several passes, and its shape must take the
    un-padded path of ``cuda_impl.linear_bias_act_bwd`` (both dimensions multiples of ``block`` = elements per 16 bytes)."""
    return (getattr(p, "rs_ok", False) and p.dim() == 2 and not getattr(p, "gaccum", False)
            and p.shape[0] % block == 0 and p.shape[1] % block == 0)


def complement_ranges(arena, armed):
    """Arena element ranges ``[lo, hi)`` (block aligned, sorted) NOT covered by the parameters at indices ``armed``."""
    out, lo = [], 0
    for i in sorted(armed, key=lambda j: arena.offsets[j]):
        o = arena.offsets[i]
        end = o + -(-arena.sizes[i] // BLOCK) * BLOCK
        if o > lo:
            out.append((lo, o))
        lo = max(lo, end)
    if lo < arena.numel:
        out.append((lo, arena.numel))
    return out


class FlatOptimizer(object):
    """A local optimizer over the whole flat arena.  On CUDA one native launch per step (``csrc/comm_kernels.cu:
    flat_update_kernel``, Adam adds the launch that advances its step counter), with lr read from ``arena.hyper[0]`` on the
    device and the bf16 shadow refreshed in the same pass, so the step is CUDA-graph capturable.  On the CPU the same update
    runs through its ``ops/reference.py`` function.

    A subclass names its kernel ``rule``, whether the rule keeps state in the arena's U region (``uses_u``), its extra flat
    ``buffers`` (zero-initialised, saved by :meth:`state_dict` under their names), its ``reference`` function and, in
    :meth:`hyper`, its float hyper-parameters in the order both take them.

    :meth:`set_grad_clip` adds global gradient-norm clipping to every step (``torch.nn.utils.clip_grad_norm_``).  On CUDA that is
    two more launches before the update (``cuda_impl.grad_clip_norm``), whose record the update pass reads: it applies s·g, or
    returns before it touches memory when the norm is NaN or Inf.  G itself is not changed."""

    rule = None
    uses_u = True
    buffers = ()
    reference = None
    t = None                         # device step counter of a rule that reads one (Adam)
    max_norm = None                  # gradient clipping threshold (set_grad_clip), None: off
    skipped = None                   # with clipping: int64 [1], the number of steps skipped for a non-finite gradient norm

    def __init__(self, arena):
        self.arena = arena
        for name in self.buffers:
            setattr(self, name, torch.zeros_like(arena.W))

    def hyper(self):
        raise NotImplementedError

    def _state(self):
        return ([self.arena.U] if self.uses_u else []) + [getattr(self, n) for n in self.buffers]

    # ---- global gradient-norm clipping
    def set_grad_clip(self, max_norm):
        """Before every step, compute the global L2 norm n of the gradient over the real elements of every arena tensor.  A finite n
        scales the step's gradient by s = min(1, max_norm / (n + 1e-6)) (``torch.nn.utils.clip_grad_norm_``; weight decay is added
        after the scaling).  A NaN or Inf n skips the step: W, the bf16 shadow, the optimizer state and Adam's counter are left as
        they are, and :attr:`skipped` counts it.  ``None`` turns clipping off.  On CUDA ``max_norm`` is a launch argument: a step
        captured in a CUDA graph keeps the value it was captured with."""
        if max_norm is None:
            self.max_norm = None
            return
        if self.rule in ("lars", "lamb"):
            raise ValueError("gradient-norm clipping is for the sgd, adam, rmsprop, adadelta and rmsprop_centered flat optimizers; "
                             "%s's trust ratios already normalise every tensor's step" % self.rule.upper())
        max_norm = float(max_norm)
        if not max_norm > 0:
            raise ValueError("grad_clip must be a positive maximum norm, not %r" % max_norm)
        self.max_norm = max_norm
        if self.skipped is None:
            dev = self.arena.W.device
            self._clip_rec = torch.zeros(4, dtype=torch.float32, device=dev)      # csrc/api.h: ClipRecord
            self.skipped = torch.zeros(1, dtype=torch.int64, device=dev)
            self._clip_partial = torch.zeros(self.arena.n_blocks, dtype=torch.float32, device=dev) if self.arena.W.is_cuda else None

    @property
    def grad_norm(self):
        """The global gradient norm of the last clipped step, before clipping (a device scalar); None without clipping."""
        return None if self.max_norm is None else self._clip_rec[0]

    def _clip_cuda(self, g):
        """With clipping on, the two norm launches over ``g``; returns the record the update pass reads (None: no clipping)."""
        if self.max_norm is None:
            return None
        from ..ops import cuda_impl
        cuda_impl.grad_clip_norm(self.arena, g, self.max_norm, self._clip_partial, self._clip_rec, self.skipped)
        return self._clip_rec

    def _clip_cpu(self, g):
        """The CPU twin of :meth:`_clip_cuda`: returns s (1.0 without clipping), or None when the step is skipped."""
        if self.max_norm is None:
            return 1.0
        a = self.arena
        n, s, finite = ref.clip_scale(g, a.offsets, a.sizes, self.max_norm)
        self._clip_rec[0], self._clip_rec[1] = n, s
        self._clip_rec[2:3].view(torch.int32).fill_(int(finite))
        if not finite:
            self.skipped += 1
            return None
        return s

    def step(self, lr=None):
        a = self.arena
        if a.W.is_cuda:
            from ..ops import cuda_impl
            cuda_impl.flat_update(a, self.rule, self.hyper(), self._state(), step=self.t, clip=self._clip_cuda(a.G))
            return
        s = self._clip_cpu(a.G)
        if s is None:
            return
        self._reference_step(float(a.hyper[0]) if lr is None else lr, a.G if s == 1.0 else a.G * s)

    def _reference_step(self, lr, g):
        a = self.arena
        type(self).reference(a.W, g, *self._state(), a.lr_mult_vector(), a.wd_vector(), lr, *self.hyper(), w_half=a.H)

    def state_dict(self):
        sd = {n: getattr(self, n).detach().cpu() for n in self.buffers}
        if self.max_norm is not None:
            sd["skipped"] = int(self.skipped)
        return sd

    def load_state_dict(self, sd):
        for n in self.buffers:
            getattr(self, n).copy_(sd[n].to(self.arena.W.device))
        if self.max_norm is not None and "skipped" in sd:
            self.skipped.fill_(int(sd["skipped"]))


class FlatSGD(FlatOptimizer):
    """Fused momentum-SGD over the whole arena (or a block range); momentum in the arena's U region.

    :meth:`arm` (single GPU, k = 1) moves the update of the FC / Softmax weights into the epilogue of their weight-gradient GEMM
    (``cuda_impl.gemm_sgd``): their fp32 gradient is never written, and ``step(lr, 1)`` updates only the rest of the arena.  With
    gradient clipping (:meth:`FlatOptimizer.set_grad_clip`) nothing is armed: an epilogue would update its weight before the
    global norm exists.  Nor with gradient accumulation (``model.grad_accum`` > 1): the epilogue would update the weight on every
    micro-step.  Nor with sharpness-aware minimization (``model.sam_opt``): the first backward of the step would update the weight
    before the ascent step.  The clipping factor is folded into inv_k."""

    rule = "sgd"

    def __init__(self, arena, mu=0.9, nesterov=False, use_momentum=True):
        super().__init__(arena)
        self.mu = mu if use_momentum else 0.0
        self.nesterov = nesterov
        self.armed = []
        self.rest = None              # complement of the armed weights, set by arm()

    def arm(self, model, enable=True):
        """Arm the eligible weights of ``model`` (CUDA, no gradient monitoring: that reads G); ``enable=False`` disarms.
        ``model.monitor_grad`` is read here, when the iteration functions are compiled: set it before; ``grad_norms()`` refuses
        to run while weights are armed."""
        a = self.arena
        for p in a.params:
            p.sgd_epilogue = None
        self.armed, self.rest = [], None
        if (not enable or not a.W.is_cuda or getattr(model, "monitor_grad", False) or self.max_norm is not None
                or getattr(model, "grad_accum", 1) > 1 or getattr(model, "sam_opt", None) is not None):
            return
        dt = getattr(model, "act_dtype", None)
        block = 16 // torch.empty((), dtype=dt).element_size() if dt is not None else 8
        self.armed = [i for i, p in enumerate(a.params) if _fc_fusable(p, block)]
        for i in self.armed:
            p = a.params[i]
            p.sgd_epilogue = self
            p.arena_group = a.group_of[i]
        self.rest = complement_ranges(a, self.armed)

    def step(self, lr=None, k=1, src="G", lo=0, hi=None, only_local=False, only_exchanged=False):
        """With clipping, the norm is the one of the whole gradient region ``src``, whatever range or groups the step updates."""
        a = self.arena
        g = getattr(a, src)
        if a.W.is_cuda:
            from ..ops import cuda_impl
            clip = self._clip_cuda(g)
            ranges = [(lo, a.numel if hi is None else hi)]
            if self.rest is not None and k == 1 and src == "G" and (lo, hi) == (0, None) and not (only_local or only_exchanged):
                ranges = self.rest    # the armed weights were updated by their wgrad GEMMs during backward
            for rlo, rhi in ranges:
                cuda_impl.sgd_flat(a, g, lr, self.mu, self.nesterov, 1.0 / k, rlo, rhi, only_local, only_exchanged, clip=clip)
            return
        inv_k = 1.0 / k
        if self.max_norm is not None:
            s = self._clip_cpu(g)
            if s is None:
                return
            inv_k = float(np.float32(inv_k) * np.float32(s))          # the kernel's inv_k·s in fp32
        lr = float(a.hyper[0]) if lr is None else lr
        hi = a.numel if hi is None else hi
        sl = slice(lo, hi)
        lrm, wd = a.lr_mult_vector()[sl], a.wd_vector()[sl]
        w, gg, u = a.W[sl], g[sl], a.U[sl]
        if only_local or only_exchanged:
            ex = a.exch_vector()[sl]
            m = ~ex if only_local else ex
            idx = m.nonzero().squeeze(1)
            if idx.numel() == 0:
                return
            w2, u2 = w[idx].clone(), u[idx].clone()
            ref.sgd_flat(w2, gg[idx], u2, lrm[idx], wd[idx], lr, self.mu, self.nesterov, inv_k)
            w[idx] = w2
            u[idx] = u2
        else:
            ref.sgd_flat(w, gg, u, lrm, wd, lr, self.mu, self.nesterov, inv_k)
        if a.H is not None:
            a.H[sl].copy_(w)


class FlatAdam(FlatOptimizer):
    """Adam: first moment in the arena's U region, second moment in ``V``, step counter ``t`` in device memory.  The
    reference's Wide-ResNet uses Keras Adam (``keras_model_zoo/wresnet.py:159``)."""

    rule, buffers = "adam", ("V",)

    def __init__(self, arena, b1=0.9, b2=0.999, eps=1e-8):
        super().__init__(arena)
        self.b1, self.b2, self.eps = b1, b2, eps
        self.t = torch.zeros(1, dtype=torch.int64, device=arena.W.device)

    def hyper(self):
        return (self.b1, self.b2, self.eps)

    def _reference_step(self, lr, g):
        a = self.arena
        self.t += 1
        ref.adam_flat(a.W, g, a.U, self.V, a.lr_mult_vector(), a.wd_vector(), lr, *self.hyper(), t=float(self.t), w_half=a.H)

    def state_dict(self):
        return dict(super().state_dict(), t=int(self.t))

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        self.t.fill_(int(sd["t"]))


class FlatRMSProp(FlatOptimizer):
    """RMSProp, the squared-gradient average in ``V``: ``torch.optim.RMSprop(alpha=0.99, eps=1e-8)`` without momentum, plus an
    optional clip of the updated weights to ``[-clip, clip]`` (the WGAN critic's weight clipping, folded into the same pass).  It
    is the optimizer of the torch GAN twins, not the reference's: the reference's MNIST GANs (``lasagne_model_zoo/wgan.py:18-59``)
    use a centred RMSProp with momentum 0.5 that rescales the gradient by its norm first.  That rescaling is
    :meth:`FlatOptimizer.set_grad_clip` (``grad_clip=5``)."""

    rule, uses_u, buffers, reference = "rmsprop", False, ("V",), ref.rmsprop_flat

    def __init__(self, arena, alpha=0.99, eps=1e-8, clip=0.0):
        super().__init__(arena)
        self.alpha, self.eps, self.clip = alpha, eps, clip

    def hyper(self):
        return (self.alpha, self.eps, self.clip)


class FlatAdadelta(FlatOptimizer):
    """Adadelta, the update accumulator in the arena's U region (saved with the arena), the squared-gradient average in ``V``:
    ``torch.optim.Adadelta(rho=0.95, eps=1e-6)``, which at lr = 1 is the reference LSTM's ``adadelta``
    (``models/lstm.py:284-342``)."""

    rule, buffers, reference = "adadelta", ("V",), ref.adadelta_flat

    def __init__(self, arena, rho=0.95, eps=1e-6):
        super().__init__(arena)
        self.rho, self.eps = rho, eps

    def hyper(self):
        return (self.rho, self.eps)


class FlatCenteredRMSProp(FlatOptimizer):
    """The reference LSTM's ``rmsprop`` (``models/lstm.py:376-402``: centred, momentum 0.9, eps 1e-4 inside the square root):
    the momentum in the arena's U region, the gradient and squared-gradient averages in ``R`` and ``S``."""

    rule, buffers, reference = "rmsprop_centered", ("R", "S"), ref.rmsprop_centered_flat

    def __init__(self, arena, rho=0.95, mu=0.9, eps=1e-4):
        super().__init__(arena)
        self.rho, self.mu, self.eps = rho, mu, eps

    def hyper(self):
        return (self.rho, self.mu, self.eps)


class FlatLARS(FlatOptimizer):
    """LARS (layer-wise adaptive rate scaling; You, Gitman and Ginsburg, 2017): momentum SGD in which every weight tensor's
    effective gradient is scaled by its trust ratio ``eta·‖W‖ / (‖g‖ + wd·‖W‖)``; biases and batch-norm parameters keep ratio 1.
    Momentum lives in the arena's U region, so checkpoints carry it.

    On CUDA a step is three launches that read only device memory (CUDA-graph capturable, bit-reproducible): per-block sums of
    squares, one per-tensor reduction that writes :attr:`norms` ([n_tensors, 2]: ‖W‖, ‖g‖) and :attr:`trust` ([n_tensors]), and
    the ``flat_update`` pass of the LARS rule.  The update needs every tensor's whole gradient before it changes any element, so
    LARS never runs in the FC weight-gradient GEMM epilogue (:meth:`FlatSGD.arm`)."""

    rule = "lars"

    def __init__(self, arena, mu=0.9, nesterov=False, eta=0.001):
        super().__init__(arena)
        self.mu, self.nesterov, self.eta = mu, nesterov, eta
        n, dev = len(arena.sizes), arena.W.device
        self.trust = torch.ones(n, dtype=torch.float32, device=dev)
        self.norms = torch.zeros(n, 2, dtype=torch.float32, device=dev)
        self._partial = torch.zeros(arena.n_blocks, 2, dtype=torch.float32, device=dev) if arena.W.is_cuda else None

    def step(self, lr=None, k=1, src="G", only_local=False, only_exchanged=False):
        """``k``: the gradient region holds the sum of k gradients (inv_k = 1/k); ``src``: that region ("G", or "R" after the
        exchange); ``only_local`` / ``only_exchanged``: update only the non-exchanged (batch-norm) or only the exchanged groups."""
        a = self.arena
        g = getattr(a, src)
        if a.W.is_cuda:
            from ..ops import cuda_impl
            cuda_impl.lars_trust(a, g, 1.0 / k, self.eta, self._partial, self.norms, self.trust)
            filt = 1 if only_local else (2 if only_exchanged else 0)
            cuda_impl.flat_update(a, "lars", (self.mu, float(bool(self.nesterov)), 1.0 / k), [a.U], g=g, filt=filt, trust=self.trust)
            return
        update = None
        if only_local or only_exchanged:
            update = [m != only_local for m in a.exchanged_mask()]
        trust, norms = ref.lars_flat(a.W, g, a.U, a.offsets, a.sizes, a.group_of, a.group_lr_mult_np, a.group_wd_np,
                                     float(a.hyper[0]) if lr is None else lr, self.mu, self.nesterov, self.eta, 1.0 / k,
                                     update=update, w_half=a.H)
        self.trust.copy_(trust)
        self.norms.copy_(norms)


class FlatLAMB(FlatOptimizer):
    """LAMB (You et al., 2019, "Large Batch Optimization for Deep Learning"): Adam moments (first in the arena's U region, second in
    ``V``, step counter ``t`` in device memory) with decoupled weight decay, r = m̂ / (sqrt(v̂) + eps) + wd·W, and every weight
    tensor's step scaled by its trust ratio ``‖W‖ / ‖r‖``; biases and batch-norm parameters keep ratio 1.  With every ratio 1 it is
    AdamW, not :class:`FlatAdam` (which adds the decay to the gradient).

    On CUDA a step is three launches plus the counter's, all reading only device memory (CUDA-graph capturable, bit-reproducible):
    the moments and the per-block sums of squares of W and r, one per-tensor reduction that writes :attr:`norms` ([n_tensors, 2]:
    ‖W‖, ‖r‖) and :attr:`trust` ([n_tensors]), and the ``flat_update`` pass of the LAMB rule, which recomputes r from the new
    moments.  G is left as it was.  Like LARS, LAMB never runs in the FC weight-gradient GEMM epilogue."""

    rule, buffers = "lamb", ("V",)

    def __init__(self, arena, b1=0.9, b2=0.999, eps=1e-6):
        super().__init__(arena)
        self.b1, self.b2, self.eps = b1, b2, eps
        n, dev = len(arena.sizes), arena.W.device
        self.t = torch.zeros(1, dtype=torch.int64, device=dev)
        self.trust = torch.ones(n, dtype=torch.float32, device=dev)
        self.norms = torch.zeros(n, 2, dtype=torch.float32, device=dev)
        self._partial = torch.zeros(arena.n_blocks, 2, dtype=torch.float32, device=dev) if arena.W.is_cuda else None

    def hyper(self):
        return (self.b1, self.b2, self.eps)

    def step(self, lr=None, k=1, src="G", only_local=False, only_exchanged=False):
        """``k``: the gradient region holds the sum of k gradients (inv_k = 1/k); ``src``: that region ("G", or "R" after the
        exchange); ``only_local`` / ``only_exchanged``: update only the non-exchanged (batch-norm) or only the exchanged groups.
        An ``only_local`` step does not advance :attr:`t`: the ``only_exchanged`` step of the same training step does."""
        a = self.arena
        g = getattr(a, src)
        filt = 1 if only_local else (2 if only_exchanged else 0)
        if a.W.is_cuda:
            from ..ops import cuda_impl
            cuda_impl.lamb_trust(a, g, a.U, self.V, self.t, *self.hyper(), 1.0 / k, filt, self._partial, self.norms, self.trust)
            cuda_impl.flat_update(a, "lamb", self.hyper(), [a.U, self.V], step=self.t, g=g, filt=filt, trust=self.trust)
            return
        update = None
        if filt:
            update = [m != only_local for m in a.exchanged_mask()]
        ref.lamb_flat(a.W, g, a.U, self.V, self.trust, self.norms, a.offsets, a.sizes, a.group_of, a.group_lr_mult_np,
                      a.group_wd_np, float(a.hyper[0]) if lr is None else lr, *self.hyper(), t=int(self.t) + 1, inv_k=1.0 / k,
                      update=update, w_half=a.H)
        if filt != 1:
            self.t += 1

    def state_dict(self):
        return dict(super().state_dict(), t=int(self.t))

    def load_state_dict(self, sd):
        super().load_state_dict(sd)
        self.t.fill_(int(sd["t"]))


# --------------------------------------------------------------------------- classic split (API parity)
def _ex(a):
    return a.exch_vector()


def _set_clip(model, opt, k):
    """``model.grad_clip``: clip the gradient of every step of ``opt`` by its global norm (:meth:`FlatOptimizer.set_grad_clip`);
    ``model.clip_opt`` is then ``opt``, whose skip counter the checkpoints carry.  Only a local k = 1 step has the whole gradient
    before it updates anything."""
    if getattr(model, "grad_clip", None) is None:
        return
    if k != 1:
        raise ValueError("grad_clip needs the global norm of the reduced gradient before any update; it runs on local k = 1 steps only")
    opt.set_grad_clip(model.grad_clip)
    model.clip_opt = opt


def _step_lr(model):
    """The lr argument of a :class:`FlatSGD` step in a closure: the host value of ``shared_lr``, or None under a per-update
    :class:`LrSchedule`, so that the CPU step reads ``arena.hyper[0]`` as the kernel does."""
    return None if getattr(model, "lr_sched", None) is not None else model.shared_lr.get_value()


def _device_lr(model):
    """The lr of a torch expression in a closure: the host value of ``shared_lr``, or under a per-update :class:`LrSchedule`
    ``arena.hyper[0]`` as a device scalar, which the schedule's launch earlier in the step wrote.  A host read there would break
    the capture of a step that runs the closure."""
    return model.arena.hyper[0] if getattr(model, "lr_sched", None) is not None else model.shared_lr.get_value()


def _pre_post_msgd(model, use_nesterov, k, arm=True):
    """BSP_MSGD: aggregate momentum."""
    a, mu = model.arena, (model.mu if model.use_momentum else 0.0)
    sgd = FlatSGD(a, mu, use_nesterov, True)
    _set_clip(model, sgd, k)
    sgd.arm(model, k == 1 and arm)

    def pre():
        lr = _step_lr(model)
        if k == 1:
            sgd.step(lr, 1)
            return
        sgd.step(lr, 1, only_local=True)                      # BN params: full local update
        ex = _ex(a)
        g_eff = a.G + a.wd_vector() * a.W
        a.U.copy_(torch.where(ex, mu * a.U + g_eff, a.U))
        model._send_region = "U"

    def post():
        if k == 1:
            return
        lr = _device_lr(model)
        ex = _ex(a)
        a.W.sub_(torch.where(ex, lr * a.lr_mult_vector() * a.R / float(k), torch.zeros_like(a.W)))
        a.refresh_shadow()

    return pre, post, "U"


def _pre_post_msgd_grad(model, use_nesterov, k, arm=True):
    """_BSP_MSGD: aggregate gradient."""
    a, mu = model.arena, (model.mu if model.use_momentum else 0.0)
    sgd = FlatSGD(a, mu, use_nesterov, True)
    _set_clip(model, sgd, k)
    sgd.arm(model, k == 1 and arm)

    def pre():
        lr = _step_lr(model)
        if k == 1:
            sgd.step(lr, 1)
            return
        sgd.step(lr, 1, only_local=True)
        ex = _ex(a)
        a.G.copy_(torch.where(ex, (a.G + a.wd_vector() * a.W) / float(k), a.G))

    def post():
        if k == 1:
            return
        lr = _device_lr(model)
        ex = _ex(a)
        u_new = mu * a.U + a.R
        step = a.R + mu * u_new if use_nesterov else u_new
        a.U.copy_(torch.where(ex, u_new, a.U))
        a.W.sub_(torch.where(ex, lr * a.lr_mult_vector() * step, torch.zeros_like(a.W)))
        a.refresh_shadow()

    return pre, post, "G"


def _pre_post_sgd(model, k, arm=True):
    a = model.arena
    sgd = FlatSGD(a, 0.0, False, False)
    _set_clip(model, sgd, k)
    sgd.arm(model, k == 1 and arm)

    def pre():
        lr = _step_lr(model)
        if k == 1:
            sgd.step(lr, 1)
            return
        sgd.step(lr, 1, only_local=True)
        ex = _ex(a)
        lr = _device_lr(model)
        a.G.copy_(torch.where(ex, lr * a.lr_mult_vector() * (a.G + a.wd_vector() * a.W) / float(k), a.G))

    def post():
        if k == 1:
            return
        ex = _ex(a)
        a.W.sub_(torch.where(ex, a.R, torch.zeros_like(a.W)))
        a.refresh_shadow()

    return pre, post, "G"


def _pre_post_lars(model, k):
    """LARS, aggregate gradient.  k = 1: the whole step in ``pre``.  k > 1: ``pre`` updates the non-exchanged (batch-norm) groups
    and sends G; ``post`` updates the exchanged groups from R = Σ_ranks G, so the trust ratios come from the averaged gradient."""
    lars = model.lars = FlatLARS(model.arena, model.mu if model.use_momentum else 0.0, model.use_nesterov_momentum, model.lars_eta)

    def pre():
        if k == 1:
            lars.step()
            return
        lars.step(only_local=True)

    def post():
        if k == 1:
            return
        lars.step(k=k, src="R", only_exchanged=True)

    return pre, post, "G"


def _pre_post_lamb(model, k):
    """LAMB, aggregate gradient, as :func:`_pre_post_lars`: k = 1, the whole step in ``pre``; k > 1, ``pre`` updates the batch-norm
    groups and sends G, ``post`` updates the exchanged groups from R = Σ_ranks G and advances the step counter."""
    lamb = model.lamb = FlatLAMB(model.arena)

    def pre():
        if k == 1:
            lamb.step()
            return
        lamb.step(only_local=True)

    def post():
        if k == 1:
            return
        lamb.step(k=k, src="R", only_exchanged=True)

    return pre, post, "G"


def _publish(model, pre, post, send_region, k):
    a = model.arena
    mask = a.exchanged_mask()
    if k > 1:
        model.vels = [v for v, m in zip(a.views(send_region), mask) if m]
        model.vels2 = [v for v, m in zip(a.views("R"), mask) if m]
    else:
        model.vels, model.vels2 = [], []
    model._send_region = send_region
    return pre, post


def BSP_MSGD(model, use_nesterov_momentum, k=1, arm=True):
    return _publish(model, *_pre_post_msgd(model, use_nesterov_momentum, k, arm), k)


def _BSP_MSGD(model, use_nesterov_momentum, k=1, arm=True):
    return _publish(model, *_pre_post_msgd_grad(model, use_nesterov_momentum, k, arm), k)


def BSP_SGD(model, k=1, arm=True):
    return _publish(model, *_pre_post_sgd(model, k, arm), k)


def BSP_LARS(model, k=1):
    return _publish(model, *_pre_post_lars(model, k), k)


def BSP_LAMB(model, k=1):
    return _publish(model, *_pre_post_lamb(model, k), k)


def _clip_paramlist(param_list, scale=10):
    """``T.clip(param,-10,10)`` helper (ref ``opt.py:67-75``; unused there too)."""
    with torch.no_grad():
        for p in param_list:
            p.clamp_(-scale, scale)
    return param_list


def prepare_update_dict(model, k=1, aggregate="momentum", arm=True):
    """``arm``: at k = 1, let the FC weight-gradient GEMMs apply the update of their weights (:meth:`FlatSGD.arm`); only valid
    when the returned ``pre`` is what updates the arena after every backward.  ``model.optimizer == 'lars'`` / ``'lamb'``:
    :func:`BSP_LARS` / :func:`BSP_LAMB`, which never arm."""
    optimizer = getattr(model, "optimizer", "sgd")
    if optimizer == "lars":
        return BSP_LARS(model, k=k)
    if optimizer == "lamb":
        return BSP_LAMB(model, k=k)
    if model.use_momentum:
        if aggregate == "gradient":
            return _BSP_MSGD(model, model.use_nesterov_momentum, k=k, arm=arm)
        return BSP_MSGD(model, model.use_nesterov_momentum, k=k, arm=arm)
    return BSP_SGD(model, k=k, arm=arm)


def pre_model_iter_fn(model, k=1, f_train=True, f_val=True, aggregate="momentum", fused_tail=None):
    """Build ``model.get_vel / descent_vel / train_iter_fn / val_iter_fn``
    (ref ``opt.py:2-52``).  ``get_vel(subb)`` = forward + backward + pre update and
    returns ``(cost, error)``; ``descent_vel()`` = post update.

    When the update is self-contained (k = 1) or a fused exchanger supplies
    ``fused_tail`` (allreduce + SGD in one kernel family) the update is registered as
    the model's *step tail* so it is part of the CUDA-graph-captured step, and
    ``descent_vel`` is a no-op."""
    if f_train:
        pre, post = prepare_update_dict(model, k=k, aggregate=aggregate, arm=fused_tail is None)
        tail = fused_tail if fused_tail is not None else (pre if k == 1 else None)
        model.set_step_tail(tail)

        def get_vel(subb_ind=0):
            cost, err = model.forward_backward(subb_ind)
            if tail is None:
                with torch.no_grad():
                    pre()
            return cost, err

        def descent_vel():
            if tail is None:
                with torch.no_grad():
                    post()

        model.get_vel, model.descent_vel = get_vel, descent_vel
        model.compiled_train_fn_list = [get_vel, descent_vel]
        model.train_iter_fn = choose_iter_fn(model)
    if f_val:
        model.compile_val()
        model.val_iter_fn = model.val_fn


def choose_iter_fn(model):
    """The reference returns ``cdd_iter_fn`` = descent_vel(); get_vel() (one step
    late).  We return get_vel only — the exchanger calls ``descent_vel`` right after
    the collective (see module docstring)."""

    def cdd_iter_fn(subb_ind=0):
        return model.get_vel(subb_ind)

    return cdd_iter_fn
