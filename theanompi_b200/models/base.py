"""Shared machinery behind the model contract.

The reference duplicates ~300 lines of iteration protocol in every model file
(``alex_net.py:300-585``, ``googlenet.py:650-950``, ``cifar10.py:254-493`` …): shared
input buffers + sub-batch slicing, the loader handshake, ``train_iter`` / ``val_iter``
/ ``reset_iter`` / ``adjust_hyperp`` / ``cleanup`` and the compile helpers.
:class:`ModelBase` implements that protocol once; a concrete model only provides
hyper-parameters, its data object and ``build_model()`` / ``forward()``.

Contract exposed (ref ``helper_funcs.py:163-205``, ``README.md:54-67``):
``params`` (list of torch tensors — views into the flat arena), ``data``,
``compile_iter_fns(sync_type)``, ``train_iter(count, recorder)``,
``val_iter(count, recorder)``, ``reset_iter(mode)``, ``adjust_hyperp(epoch)``,
``cleanup()``, ``n_epochs``, ``epoch``, ``n_subb``; plus ``vels``/``vels2``,
``shared_lr``, ``get_vel``/``descent_vel``/``train_iter_fn``/``val_iter_fn``.

H100-native pieces: bf16 NHWC activations with fp32 master weights in the arena;
the whole step (H2D hand-off excluded) can be captured in a CUDA graph
(``config['cuda_graph']``); lr/momentum live in device memory so the graph never
needs re-capture; costs/errors stay on the device until the recorder prints.
"""
from __future__ import annotations

import contextlib
import gc
import math
import time

import numpy as np
import torch

from .. import ops
from ..parallel.arena import FlatArena
from ..utils import nvtx
from ..utils.opt import FlatSGD, LrSchedule, ModelEma, Sam, SharedScalar, pre_model_iter_fn
from .layers2 import BatchNormal, Crop, Dropout, count_params


def pick_device(config):
    dev = config.get("device")
    if dev is not None:
        return torch.device(dev)
    if torch.cuda.is_available():
        return torch.device("cuda", torch.cuda.current_device())
    return torch.device("cpu")


class ModelBase(object):
    # ---- hyper-parameter defaults (override per model)
    n_epochs = 1
    momentum = 0.9
    weight_decay = 0.0
    batch_size = 128
    file_batch_size = 128
    learning_rate = 0.01
    lr_policy = "step"
    lr_step = ()
    lr_gamma = 0.1
    use_momentum = True
    use_nesterov_momentum = False
    input_width = 227
    input_height = 227
    batch_crop_mirror = False
    rand_crop = True
    monitor_grad = False
    bias_lr_mult = 2.0             # biases train with 2x lr in the reference's optimizer (lib/opt.py:181-268)
    graph_safe = True              # False: the step draws host-side randomness / has host control flow → never auto-capture
    supports_grad_clip = True      # config['grad_clip'] (False: the model's step has no clipping pass; refused at compile_iter_fns)
    supports_grad_accum = True     # config['grad_accum'] > 1 (False: the model refuses it at compile_iter_fns)
    supports_lr_schedule = True    # config['lr_schedule'] (False: the model refuses it at compile_iter_fns)
    supports_label_smoothing = True    # config['label_smoothing'] > 0 (False: no classifier head; refused at compile_iter_fns)
    supports_mixup = True          # config['mixup'] (False: no image batch before a first convolution; refused at compile_iter_fns)
    supports_drop_path = False     # config['drop_path_rate'] > 0 (True: residual blocks in self.body that read drop_row(l))
    supports_cifar_augment = False  # config['cifar_augment'] (True: a CIFAR model whose training forward reads train_augment())
    supports_model_ema = True      # config['model_ema'] (False: no single arena updated by the step tail; refused at compile_iter_fns)
    # config['sam'] (False: the step cannot run its training forward twice on the same draws; refused at compile_iter_fns)
    supports_sam = True
    # config['distill'] (True: a native ImageNet classifier whose teacher can be one of the five in ops/distill.py; refused otherwise)
    supports_distill = False
    # True: an ImageNet model fed by ParaLoader, so config['random_resized_crop'], config['color_jitter'] and
    # config['random_erasing'] reach its loader
    # (refused at construction otherwise)
    supports_resized_crop = False
    name = "Model"

    def __init__(self, config):
        self.config = config
        self.verbose = config.get("verbose", False)
        self.rank = config.get("rank", 0)
        self.size = config.get("size", 1)
        self.no_paraload = config.get("no_paraload", False)
        self.device = pick_device(config)
        self.cuda = self.device.type == "cuda"
        # compute precision of the native path: 'bf16' (bf16 operands, fp32 accumulate / master weights) or 'tf32' (fp32 storage
        # end to end, wgmma tf32 — the reference's precision class); see ops/precision.py
        from ..ops import precision
        if config.get("dtype"):
            precision.set_precision(config["dtype"])
        self.precision = precision.precision()
        self.act_dtype = precision.act_dtype() if self.cuda else torch.float32
        # "auto" (default on CUDA): capture the whole step into a CUDA graph, fall back to eager launches if the model's
        # step cannot be captured (host-side control flow, library calls that synchronise, …)
        cg = config.get("cuda_graph", "auto")
        self._graph_auto = (cg == "auto")
        if self._graph_auto and not getattr(self, "graph_safe", True):
            cg = False            # e.g. in-graph random crops drawn from a host RNG every step: a replay would freeze them
        self.use_graph = bool(cg) and self.cuda
        self.epoch = 0
        self.step_idx = 0
        self.mu = self.momentum
        self.eta = self.weight_decay
        # 'sgd' (momentum SGD) or 'lars' (the same with a per-tensor trust ratio, utils/opt.py: FlatLARS) for large global batches,
        # or 'lamb' (Adam moments with per-tensor trust ratios, utils/opt.py: FlatLAMB)
        self.optimizer = config.get("optimizer", "sgd")
        self.lars_eta = float(config.get("lars_eta", 0.001))
        # global gradient-norm clipping of every step (torch.nn.utils.clip_grad_norm_; utils/opt.py: FlatOptimizer.set_grad_clip):
        # the maximum L2 norm of the whole gradient, None (default) = off
        gc = config.get("grad_clip")
        self.grad_clip = None if gc is None else float(gc)
        self.clip_opt = None
        # gradient accumulation: every optimizer step follows grad_accum micro-steps of batch_size samples whose mean gradient builds
        # up in the arena's G region (forward_backward; checked by check_grad_accum)
        self.grad_accum = config.get("grad_accum", 1)
        self.n_updates = 0             # optimizer steps taken (windows completed)
        self.n_discarded = 0           # micro-steps of windows still open at reset_iter('train'), whose gradients were dropped
        self._micro = 0                # micro-steps done in the open window
        # per-update learning-rate schedule (a dict, utils/opt.py: LrSchedule; None = off): a device launch at the start of every
        # update's step writes lr; built by setup_lr_schedule at compile_iter_fns
        self.lr_schedule = config.get("lr_schedule")
        self.lr_sched = None
        # exponential moving average of the weights and batch-norm statistics (a dict, utils/opt.py: ModelEma; None = off): two launches
        # after every update's step tail average W into E; ema_weights() validates, infers and saves with E.  Built by check_model_ema
        self.model_ema = config.get("model_ema")
        self.ema = None
        # sharpness-aware minimization (a dict, utils/opt.py: Sam; None = off): after the step's forward and backward the weights move
        # to the ascent point, a second forward and backward there on the same batch and draws gives the gradient the optimizer steps
        # on, and the weights are restored before it.  Built by check_sam
        self.sam = config.get("sam")
        self.sam_opt = None
        # knowledge distillation from a frozen teacher (a dict, ops/distill.py; None = off): every training step the teacher's eval forward
        # on x_in, after the draws and the mix, gives the loss its soft target.  Built by check_distill
        self.distill = config.get("distill")
        self.distiller = None
        # label smoothing ε of the training loss (cross-entropy against (1 − ε)·onehot + ε / C; 0 = plain NLL); validation stays
        # plain NLL.  Checked by check_label_smoothing at compile_iter_fns
        self.label_smoothing = config.get("label_smoothing", 0.0)
        # Mixup / CutMix of the training batch (a dict, ops/mixup.py; None = off): one draw per training step on the device, the
        # batch mixed at the mix point (mix_input) and the loss taken against the mixed target.  Built by check_mixup
        self.mixup = config.get("mixup")
        self.mixer = None
        # stochastic depth (ops/drop_path.py; 0 = off): one [blocks, batch] table drawn on the device per training step, block l's row
        # scaling its residual branch per sample.  Built by check_drop_path; read through drop_row only during the training forward
        self.drop_path_rate = config.get("drop_path_rate", 0.0)
        self.drop_path = None
        self._drop_on = False
        # pad-and-crop, flip and Cutout of the CIFAR training batch (a dict, ops/cifar_augment.py; None = off): one draw per training
        # step on the device, applied by the model's normalising crop.  Built by check_cifar_augment; read through train_augment only
        # during the training forward
        self.cifar_augment = config.get("cifar_augment")
        self.cifar_aug = None
        self._aug_on = False
        # random-resized crop of the training images (a dict, models/data/utils.py: check_resized_crop; None = off): per-image boxes
        # drawn by the loader and resampled by its kernel on the copy stream.  Checked here because the model's constructor builds
        # the loader; the training step never sees it
        self.resized_crop = self.check_resized_crop(config.get("random_resized_crop"))
        # colour jitter and PCA lighting of the training images (a dict, models/data/utils.py: check_color_jitter; None = off):
        # per-image colour maps drawn by the loader and applied by its crop kernel; like the crop, the training step never sees it
        self.color_jitter = self.check_color_jitter(config.get("color_jitter"))
        # random erasing of the normalised training images (a dict, models/data/utils.py: check_random_erasing; None = off): boxes
        # drawn by the loader and zeroed by one more launch on its copy stream; the training step never sees it
        self.random_erasing = self.check_random_erasing(config.get("random_erasing"))
        # TrivialAugmentWide / RandAugment on the uint8 training crop (a dict, models/data/utils.py: check_auto_augment; None = off):
        # op records drawn by the loader and applied by its kernels on the copy stream; the training step never sees it
        self.auto_augment = self.check_auto_augment(config.get("auto_augment"))
        # test-time views of every validation image (1, 2 or 10; models/data/utils.py: check_val_crops): the loader cuts them all in
        # one launch into a view-major [V, N, ...] batch and val_fn averages the views' softmax.  Checked here because the model's
        # constructor builds the loader; training never sees it
        self.val_crops = self.check_val_crops(config.get("val_crops", 1))
        self.base_lr = np.float32(self.learning_rate)
        self.current_t = self.subb_t = 0
        self.current_v = self.subb_v = 0
        self.last_one_t = self.last_one_v = False
        self.compiled_train_fn_list = []
        self.train_iter_fn = None
        self.val_iter_fn = None
        self._gstream = None
        self._tail = None
        self._graphs = {}              # keyed step graphs (run_keyed_step)
        self._graph_pool = None
        self.exchanger = None         # set by the BSP worker for fused / overlapped exchange
        self.h2d_bytes_last = 0

    # ------------------------------------------------------------------ construction helpers
    def setup_data_parallel(self, data):
        """The 'mini batching and other data parallel common routine' block of every
        reference model (``alex_net.py:73-80``)."""
        self.data = data
        data.batch_data(self.file_batch_size)
        data.extend_data(rank=self.rank, size=self.size)
        data.shuffle_data(mode="train", common_seed=1234)
        data.shuffle_data(mode="val")
        data.shard_data(mode="train", rank=self.rank, size=self.size)
        data.shard_data(mode="val", rank=self.rank, size=self.size)
        self.n_subb = max(1, self.file_batch_size // self.batch_size)

    def finalize(self, params, weight_types, input_shape):
        """Bind parameters into the flat arena and allocate the shared input buffers."""
        self.params, self.weight_types = list(params), list(weight_types)
        count_params(self.params, verbose=False)
        allocator = self.config.get("arena_allocator")
        self.arena = FlatArena(self.params, self.weight_types, self.device, weight_decay=self.eta, bias_lr_mult=self.bias_lr_mult,
                               with_recv=allocator is not None, allocator=allocator,
                               shadow=False if self.precision == "tf32" else self.config.get("_arena_shadow"))
        self.shared_lr = SharedScalar(self.arena.hyper, 0, self.base_lr)
        self.sgd = FlatSGD(self.arena, self.mu, self.use_nesterov_momentum, self.use_momentum)
        B = self.batch_size
        fb = self.file_batch_size
        self.input_shape = tuple(input_shape)           # (B, H, W, C)
        self.shared_x = torch.zeros((fb,) + self.input_shape[1:], dtype=self.act_dtype, device=self.device)
        self.shared_y = torch.zeros((fb,), dtype=torch.int64, device=self.device)
        # val_crops > 1: the view-major [V, fb, ...] validation batch, the loader's ring slot or the serial path's buffer
        self.val_x = None
        self.x_in = torch.zeros((B,) + self.input_shape[1:], dtype=self.act_dtype, device=self.device)
        self.y_in = torch.zeros((B,), dtype=torch.int64, device=self.device)
        # label staging: a small ring of pinned buffers, each guarded by the event of its last H2D copy — the host runs
        # ahead of the device (always under CUDA graphs, and whenever a step is GPU-bound), so a single buffer would be
        # overwritten with the NEXT batch's labels before the copy of the current ones has executed
        self._y_ring = [torch.zeros((fb,), dtype=torch.int64, pin_memory=self.cuda) for _ in range(4 if self.cuda else 1)]
        self._y_ev = [None] * len(self._y_ring)
        self._y_k = 0
        self.vels, self.vels2 = [], []
        if self.verbose:
            print("%s: %d tensors, %.3f M params, arena %.1f MiB on %s"
                  % (self.name, len(self.params), self.arena.n_real / 1e6,
                     self.arena.nbytes / 2 ** 20, self.device))

    # ------------------------------------------------------------------ to be provided by the model
    def build_model(self):
        raise NotImplementedError

    def forward(self, x):
        """Return logits-layer output; must leave ``self.output_layer`` evaluated."""
        raise NotImplementedError

    def loss(self, x, y, label_smoothing=0.0, mix=None, kd=None):
        """(cost, top-1 error, top-5 error); the cost is the mean NLL, or with ``label_smoothing`` ε > 0 the cross-entropy against
        (1 − ε)·onehot + ε / C.  ``mix``: the step's Mixup / CutMix record; the cost is then the cross-entropy against its mixed
        target and the errors count against the label with the larger weight.  ``kd``: the step's distillation target
        (ops/distill.py: KdTarget); the cost is then (1 − α)·that cross-entropy + α·T²·KL(teacher ‖ student) at temperature T."""
        self.forward(x)
        sm = self.output_layer
        return sm.negative_log_likelihood(y, label_smoothing, mix, kd), sm.errors(y), sm.errors_top_x(y)

    # ------------------------------------------------------------------ step functions
    def _fwd_bwd_eager(self):
        # the training loss carries the label smoothing (read on the host here, so a captured step keeps the ε it was captured with);
        # with config['mixup'] the step's draw comes first, keyed by the device step counter, so every graph replay draws anew
        # with config['drop_path_rate'] the table is drawn next (after the mix draw) from the same counter, and only this forward reads
        # it: validation and inference never drop
        # with config['cifar_augment'] the offsets, flips and Cutout boxes are drawn last, from the same counter, and likewise only this
        # forward reads them
        # with config['sam'] the second pass at the ascent point reuses every draw: the step counter only advances in _after_step
        # with config['distill'] the teacher's forward runs last, on the mixed batch, once per step: SAM's second pass reuses its logits
        rec = None
        if self.mixer is not None:
            rec = self.mixer.draw()
            self.mix_input(rec)
        if self.drop_path is not None:
            self.drop_path.draw()
        if self.cifar_aug is not None:
            self.cifar_aug.draw()
        kd = {}
        if self.distiller is not None:
            kd["kd"] = self.distiller.target(self.x_in)
            self._dbg_capture("teacher forward")
        out = self._train_pass(rec, **kd)
        if self.sam_opt is not None:
            with torch.no_grad():
                self.sam_opt.perturb()
            if rec is not None:
                self.repeat_mix(rec)
            with self.bn_stats_frozen():
                self._train_pass(rec, **kd)
            with torch.no_grad():
                self.sam_opt.restore()
            self._dbg_capture("sam")
        return out

    def _train_pass(self, rec, kd=None):
        """Forward and backward of the training step on x_in with the draws of this step already made: the drop-path table and the
        cifar_augment draw are read by the forward, ``rec`` (the Mixup / CutMix record, or None) gives the mixed target, and the
        batch is mixed at the mix point as :meth:`mix_input` left it.  ``kd`` (config['distill']: the teacher's target of this step,
        or None) makes the loss the distillation loss.  The gradient is stored in the arena's G region."""
        self._drop_on = self.drop_path is not None
        self._aug_on = self.cifar_aug is not None
        kw = {} if kd is None else {"kd": kd}
        try:
            if rec is None:
                cost, err, err5 = self.loss(self.x_in, self.y_in, self.label_smoothing, **kw)
            else:
                cost, err, err5 = self.loss(self.x_in, self.y_in, self.label_smoothing, mix=rec, **kw)
        finally:
            self._drop_on = False
            self._aug_on = False
        self._dbg_capture("forward")
        cost.backward()
        return cost.detach(), err.detach()

    def forward_backward(self, subb_ind=0):
        """Forward + backward on sub-batch ``subb_ind`` of the shared input buffer;
        gradients land in the arena's G region.  Returns device scalars (cost, error)."""
        B = self.batch_size
        if self.n_subb == 1 and self.shared_x.shape[0] == B:
            self.x_in.copy_(self.shared_x, non_blocking=True)
            self.y_in.copy_(self.shared_y, non_blocking=True)
        else:
            self.x_in.copy_(self.shared_x[subb_ind * B:(subb_ind + 1) * B], non_blocking=True)
            self.y_in.copy_(self.shared_y[subb_ind * B:(subb_ind + 1) * B], non_blocking=True)
        if self.grad_accum > 1:
            return self._micro_step()
        self.n_updates += 1
        return self.run_keyed_step("step", self._step_body)

    def _step_body(self, kind="step"):
        """Forward + backward of a whole training step (``kind`` 'step') or of a ``grad_accum`` micro-step ('first', 'mid' or
        'last').  The micro kinds run under the accumulate switch (ops.accum): G is stored by 'first' and added to by 'mid' /
        'last', the loss gradient carries 1/n.  The step tail runs after 'step' and 'last'."""
        if kind in ("step", "first"):
            self._schedule_lr()                  # every micro-step of a window trains with the lr of its update
        if kind == "step":
            out = self._fwd_bwd_eager()
        else:
            with ops.accum.mode(kind != "first", float(np.float32(1.0 / self.grad_accum))):
                out = self._fwd_bwd_eager()
        self._dbg_capture("forward+backward (%s)" % kind)
        if kind in ("step", "last") and self._tail is not None:
            with torch.no_grad():
                self._tail()
                if self.ema is not None:
                    self.ema.update()
            self._dbg_capture("step tail")
        self._after_step()
        return out

    # ------------------------------------------------------------------ gradient accumulation
    def micro_step_kind(self):
        """Kind of the next micro-step of a ``grad_accum`` = n window: 'first' (the backward stores G), 'mid' (it adds into G) or
        'last' (it adds into G, then the step tail updates the weights).  n = 2 has no 'mid'."""
        if self._micro == 0:
            return "first"
        return "last" if self._micro == self.grad_accum - 1 else "mid"

    def _micro_step(self):
        """One micro-step on the input buffers, with graphs a replay of the CUDA graph captured for its kind."""
        kind = self.micro_step_kind()
        out = self.run_keyed_step(kind, lambda: self._step_body(kind))
        self._micro += 1
        if kind == "last":
            self._micro = 0
            self.n_updates += 1
        return out

    def check_grad_accum(self, fused_tail=None):
        """Refuse ``grad_accum`` > 1 where it is not implemented: models without it (the LSTM, the GANs, the torch twins), more than
        one worker (BSP, EASGD, GOSGD: the exchange would have to wait for the end of a window) and a fused exchange strategy's
        ``fused_tail`` (its bucket launches fire during every backward)."""
        n = self.grad_accum
        if isinstance(n, bool) or not isinstance(n, (int, np.integer)) or n < 1:
            raise ValueError("%s: grad_accum must be an int >= 1, not %r" % (self.name, n))
        self.grad_accum = n = int(n)
        if n == 1:
            return
        supported = ("grad_accum > 1 runs on one worker (size = 1) with a local optimizer step: AlexNet, GoogLeNet, Cifar10_model, "
                     "VGG16, ResNet50 and Wide_ResNet, with optimizer 'sgd', 'lars', 'lamb' or Wide_ResNet's 'adam', and grad_clip")
        if not self.supports_grad_accum:
            raise ValueError("%s does not accumulate gradients (grad_accum = %d); %s" % (self.name, n, supported))
        if self.size > 1:
            raise ValueError("%s: grad_accum = %d with %d workers is not implemented: the exchange would have to happen once per "
                             "window; %s" % (self.name, n, self.size, supported))
        if fused_tail is not None:
            raise ValueError("%s: grad_accum = %d does not combine with a fused exchange strategy, whose bucket launches fire during "
                             "every backward; %s" % (self.name, n, supported))

    # ------------------------------------------------------------------ label smoothing
    def check_label_smoothing(self):
        """``config['label_smoothing']`` must be a finite real ε in [0, 1] (not a bool), and ε > 0 needs a classifier head; anything
        else is a ValueError that names the key."""
        eps = self.label_smoothing
        ok = not isinstance(eps, bool) and isinstance(eps, (int, float, np.integer, np.floating))
        if not (ok and math.isfinite(eps) and 0.0 <= eps <= 1.0):
            raise ValueError("%s: label_smoothing must be a real number in [0, 1], not %r" % (self.name, eps))
        self.label_smoothing = float(eps)
        if self.label_smoothing and not self.supports_label_smoothing:
            raise ValueError("%s has no classifier head: label_smoothing = %r is not supported; it applies to the softmax "
                             "cross-entropy of AlexNet, GoogLeNet, Cifar10_model, VGG16, ResNet50, Wide_ResNet, the LSTM and their "
                             "torch twins" % (self.name, eps))

    # ------------------------------------------------------------------ Mixup / CutMix
    @property
    def mix_hw(self):
        """(H, W) of the batch at the mix point, the tensor that enters the first convolution: x_in by default."""
        return tuple(self.input_shape[1:3])

    def mix_input(self, rec):
        """Mix this step's batch at the mix point as the record ``rec`` says: x_in, in place.  x_in is refilled from shared_x every
        step; shared_x itself (the loader's buffer, sliced into sub-batches and read by validation) is never mixed."""
        ops.mix_batch(self.x_in, rec)

    def repeat_mix(self, rec):
        """Before a second training forward of the same step (``config['sam']``): mix the mix point again as :meth:`mix_input` did with
        ``rec``.  x_in still holds the mixed batch, so by default there is nothing to do."""

    def check_mixup(self):
        """``config['mixup']`` must be None or a valid dict (ops/mixup.py: check_config; a ValueError names the offending key), and a
        dict needs a model with an image batch before its first convolution; builds the step's :class:`Mixer`."""
        self.mixer = None
        if self.mixup is None:
            return
        from ..ops.mixup import Mixer, check_config
        cfg = check_config(self.mixup)
        if not self.supports_mixup:
            raise ValueError("%s: mixup is not supported; it mixes the image batch of AlexNet, GoogLeNet, Cifar10_model, VGG16, "
                             "ResNet50 and Wide_ResNet" % self.name)
        self.mixer = Mixer(cfg, self.rank, self.mix_hw, self.device)

    # ------------------------------------------------------------------ CIFAR augmentation
    def check_cifar_augment(self):
        """``config['cifar_augment']`` must be None or a valid dict (ops/cifar_augment.py: check_config; a ValueError names the key),
        and a dict needs a model that applies it (``supports_cifar_augment``); builds the step's :class:`CifarAugment`."""
        from ..ops.cifar_augment import KEY, CifarAugment, check_config
        self.cifar_aug = None
        cfg = check_config(self.cifar_augment)
        if cfg is None:
            return
        if not self.supports_cifar_augment:
            raise ValueError("%s: %s is not supported; it augments the CIFAR-10 batch of Wide_ResNet inside its normalising crop"
                             % (self.name, KEY))
        self.cifar_aug = CifarAugment(cfg, self.rank, self.batch_size, self.device)

    def train_augment(self):
        """This training step's :class:`CifarAugment` (its offsets, flips and Cutout boxes already drawn), or None: outside the
        training forward or without cifar_augment."""
        return self.cifar_aug if self._aug_on else None

    # ------------------------------------------------------------------ random-resized crop
    def check_resized_crop(self, cfg):
        """The validated ``config['random_resized_crop']`` (models/data/utils.py: check_resized_crop; a ValueError names the key), or
        None.  A dict needs a model whose ImageNet loader draws a random crop per image: ``supports_resized_crop``, and neither
        ``batch_crop_mirror`` (one crop for the whole batch) nor ``rand_crop = False`` (always the centre crop)."""
        from .data.utils import RRC_KEY, check_resized_crop
        cfg = check_resized_crop(cfg)
        if cfg is None:
            return None
        name = type(self).__name__
        if not self.supports_resized_crop:
            raise ValueError("%s: %s is not supported; it augments the ImageNet loader of AlexNet, GoogLeNet, VGG16, ResNet50, "
                             "ResNet152 and ResNet50Torch" % (name, RRC_KEY))
        if self.batch_crop_mirror or not self.rand_crop:
            raise ValueError("%s: %s draws a random box per image, which contradicts %s" % (
                name, RRC_KEY, "batch_crop_mirror = True" if self.batch_crop_mirror else "rand_crop = False"))
        return cfg

    def check_color_jitter(self, cfg):
        """The validated ``config['color_jitter']`` (models/data/utils.py: check_color_jitter; a ValueError names the key), or None.
        A dict needs a model fed by the ImageNet loader (``supports_resized_crop``); any crop mode composes with it."""
        from .data.utils import CJ_KEY, check_color_jitter
        cfg = check_color_jitter(cfg)
        if cfg is not None and not self.supports_resized_crop:
            raise ValueError("%s: %s is not supported; it augments the ImageNet loader of AlexNet, GoogLeNet, VGG16, ResNet50, "
                             "ResNet152 and ResNet50Torch" % (type(self).__name__, CJ_KEY))
        return cfg

    def check_auto_augment(self, cfg):
        """The validated ``config['auto_augment']`` (models/data/utils.py: check_auto_augment; a ValueError names the key), or None.
        A dict needs a model fed by the ImageNet loader (``supports_resized_crop``) and no ``color_jitter``."""
        from .data.utils import AA_KEY, check_auto_augment
        cfg = check_auto_augment(cfg)
        if cfg is not None and not self.supports_resized_crop:
            raise ValueError("%s: %s is not supported; it augments the ImageNet loader of AlexNet, GoogLeNet, VGG16, ResNet50, "
                             "ResNet152 and ResNet50Torch" % (type(self).__name__, AA_KEY))
        if cfg is not None and self.color_jitter is not None:
            raise ValueError("%s: %s and color_jitter are two different colour recipes (torchvision's clamped uint8 ops against "
                             "fb.resnet.torch's unclamped affine jitter); choose one" % (type(self).__name__, AA_KEY))
        return cfg

    def check_random_erasing(self, cfg):
        """The validated ``config['random_erasing']`` (models/data/utils.py: check_random_erasing; a ValueError names the key), or
        None.  A dict needs a model fed by the ImageNet loader (``supports_resized_crop``); every crop path composes with it."""
        from .data.utils import RE_KEY, check_random_erasing
        cfg = check_random_erasing(cfg)
        if cfg is not None and not self.supports_resized_crop:
            raise ValueError("%s: %s is not supported; it augments the ImageNet loader of AlexNet, GoogLeNet, VGG16, ResNet50, "
                             "ResNet152 and ResNet50Torch" % (type(self).__name__, RE_KEY))
        return cfg

    def check_val_crops(self, v):
        """The validated ``config['val_crops']`` (models/data/utils.py: check_val_crops; a ValueError names the key).  A value other
        than 1 needs a model fed by the ImageNet loader (``supports_resized_crop``)."""
        from .data.utils import VC_KEY, check_val_crops
        v = check_val_crops(v)
        if v != 1 and not self.supports_resized_crop:
            raise ValueError("%s: %s = %d is not supported; multi-crop validation runs on the ImageNet loader of AlexNet, GoogLeNet, "
                             "VGG16, ResNet50, ResNet152 and ResNet50Torch" % (type(self).__name__, VC_KEY, v))
        return v

    # ------------------------------------------------------------------ stochastic depth (drop-path)
    def check_drop_path(self):
        """``config['drop_path_rate']`` must be a finite real p in [0, 1) (ops/drop_path.py: check_rate; a ValueError names the key),
        and p > 0 needs a model with residual blocks (``supports_drop_path``); builds the step's :class:`DropPath` over the
        ``len(self.body)`` blocks."""
        from ..ops.drop_path import KEY, DropPath, check_rate
        self.drop_path = None
        p = self.drop_path_rate = check_rate(self.drop_path_rate)
        if p == 0.0:
            return
        if not self.supports_drop_path:
            raise ValueError("%s: %s = %r is not supported; drop-path scales the residual blocks of ResNet50, ResNet152 and "
                             "Wide_ResNet" % (self.name, KEY, p))
        self.drop_path = DropPath(p, len(self.body), self.batch_size, self.rank, self.device)

    def drop_row(self, l):
        """Block l's row of this training step's drop-path table (fp32, one scale per sample), or None: outside the training
        forward, without drop_path_rate, or where p_l = 0."""
        return self.drop_path.row(l) if self._drop_on else None

    # ------------------------------------------------------------------ per-update learning-rate schedule
    @property
    def updates_per_epoch(self):
        """Optimizer updates in one epoch of this worker: its train batches × sub-batches, over the gradient-accumulation window."""
        return self.data.n_batch_train * self.n_subb // self.grad_accum

    def setup_lr_schedule(self):
        """Build ``config['lr_schedule']`` (:class:`LrSchedule`, peak = the model's learning_rate, total_steps by default
        n_epochs × :attr:`updates_per_epoch`); a malformed dict, or a model that does not support a schedule, is a ValueError."""
        self.lr_sched = None
        if self.lr_schedule is None:
            return
        if not self.supports_lr_schedule:
            raise ValueError("%s: lr_schedule is not supported; it runs on AlexNet, GoogLeNet, Cifar10_model, VGG16, ResNet50, "
                             "Wide_ResNet and the LSTM" % self.name)
        self.lr_sched = LrSchedule(self.arena, self.lr_schedule, self.learning_rate, int(self.n_epochs) * self.updates_per_epoch)

    def _schedule_lr(self):
        """The first launch of a step that starts an update: lr(u) into arena.hyper[0] before anything reads it."""
        if self.lr_sched is not None:
            self.lr_sched.step()

    def _report_lr(self, dropped=False):
        """Once per epoch, at reset_iter('train'): the host copy of shared_lr (recorder, lr_<epoch>.npy, checkpoints, prints) takes
        the lr of the epoch's last update, read from the device once.  After a ``dropped`` window arena.hyper[0] holds the dropped
        window's lr, so the host evaluates the last update's (``reference.lr_at``) from the update index instead."""
        if self.lr_sched is None:
            return
        u = int(self.lr_sched.u) if dropped else 0
        self.shared_lr.mirror(self.lr_sched.lr_at(u - 1) if u > 0 else self.lr_sched.value())

    def _dbg_capture(self, where):
        """TMPI_DEBUG_CAPTURE=1: name the stage that invalidated an ongoing CUDA-graph capture."""
        import os
        if not self.cuda or os.environ.get("TMPI_DEBUG_CAPTURE") != "1":
            return
        from ..ops import native
        err, status = native.require().capture_status(torch.cuda.current_stream(self.device).cuda_stream)
        if err != 0 or status == 2:
            raise RuntimeError("CUDA graph capture invalidated during %s (err %d status %d)" % (where, err, status))

    def _after_step(self):
        if self.cuda:
            from ..ops import cuda_impl
            cuda_impl.advance_step(self.device)
        else:
            ops.advance_rng_step()

    def run_keyed_step(self, key, body):
        """Run ``body()`` — a whole training step that reads only static buffers — as a replay of the CUDA graph captured for
        ``key`` (any hashable: a step kind, a sequence-length bucket, ...).  Without graphs (CPU, ``cuda_graph=False``) ``body`` runs
        eagerly.  Per key: two eager warm-up runs on the capture stream, then the capture, then replays.  All keys share one
        capture stream and one graph memory pool: only one graph of a model replays at a time.  A replay overwrites the graph's
        outputs (a tensor or a tuple of scalars), so it returns copies, made by one launch.

        Under ``cuda_graph='auto'`` a capture that fails turns graphs off for every key, and the step runs eagerly.  With a fused
        exchange on more than one rank the ranks agree on it first, so that either all of them replay or all run eagerly."""
        if not self.use_graph:
            return body()
        if self._gstream is None:
            self._gstream = torch.cuda.Stream(device=self.device)
            self._graph_pool = torch.cuda.graph_pool_handle()
        st = self._graphs.setdefault(key, {"warm": 0, "graph": None, "out": None})
        if st["graph"] is None:
            s, cur = self._gstream, torch.cuda.current_stream(self.device)
            s.wait_stream(cur)
            if st["warm"] < 2:
                # Eager warm-up ON THE CAPTURE STREAM: autograd caches each leaf's AccumulateGrad node together
                # with the stream that was current when it was first built; if that were the default stream the
                # engine would make the capturing stream wait on uncaptured work at the end of backward
                # (cudaErrorStreamCaptureIsolation).
                st["warm"] += 1
                with torch.cuda.stream(s):
                    out = body()
                cur.wait_stream(s)
                return out
            g, inner, why = torch.cuda.CUDAGraph(), None, ""
            # No automatic garbage collection while capturing: a collection could finalise an unreachable model (a reference
            # cycle) whose CUDA graph, events or pinned buffers are released by calls a capturing thread must not make, which
            # invalidates the capture.  The garbage is collected after it.
            gc_on = gc.isenabled()
            gc.disable()
            try:
                with torch.cuda.stream(s), torch.cuda.graph(g, pool=self._graph_pool, stream=s, capture_error_mode="thread_local"):
                    try:
                        out = body()
                    except BaseException as e:       # capture_end would mask it with "invalidated"
                        inner = e
                        raise
            except Exception as e:  # noqa: BLE001
                err = e if inner is None else inner
                if not self._graph_auto or not isinstance(err, Exception):
                    raise err
                why = "%s: %s" % (type(err).__name__, str(err)[:200])
            finally:
                if gc_on:
                    gc.enable()
            cur.wait_stream(s)
            ex = self.exchanger
            fused = ex is not None and getattr(ex, "fused", False)
            ok = not why
            if fused and getattr(ex, "size", 1) > 1:
                # the fused exchange pairs device-side barriers by launch order: either every rank replays the graph or
                # every rank runs eager — agree on it (a capture that failed on one rank only would desynchronise them)
                ok = all(ex.comm.allgather(ok))
            if not ok:
                print("[%s] CUDA-graph capture of the %r step failed (%s) — running eager" % (self.name, key, why or "on another rank"))
                self.use_graph = False
                self._graphs = {}
                if fused and hasattr(ex, "_reset_pending"):
                    ex._reset_pending()          # a half-captured step consumed some grad-ready callbacks
                torch.cuda.synchronize()
                return body()
            st["graph"], st["out"] = g, out
        st["graph"].replay()
        out = st["out"]
        return torch.stack(out).unbind() if isinstance(out, tuple) else out.clone()

    def captured_steps(self):
        """The keys of :meth:`run_keyed_step` that replay a captured CUDA graph: 'step' (a training step), a micro-step kind, an
        LSTM bucket length, ..."""
        return {k for k, st in self._graphs.items() if st["graph"] is not None}

    @property
    def _graph(self):
        """The captured graph of the training step (key 'step'), or None; read-only, for code that inspected it before
        :meth:`captured_steps`."""
        st = self._graphs.get("step")
        return None if st is None else st["graph"]

    def set_step_tail(self, fn):
        """Register work that runs right after backward as part of the step — and
        therefore *inside* the captured CUDA graph: the local fused SGD (k = 1) or the
        fused allreduce+SGD exchange kernels (k > 1)."""
        self._tail = fn
        self._graphs = {}

    def compile_val(self):
        def val_fn(subb_ind=0):
            B = self.batch_size
            x = self.shared_x[subb_ind * B:(subb_ind + 1) * B]
            y = self.shared_y[subb_ind * B:(subb_ind + 1) * B]
            with torch.no_grad():
                c, e, e5 = self.loss(x, y)
            return c, e, e5

        def multi_view_val_fn(subb_ind=0):
            # val_crops = V > 1: V forwards on the views of the sub-batch, each followed by view_softmax_accum on the main head's
            # logits (the last one also reduces the metrics: V + 1 launches besides the forwards); the CPU runs the reference
            B, V = self.batch_size, self.val_crops
            y = self.shared_y[subb_ind * B:(subb_ind + 1) * B]
            with torch.no_grad():
                if not self.cuda:
                    logits = []
                    for v in range(V):
                        self.forward(self.val_x[v, subb_ind * B:(subb_ind + 1) * B])
                        logits.append(self.output_layer.logits)
                    return ops.reference.multi_view_xent(logits, y, torch.float32)[:3]
                from ..ops import cuda_impl
                acc = None
                for v in range(V):
                    self.forward(self.val_x[v, subb_ind * B:(subb_ind + 1) * B])
                    lg = self.output_layer.logits
                    if acc is None:
                        acc = torch.empty(tuple(lg.shape), dtype=torch.float32, device=self.device)
                    out = cuda_impl.view_softmax_accum(lg, y, acc, v, V)
            return out
        self.val_fn = val_fn if self.val_crops == 1 else multi_view_val_fn

    def compile_inference(self):
        def inf_fn(x):
            with torch.no_grad():
                Dropout.SetDropoutOff(); Crop.SetRandCropOff(); BatchNormal.SetTrainOff()
                out = torch.softmax(self.forward(x).float(), dim=1)
                Dropout.SetDropoutOn(); Crop.SetRandCropOn(); BatchNormal.SetTrainOn()
            return out
        self.inf_fn = inf_fn

    def compile_train(self, *args):
        self.compiled_train_fn_list.extend(args)

    def compile_iter_fns(self, sync_type="avg", aggregate="momentum", fused_tail=None):
        """``sync_type='cdd'``: split step (get_vel / exchange / descent_vel);
        ``'avg'``: self-contained local update (k = 1), the exchanger then averages
        weights.  Fixes SURVEY §2.9 #5/#7: every model accepts ``sync_type`` and 'avg'
        really updates.

        ``optimizer='lars'`` and ``'lamb'`` need each tensor's whole reduced gradient before they update any of its elements, so
        they run on the split strategies (``ar``, ``nccl32``, ``nccl16``, ``asa32``, ``p2p32``, …) and not on a fused exchange
        (``fused_tail``).

        ``grad_clip`` needs the global norm of the whole gradient before any element is updated: it runs on local k = 1 steps only
        (see :meth:`check_grad_clip`)."""
        if self.optimizer not in ("sgd", "lars", "lamb"):
            raise ValueError("%s: optimizer must be 'lamb', 'sgd' or 'lars', not %r" % (self.name, self.optimizer))
        k = self.size if sync_type == "cdd" else 1
        self.setup_train_options(k, fused_tail)
        start = time.time()
        self.sync_type = sync_type
        if k > 1 and fused_tail is None:
            _ = self.arena.R                      # allocate the receive region
        pre_model_iter_fn(self, k, aggregate=aggregate, fused_tail=fused_tail)
        if self.ema is not None and k > 1:
            # BSP 'cdd' over a split strategy: W is the same on every rank once post() has run, so the average follows it there
            post = self.descent_vel

            def descent_vel():
                post()
                with torch.no_grad():
                    self.ema.update()
            self.descent_vel = descent_vel
            self.compiled_train_fn_list = [self.get_vel, descent_vel]
        if self.verbose:
            print("Compile time: %.3f s" % (time.time() - start))

    def setup_train_options(self, k=1, fused_tail=None, optimizer=None):
        """Check and build the training options of the config for a step of ``k`` workers (k > 1: BSP ``sync_type='cdd'``),
        ``fused_tail`` (a fused exchange strategy's step tail, or None) and ``optimizer`` (default: the model's): grad_accum,
        label_smoothing, mixup, cifar_augment, drop_path_rate, lr_schedule, grad_clip, model_ema, sam and distill.  A model refuses every
        option it does not support here, with a ValueError that names it."""
        self.check_grad_accum(fused_tail)
        self.check_label_smoothing()
        self.check_mixup()
        self.check_cifar_augment()
        self.check_drop_path()
        self.setup_lr_schedule()
        opt = self.optimizer if optimizer is None else optimizer
        if opt in ("lars", "lamb") and fused_tail is not None:
            raise ValueError("optimizer=%r needs every tensor's whole reduced gradient before its update; the fused exchange "
                             "strategies (fused*, oneshot*, twoshot*, nvls*, fused_rs) update bucket slices as they are reduced. "
                             "Use a split strategy: ar, nccl32, nccl16, asa32, asa16 or p2p32" % opt)
        self.check_grad_clip(k, fused_tail, opt)
        self.check_model_ema(k, fused_tail)
        self.check_sam(fused_tail)
        self.check_distill()

    def check_distill(self):
        """``config['distill']`` must be None or a valid dict (ops/distill.py: check_config; a ValueError names the key), on a model that
        supports it (``supports_distill``).  Builds the teacher (:class:`ops.distill.Distill`) from its class and checkpoint, after this
        model is finalised: a teacher class, input or class count that does not fit, or a checkpoint that is missing or does not match the
        teacher's layout, is a ValueError that names the key.  The key changes only the loss of the training step, so every optimizer,
        training option and exchange strategy runs with it."""
        self.distiller = None
        if self.distill is None:
            return
        from ..ops.distill import KEY, Distill, check_config
        cfg = check_config(self.distill)
        if not self.supports_distill:
            raise ValueError("%s: %s is not supported; the students and teachers are the native ImageNet classifiers AlexNet, GoogLeNet, "
                             "VGG16, ResNet50 and ResNet152" % (self.name, KEY))
        self.distiller = Distill(self, cfg)

    def check_sam(self, fused_tail=None):
        """``config['sam']`` must be None or a valid dict (utils/opt.py: Sam.check_config; a ValueError names the key).  A dict needs a
        model that can run its training forward twice on the same draws (``supports_sam``), ``grad_accum`` = 1 (the ascent step needs
        the whole window's gradient) and no ``fused_tail`` (a fused exchange strategy's bucket launches would fire during the first
        backward).  Each worker perturbs by its own gradient (m-sharpness, m = its batch): one worker, BSP 'avg' or 'cdd' over a split
        strategy, EASGD, ASGD and GOSGD.  Builds :class:`Sam`."""
        self.sam_opt = None
        if self.sam is None:
            return
        key = Sam.KEY
        cfg = Sam.check_config(self.sam)
        supported = ("%s runs on AlexNet, GoogLeNet, VGG16, ResNet50, ResNet152 and Wide_ResNet with grad_accum = 1: on one worker, BSP "
                     "sync_type='avg' or 'cdd' over a split strategy (ar, nccl32, nccl16, asa32, asa16, p2p32), EASGD, ASGD or GOSGD" % key)
        if not self.supports_sam:
            raise ValueError("%s: %s is not supported; %s" % (self.name, key, supported))
        if self.grad_accum > 1:
            raise ValueError("%s: %s does not combine with grad_accum = %d: the ascent step needs the gradient of the whole window; %s"
                             % (self.name, key, self.grad_accum, supported))
        if fused_tail is not None:
            raise ValueError("%s: %s does not combine with a fused exchange strategy, whose bucket launches would fire during the first "
                             "backward; %s" % (self.name, key, supported))
        self.sam_opt = Sam(self.arena, cfg)

    @property
    def sam_norm(self):
        """n = ‖g‖ (ASAM: ‖|w|⊙g‖) of the last training step's first gradient (``config['sam']``; a device scalar, NaN or Inf when the
        weights were not moved), or None without the key."""
        return None if self.sam_opt is None else self.sam_opt.norm

    @contextlib.contextmanager
    def bn_stats_frozen(self):
        """Inside the block this model's batch-norm layers still normalise with batch statistics in training mode, but do not update
        their running mean and variance (SAM's second pass)."""
        layers = self._bn_layers()
        for l in layers:
            l.update_stats = False
        try:
            yield
        finally:
            for l in layers:
                l.update_stats = True

    def check_model_ema(self, k=1, fused_tail=None):
        """``config['model_ema']`` must be None or a valid dict (utils/opt.py: ModelEma.check_config; a ValueError names the key).  A
        dict needs a model whose step tail updates one arena (``supports_model_ema``), on one worker or on BSP ``sync_type='cdd'`` over a
        split strategy (``k`` = the number of workers, no ``fused_tail``): elsewhere the weights change after the step, in the exchange
        (BSP 'avg', EASGD, ASGD, GOSGD), or non-owners' fp32 masters are stale (the fused strategies).  Builds :class:`ModelEma`, whose
        average starts from the weights and statistics as they are now."""
        self.ema = None
        if self.model_ema is None:
            return
        key = ModelEma.KEY
        cfg = ModelEma.check_config(self.model_ema)
        supported = ("%s runs on AlexNet, GoogLeNet, Cifar10_model, VGG16, ResNet50, ResNet152 and Wide_ResNet, on one worker or on BSP "
                     "sync_type='cdd' over a split strategy (ar, nccl32, nccl16, asa32, asa16, p2p32)" % key)
        if not self.supports_model_ema:
            raise ValueError("%s: %s is not supported; %s" % (self.name, key, supported))
        if self.size > 1 and fused_tail is not None:
            raise ValueError("%s: %s does not combine with a fused exchange strategy on %d workers, whose non-owners' fp32 master weights "
                             "are stale; %s" % (self.name, key, self.size, supported))
        if self.size > 1 and k != self.size:
            raise ValueError("%s: %s needs the same updated weights on every worker after the step; with BSP sync_type='avg', EASGD, "
                             "ASGD or GOSGD on %d workers they change in the exchange; %s" % (self.name, key, self.size, supported))
        self.ema = ModelEma(self.arena, self._bn_layers, cfg)

    @contextlib.contextmanager
    def ema_weights(self):
        """Inside the block the model's weights W, their bf16 shadow and its batch-norm running statistics are the moving average E
        (``config['model_ema']``), so that ``val_iter``, ``inf_fn`` and ``save_weights`` run on the averaged model; on exit all three
        are restored bit for bit.  One ``ema_swap`` launch each way."""
        if self.ema is None:
            raise RuntimeError("%s: ema_weights() needs config['model_ema'] and compile_iter_fns()" % self.name)
        self.ema.swap()
        try:
            yield
        finally:
            self.ema.swap()

    def check_grad_clip(self, k=1, fused_tail=None, optimizer=None):
        """Refuse ``grad_clip`` where the native step cannot clip by the global norm: with ``optimizer`` (default: the model's)
        'lars' or 'lamb', whose trust ratios already normalise every tensor's step, and on any step that is not a local k = 1
        update (BSP ``sync_type='cdd'`` with more than one worker, a fused exchange strategy's ``fused_tail``), which would need
        the norm of the reduced gradient before any slice is updated."""
        if self.grad_clip is None:
            return
        if not self.supports_grad_clip:
            raise ValueError("%s: grad_clip is not supported by the torch twins; it runs on the native models (AlexNet, GoogLeNet, "
                             "Cifar10_model, VGG16, ResNet50, Wide_ResNet, LSTM, NativeWGAN, NativeLSGAN)" % self.name)
        supported = ("grad_clip runs on the local k = 1 steps of the sgd, adam, rmsprop, adadelta and rmsprop_centered flat "
                     "optimizers: one worker, BSP sync_type='avg' with a split strategy, EASGD, ASGD or GOSGD")
        if not self.grad_clip > 0:
            raise ValueError("%s: grad_clip must be a positive maximum norm or None, not %r" % (self.name, self.grad_clip))
        opt = self.optimizer if optimizer is None else optimizer
        if opt in ("lars", "lamb"):
            raise ValueError("%s: grad_clip does not combine with optimizer=%r, whose trust ratios already normalise every "
                             "tensor's step; %s" % (self.name, opt, supported))
        if fused_tail is not None or k > 1:
            raise ValueError("%s: grad_clip needs the global norm of the reduced gradient before any update, which %s does not "
                             "have; %s" % (self.name, "a fused exchange strategy" if fused_tail is not None
                                           else "sync_type='cdd' with %d workers" % k, supported))

    # ------------------------------------------------------------------ data movement
    def _labels_to_device(self, labels):
        n = len(labels)
        k = self._y_k
        self._y_k = (k + 1) % len(self._y_ring)
        if self._y_ev[k] is not None:
            self._y_ev[k].synchronize()
        buf = self._y_ring[k]
        buf[:n] = torch.as_tensor(np.asarray(labels, dtype=np.int64))
        self.shared_y[:n].copy_(buf[:n], non_blocking=True)
        if self.cuda:
            if self._y_ev[k] is None:
                self._y_ev[k] = torch.cuda.Event()
            self._y_ev[k].record(torch.cuda.current_stream(self.device))
        return n * 8

    def _load_file_batch(self, mode, idx, img, labels, n_batches):
        """Loader handshake (ref ``alex_net.py:394-448``): request the next file,
        wait for the current one, put labels on the device."""
        loader = getattr(self.data, "loader", None)
        last = idx == n_batches - 1
        nbytes = 0
        if loader is not None:
            if idx == 0:
                # a new pass over the files: first consume the look-ahead issued for the last file of the previous pass, as
                # reset_iter does.  Left outstanding, every later get() would return the batch one request behind its labels, and
                # with two requests in flight the loader would refill the ring slot the trainer is still reading
                loader.drain()
                loader.set_mode(mode)
                loader.request(img[idx], mode)
            loader.request(img[idx + 1] if not last else img[idx], mode)
            b = loader.get()
            if b.x.dim() == 5:                   # val_crops > 1: the view-major validation batch
                self.val_x = b.x
            else:
                self.shared_x = b.x
            nbytes += b.h2d_bytes
        else:
            x = self.data.load_batch(img[idx], mode, self)
            if x.dim() == 5:
                if self.val_x is None:
                    self.val_x = torch.zeros((x.shape[0], self.file_batch_size) + self.input_shape[1:], dtype=self.act_dtype,
                                             device=self.device)
                self.val_x[:, :x.shape[1]].copy_(x.to(self.act_dtype), non_blocking=True)
            else:
                self.shared_x[:x.shape[0]].copy_(x.to(self.act_dtype), non_blocking=True)
            nbytes += x.numel() * x.element_size()
        nbytes += self._labels_to_device(labels[idx])
        self.h2d_bytes_last = nbytes
        return last

    # ------------------------------------------------------------------ the contract
    def reset_iter(self, mode):
        if mode == "train":
            self.current_t = self.subb_t = 0
            self.last_one_t = False
            # a gradient-accumulation window still open at the end of the epoch is dropped: the next micro-step is a 'first' again,
            # which overwrites G; it gives its update index back to the schedule, so the next window trains with the same lr
            dropped = self._micro > 0 and self.lr_sched is not None
            if dropped:
                self.lr_sched.give_back()
            self.n_discarded += self._micro
            self._micro = 0
            self._report_lr(dropped)
        else:
            self.current_v = self.subb_v = 0
            self.last_one_v = False
        loader = getattr(self.data, "loader", None)
        if loader is not None:
            loader.drain()       # the one look-ahead request issued for the last file

    def train_iter(self, count, recorder):
        if self.current_t == 0 and self.subb_t == 0:
            self.data.shuffle_data(mode="train", common_seed=self.epoch)
            self.data.shard_data(mode="train", rank=self.rank, size=self.size)
        img, labels = self.data.train_img_shard, self.data.train_labels_shard
        if self.subb_t == 0:
            recorder.start()
            with nvtx.range("load"):
                self.last_one_t = self._load_file_batch("train", self.current_t, img, labels,
                                                        self.data.n_batch_train)
            recorder.end("wait")
        recorder.start()
        with nvtx.range("train_iter_fn"):
            cost, error = self.train_iter_fn(self.subb_t)
        recorder.train_error(count, cost, error)
        recorder.end("calc")
        if self.monitor_grad and self.verbose:
            print(self.grad_norms())
        if (self.subb_t + 1) // self.n_subb == 1:
            self.current_t = 0 if self.last_one_t else self.current_t + 1
            self.subb_t = 0
        else:
            self.subb_t += 1
        self.step_idx += 1

    def val_iter(self, count, recorder):
        if self.current_v == 0 and self.subb_v == 0:
            self.data.shuffle_data(mode="val")
            self.data.shard_data(mode="val", rank=self.rank, size=self.size)
        img, labels = self.data.val_img_shard, self.data.val_labels_shard
        if self.subb_v == 0:
            self.last_one_v = self._load_file_batch("val", self.current_v, img, labels,
                                                    self.data.n_batch_val)
        Dropout.SetDropoutOff(); Crop.SetRandCropOff(); BatchNormal.SetTrainOff()
        cost, error, error_top5 = self.val_iter_fn(self.subb_v)
        Dropout.SetDropoutOn(); Crop.SetRandCropOn(); BatchNormal.SetTrainOn()
        recorder.val_error(count, cost, error, error_top5)
        if (self.subb_v + 1) // self.n_subb == 1:
            self.current_v = 0 if self.last_one_v else self.current_v + 1
            self.subb_v = 0
        else:
            self.subb_v += 1

    def adjust_hyperp(self, epoch):
        """Once per epoch (ref ``alex_net.py:569-579``, ``googlenet.py:925-945``).  A per-update ``lr_schedule`` owns lr: nothing
        changes here."""
        if self.lr_sched is not None:
            return
        if self.lr_policy == "step":
            if epoch in self.lr_step:
                self.shared_lr.set_value(np.float32(self.shared_lr.get_value() * self.lr_gamma))
        elif self.lr_policy == "poly":
            power = getattr(self, "lr_power", 0.5)
            self.shared_lr.set_value(np.float32(self.base_lr * (1.0 - float(epoch + 1) / self.n_epochs) ** power))
        elif self.lr_policy == "auto":
            pass

    def scale_lr(self, size):
        self.shared_lr.set_value(np.float32(self.shared_lr.get_value() * size))

    def grad_norms(self):
        """L2 grad-norm monitor (ref ``alex_net.py:311-320``): (sum, max) of log10 norms."""
        armed = [p for p in self.arena.params if getattr(p, "sgd_epilogue", None) is not None]
        if armed:
            # their wgrad GEMMs apply the update instead of writing G (utils/opt.py: FlatSGD.arm)
            raise RuntimeError("grad_norms(): %d weights are updated in their wgrad GEMM epilogue and have no gradient in G; set "
                               "monitor_grad = True before compile_iter_fns()" % len(armed))
        norms = torch.stack([g.float().norm() for g in self.arena.views("G")]).clamp_min(1e-30).log10()
        return [float(norms.sum()), float(norms.max())]

    # ------------------------------------------------------------------ checkpoint extras (non-parameter state)
    def _bn_layers(self):
        return [l for l in (getattr(self, "layers", None) or []) if isinstance(l, BatchNormal)]

    def extra_state(self):
        """Batch-norm running statistics (not parameters, so not in the arena) and the LAMB second moment and step counter (its
        first moment is the arena's U region)."""
        sd = {"bn": [(l.running_mean.detach().cpu(), l.running_var.detach().cpu()) for l in self._bn_layers()]}
        if getattr(self, "lamb", None) is not None:
            sd["lamb"] = self.lamb.state_dict()
        if self.clip_opt is not None:                   # the SGD step's skip counter (gradient clipping)
            sd["grad_clip"] = self.clip_opt.state_dict()
        if self.lr_sched is not None:                   # the update index of the lr schedule
            sd["lr_schedule"] = self.lr_sched.state_dict()
        if self.ema is not None:                        # the moving average and its counters
            sd["model_ema"] = self.ema.state_dict()
        return sd

    def load_extra_state(self, sd):
        for l, (m, v) in zip(self._bn_layers(), sd.get("bn", [])):
            l.running_mean = m.to(self.device).clone()
            l.running_var = v.to(self.device).clone()
        if "lamb" in sd and getattr(self, "lamb", None) is not None:
            self.lamb.load_state_dict(sd["lamb"])
        if "grad_clip" in sd and self.clip_opt is not None:
            self.clip_opt.load_state_dict(sd["grad_clip"])
        if "lr_schedule" in sd and self.lr_sched is not None:
            self.lr_sched.load_state_dict(sd["lr_schedule"])
        if "model_ema" in sd and self.ema is not None:
            self.ema.load_state_dict(sd["model_ema"])

    def cleanup(self):
        if getattr(self.data, "para_load", False) and hasattr(self.data, "para_load_close"):
            self.data.para_load_close()
