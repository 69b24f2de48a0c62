"""Autograd-aware functional ops.

Each op dispatches on the device of its input:

* CUDA  → :mod:`theanompi_b200.ops.cuda_impl` (hand-written sm_90a kernels from
  ``csrc/``; hard error when the extension is missing),
* CPU   → :mod:`theanompi_b200.ops.reference` (plain torch, fp32).

Weight gradients do not travel through autograd's AccumulateGrad: when a
parameter carries a ``gbuf`` attribute (a view into the flat gradient arena, see
:class:`theanompi_b200.parallel.arena.FlatArena`) the backward kernel writes the
fp32 gradient straight into it and then fires ``on_ready`` — that callback is
what lets the BSP exchanger launch the fused allreduce+SGD kernel for a bucket
on a side stream while backward is still running on the main stream
(the reference is strictly sequential, ``theanompi/worker.py:94-97``).

Under gradient accumulation (:mod:`.accum`) the kernels add into those views and the CPU path adds in :func:`_sink`.
"""
from __future__ import annotations

import torch

import os

from . import accum
from . import reference as ref


def _impl(x):
    if x.is_cuda:
        from . import cuda_impl
        return cuda_impl
    return ref


def compute_weight(p):
    """bf16 shadow of a master parameter when one exists (GPU), else itself."""
    sh = getattr(p, "shadow", None)
    return sh if sh is not None else p


def _sink(p, grad):
    """Deliver a parameter gradient. Returns what autograd should see."""
    if p is None or grad is None and getattr(p, "gbuf", None) is None:
        return None
    gbuf = getattr(p, "gbuf", None)
    if gbuf is None:
        return grad.to(p.dtype).view_as(p)
    if grad is not None and grad.data_ptr() != gbuf.data_ptr():
        if getattr(p, "gaccum", False) or accum.accumulating():
            gbuf.add_(grad.view_as(gbuf))
        else:
            gbuf.copy_(grad.view_as(gbuf))
    cb = getattr(p, "on_ready", None)
    if cb is not None:
        cb(p)
    return None


def _gout(p):
    """Output buffer the backward kernel may write the fp32 grad into directly."""
    if getattr(p, "gaccum", False):
        return None
    return getattr(p, "gbuf", None)


# --------------------------------------------------------------------------- linear
class _LinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, relu):
        impl = _impl(x)
        wc = compute_weight(w)
        y = impl.linear_bias_act(x, wc, b, relu)
        ctx.save_for_backward(x, y)
        ctx.w, ctx.b, ctx.relu = w, b, relu
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors
        w, b = ctx.w, ctx.b
        impl = _impl(x)
        wc = compute_weight(w)
        need_dx = ctx.needs_input_grad[0]
        if impl is ref:
            dx, dw, db = ref.linear_bias_act_bwd(x, wc, y, dy, ctx.relu, need_dx)
        else:
            dx, dw, db = impl.linear_bias_act_bwd(x, wc, y, dy, ctx.relu, need_dx,
                                                  dw_out=_gout(w), db_out=_gout(b),
                                                  sgd_param=w if getattr(w, "sgd_epilogue", None) is not None else None)
        gb = _sink(b, db)
        gw = _sink(w, dw)
        return dx, gw, gb, None


def linear_bias_act(x, w, b, relu=True):
    return _LinearFn.apply(x, w, b, relu)


# --------------------------------------------------------------------------- conv
def _fused_pool_ok(x, relu, pool):
    """conv(+ReLU) → max-pool blocks run their backward through ONE fused kernel (pool scatter + ReLU mask + bias grad)."""
    # (bf16 path only: the fused kernel works on packed bf16 lanes; the fp32 / tf32 path runs pool-backward and ReLU-mask +
    # bias-gradient as two kernels)
    # TMPI_DETERMINISTIC=1 also takes the two-kernel route: the fused kernel reduces the bias gradient with cross-CTA atomics
    return (pool is not None and x.is_cuda and relu in (True, "relu") and pool[3] == "max" and x.dtype == torch.bfloat16
            and os.environ.get("TMPI_DETERMINISTIC") != "1")


def _pool_fwd_after(ctx, impl, y, pool):
    """Forward of the pooling half of a fused conv→pool block; returns (pooled, argmax or None)."""
    if impl is ref:
        return ref.pool2d(y, pool[0], pool[1], pool[2], pool[3]), None
    return impl.pool2d_fwd(y, pool[0], pool[1], pool[2], pool[3])


class _ConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, pad, groups, relu, pool=None):
        impl = _impl(x)
        wc = compute_weight(w)
        ctx.cols = None
        if impl is ref:
            y = ref.conv2d_bias_act(x, wc, b, stride, pad, groups, relu)
        else:
            # keep the im2col matrix of the forward for wgrad (memory is cheap on an 80 GB part; recomputing
            # it cost ~13 % of the AlexNet step)
            y, ctx.cols = impl.conv2d_bias_act(x, wc, b, stride, pad, groups, relu, return_cols=True)
        ctx.w, ctx.b = w, b
        ctx.cfg = (stride, pad, groups, relu)
        ctx.pool = pool
        if pool is None:
            ctx.save_for_backward(x, y)
            return y
        yp, arg = _pool_fwd_after(ctx, impl, y, pool)
        ctx.has_arg = arg is not None
        if arg is not None:
            ctx.save_for_backward(x, y, arg)
        else:
            ctx.save_for_backward(x, y, yp)
        return yp

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors[0], ctx.saved_tensors[1]
        w, b = ctx.w, ctx.b
        stride, pad, groups, relu = ctx.cfg
        pool = ctx.pool
        impl = _impl(x)
        wc = compute_weight(w)
        need_dx = ctx.needs_input_grad[0]
        if impl is ref:
            if pool is not None:
                dy = ref.pool2d_bwd(y, ctx.saved_tensors[2], dy.contiguous(), *pool)
            dx, dw, db = ref.conv2d_bias_act_bwd(x, wc, y, dy, stride, pad, groups, relu, need_dx)
        else:
            pre = False
            db_out = _gout(b)
            if pool is not None:
                if _fused_pool_ok(x, relu, pool) and ctx.has_arg:
                    acc = impl._acc(db_out)
                    db_out = impl.grad_buffer(b.numel(), db_out, x.device)
                    dy = impl.maxpool_relu_bias_bwd(dy, ctx.saved_tensors[2], y, pool, db_out, None, accumulate=acc)
                    pre = True
                else:
                    dy = impl.pool2d_bwd_arg(dy, ctx.saved_tensors[2] if ctx.has_arg else None, tuple(y.shape), *pool)
            dx, dw, db = impl.conv2d_bias_act_bwd(x, wc, y, dy, stride, pad, groups, relu, need_dx,
                                                  dw_out=_gout(w), db_out=db_out, cols=ctx.cols, pre_masked=pre,
                                                  need_db=b is not None)
            ctx.cols = None
        gb = _sink(b, db)
        gw = _sink(w, dw)
        return dx, gw, gb, None, None, None, None, None


def conv2d_bias_act(x, w, b, stride=1, pad=0, groups=1, relu=True, pool=None):
    """``pool`` = (ksize, stride, pad, mode): run the pooling layer that follows inside the same autograd node, so the
    backward can fuse pool-scatter + ReLU mask + bias gradient into one pass over the conv output."""
    return _ConvFn.apply(x, w, b, stride, pad, groups, relu, pool)


class _ConvG2Fn(torch.autograd.Function):
    """AlexNet-style 2-group conv with two independent parameter sets
    (ref ``layers2.py:504-544``).  On CUDA both groups read channel slices of the
    NHWC input in place (no split/concat copies): the im2col gather takes a channel
    offset and the GEMM epilogue writes each half of the output with ldc = C_out."""

    @staticmethod
    def forward(ctx, x, w0, b0, w1, b1, stride, pad, relu, pool=None):
        impl = _impl(x)
        ws = [compute_weight(w0), compute_weight(w1)]
        if impl is ref:
            C = x.shape[-1]
            y0 = ref.conv2d_bias_act(x[..., :C // 2].contiguous(), ws[0], b0, stride, pad, 1, relu)
            y1 = ref.conv2d_bias_act(x[..., C // 2:].contiguous(), ws[1], b1, stride, pad, 1, relu)
            y = torch.cat([y0, y1], dim=-1)
            ctx.cols = None
        else:
            y, ctx.cols = impl.conv2d_group2_bias_act(x, ws[0], b0, ws[1], b1, stride, pad, relu, return_cols=True)
        ctx.p = (w0, b0, w1, b1)
        ctx.cfg = (stride, pad, relu)
        ctx.pool = pool
        if pool is None:
            ctx.save_for_backward(x, y)
            return y
        yp, arg = _pool_fwd_after(ctx, impl, y, pool)
        ctx.has_arg = arg is not None
        if arg is not None:
            ctx.save_for_backward(x, y, arg)
        else:
            ctx.save_for_backward(x, y, yp)
        return yp

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors[0], ctx.saved_tensors[1]
        w0, b0, w1, b1 = ctx.p
        stride, pad, relu = ctx.cfg
        pool = ctx.pool
        impl = _impl(x)
        need_dx = ctx.needs_input_grad[0]
        if impl is ref:
            if pool is not None:
                dy = ref.pool2d_bwd(y, ctx.saved_tensors[2], dy.contiguous(), *pool)
            C, O = x.shape[-1], y.shape[-1]
            outs = []
            for g, (w, b) in enumerate(((w0, b0), (w1, b1))):
                xs = x[..., g * C // 2:(g + 1) * C // 2].contiguous()
                ys = y[..., g * O // 2:(g + 1) * O // 2].contiguous()
                dys = dy[..., g * O // 2:(g + 1) * O // 2].contiguous()
                outs.append(ref.conv2d_bias_act_bwd(xs, compute_weight(w), ys, dys, stride, pad, 1,
                                                    relu, need_dx))
            dx = torch.cat([outs[0][0], outs[1][0]], dim=-1) if need_dx else None
            grads = (outs[0][1], outs[0][2], outs[1][1], outs[1][2])
        else:
            pre = False
            db0, db1 = _gout(b0), _gout(b1)
            if pool is not None:
                if _fused_pool_ok(x, relu, pool) and ctx.has_arg:
                    acc = impl._acc(db0, db1)
                    db0, db1 = impl.grad_buffer(b0.numel(), db0, x.device, acc), impl.grad_buffer(b1.numel(), db1, x.device, acc)
                    dy = impl.maxpool_relu_bias_bwd(dy, ctx.saved_tensors[2], y, pool, db0, db1, accumulate=acc)
                    pre = True
                else:
                    dy = impl.pool2d_bwd_arg(dy, ctx.saved_tensors[2] if ctx.has_arg else None, tuple(y.shape), *pool)
            dx, grads = impl.conv2d_group2_bias_act_bwd(
                x, compute_weight(w0), compute_weight(w1), y, dy, stride, pad, relu, need_dx,
                outs=(_gout(w0), db0, _gout(w1), db1), cols=ctx.cols, pre_masked=pre)
            ctx.cols = None
        gb1 = _sink(b1, grads[3])
        gw1 = _sink(w1, grads[2])
        gb0 = _sink(b0, grads[1])
        gw0 = _sink(w0, grads[0])
        return dx, gw0, gb0, gw1, gb1, None, None, None, None


def conv2d_group2_bias_act(x, w0, b0, w1, b1, stride=1, pad=0, relu=True, pool=None):
    return _ConvG2Fn.apply(x, w0, b0, w1, b1, stride, pad, relu, pool)


# --------------------------------------------------------------------------- transposed conv
class _ConvTFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b, stride, pad, output_padding, act, c_real):
        impl = _impl(x)
        y = impl.conv_transpose2d_bias_act(x, compute_weight(w), b, stride, pad, output_padding, act, c_real)
        ctx.save_for_backward(x, y)
        ctx.w, ctx.b, ctx.cfg = w, b, (stride, pad, act)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y = ctx.saved_tensors
        w, b = ctx.w, ctx.b
        stride, pad, act = ctx.cfg
        impl = _impl(x)
        need_dx = ctx.needs_input_grad[0]
        if impl is ref:
            dx, dw, db = ref.conv_transpose2d_bias_act_bwd(x, compute_weight(w), y, dy, stride, pad, act, need_dx)
        else:
            dx, dw, db = impl.conv_transpose2d_bias_act_bwd(x, compute_weight(w), y, dy, stride, pad, act, need_dx,
                                                            dw_out=_gout(w), db_out=_gout(b))
        gb = _sink(b, db)
        gw = _sink(w, dw)
        return dx, gw, gb, None, None, None, None, None


def conv_transpose2d_bias_act(x, w, b, stride, pad, output_padding=0, act="none", c_real=None):
    """NHWC transposed convolution + bias + activation (``act``: "none", "relu", "leaky", "sigmoid"); ``w`` is
    ``[Cin, KH, KW, Cout]``.  Output channels ``>= c_real`` are zero (16-byte channel padding of a narrow layer)."""
    return _ConvTFn.apply(x, w, b, stride, pad, output_padding, act, c_real)


# --------------------------------------------------------------------------- batch norm (+ residual)(+ ReLU)
class _BatchNormFn(torch.autograd.Function):
    """``relu(γ·x̂ + β + residual)`` as one forward pass (statistics + apply) and one backward pass (reduce + apply); the
    parameter gradients are written straight into the arena's G views (``_gout`` / ``_sink``).  Reference: Lasagne
    ``batch_norm`` + ``ElemwiseSumLayer`` + ``rectify`` (``lasagne_model_zoo/resnet50.py:14-77``)."""

    @staticmethod
    def forward(ctx, x, gamma, beta, residual, run_mean, run_var, training, momentum, eps, relu, drop):
        impl = _impl(x)
        y, mean, rstd = impl.batch_norm_fwd(x, gamma.detach(), beta.detach(), run_mean, run_var, training, momentum, eps, relu, residual,
                                            drop=drop)
        ctx.gamma, ctx.beta = gamma, beta
        ctx.relu, ctx.has_res, ctx.drop = relu, residual is not None, drop
        ctx.save_for_backward(x, y if relu else x.new_empty(0), mean, rstd)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, y, mean, rstd = ctx.saved_tensors
        gamma, beta = ctx.gamma, ctx.beta
        impl = _impl(x)
        need_dres = ctx.has_res and ctx.needs_input_grad[3]
        if impl is ref:
            dx, dres, dg, db = ref.batch_norm_bwd(x, dy, y, gamma.detach(), mean, rstd, ctx.relu, need_dres, drop=ctx.drop)
        else:
            dx, dres, dg, db = impl.batch_norm_bwd(x, dy, y, gamma.detach(), mean, rstd, ctx.relu, need_dres,
                                                   dgamma_out=_gout(gamma), dbeta_out=_gout(beta), drop=ctx.drop)
        gb = _sink(beta, db)
        gg = _sink(gamma, dg)
        return dx, gg, gb, dres, None, None, None, None, None, None, None


def batch_norm(x, gamma, beta, run_mean=None, run_var=None, training=True, momentum=0.1, eps=1e-5, relu=False, residual=None, drop=None):
    """Batch normalisation over all but the channel (last) axis, optionally fused with a residual add and a ReLU.  ``drop``: a
    drop-path row (one fp32 scale s_n per sample, ops/drop_path.py) with a residual: y = relu(s_n·bn(x) + residual); the gradient
    of x, γ and β is that of s_n·g, the residual's is g."""
    return _BatchNormFn.apply(x, gamma, beta, residual, run_mean, run_var, training, momentum, eps, relu, drop)


class _AddFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, a, b, drop):
        ctx.drop = drop
        if drop is not None:
            return _impl(a).add_scaled(a, drop, b)
        if a.is_cuda:
            from . import cuda_impl
            return cuda_impl.add(a, b)
        return a + b

    @staticmethod
    def backward(ctx, dy):
        if ctx.drop is None:
            return dy, dy, None
        return _impl(dy).add_scaled(dy, ctx.drop), dy, None


class _Fork2Fn(torch.autograd.Function):
    """Fan-out of a tensor to two consumers: the two incoming gradients are summed by the native add kernel (autograd would
    otherwise accumulate them with a library elementwise kernel)."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x), x.view_as(x)

    @staticmethod
    def backward(ctx, d1, d2):
        if d1 is None:
            return d2
        if d2 is None:
            return d1
        if d1.is_cuda:
            from . import cuda_impl
            return cuda_impl.add(d1, d2)
        return d1 + d2


def fork2(x):
    """Return two aliases of ``x`` for two consumers (residual shortcut + branch)."""
    if not x.requires_grad:
        return x, x
    return _Fork2Fn.apply(x)


def add(a, b, drop=None):
    """Residual merge ``a + b`` (native kernel on CUDA; the gradient passes to both branches unchanged).  ``drop``: a drop-path row,
    y = s_n·a + b, and the branch ``a`` gets s_n·dy."""
    return _AddFn.apply(a, b, drop)


# --------------------------------------------------------------------------- pool
class _PoolFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ksize, stride, pad, mode):
        ctx.cfg = (ksize, stride, pad, mode)
        if x.is_cuda:
            from . import cuda_impl
            y, arg = cuda_impl.pool2d_fwd(x, ksize, stride, pad, mode)
            ctx.xshape = tuple(x.shape)
            ctx.has_arg = arg is not None
            if arg is not None:
                ctx.save_for_backward(arg)
            return y
        y = ref.pool2d(x, ksize, stride, pad, mode)
        ctx.save_for_backward(x, y)
        return y

    @staticmethod
    def backward(ctx, dy):
        if dy.is_cuda:
            from . import cuda_impl
            arg = ctx.saved_tensors[0] if ctx.has_arg else None
            return cuda_impl.pool2d_bwd_arg(dy, arg, ctx.xshape, *ctx.cfg), None, None, None, None
        x, y = ctx.saved_tensors
        dx = ref.pool2d_bwd(x, y, dy.contiguous(), *ctx.cfg)
        return dx, None, None, None, None


def pool2d(x, ksize, stride, pad=0, mode="max"):
    return _PoolFn.apply(x, ksize, stride, pad, mode)


# --------------------------------------------------------------------------- LRN
class _LRNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, n, k, alpha, beta):
        impl = _impl(x)
        y, _ = impl.lrn(x, n, k, alpha, beta)
        ctx.save_for_backward(x)
        ctx.cfg = (n, k, alpha, beta)
        return y

    @staticmethod
    def backward(ctx, dy):
        (x,) = ctx.saved_tensors
        dx = _impl(x).lrn_bwd(x, dy.contiguous(), *ctx.cfg)
        return dx, None, None, None, None


def lrn(x, n=5, k=2.0, alpha=1e-4, beta=0.75):
    return _LRNFn.apply(x, n, k, alpha, beta)


# --------------------------------------------------------------------------- dropout
class _DropoutFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, p_drop, layer_id):
        if x.is_cuda:
            from . import cuda_impl
            y, mask = cuda_impl.dropout_fwd(x, p_drop, layer_id)
        else:
            st = rng_state()
            mask = ref.dropout_mask(x.shape, p_drop, st["seed"] + layer_id, st["step"], x.device)
            y = ref.dropout(x, p_drop, mask)
        ctx.save_for_backward(mask)
        return y

    @staticmethod
    def backward(ctx, dy):
        (mask,) = ctx.saved_tensors
        if dy.is_cuda:
            from . import cuda_impl
            return cuda_impl.dropout_bwd(dy.contiguous(), mask), None, None
        return dy * mask.to(dy.dtype), None, None


_RNG = {"seed": 0x5EED, "step": 0}


def rng_state():
    return _RNG


def seed_dropout(seed: int):
    _RNG["seed"] = int(seed)
    _RNG["step"] = 0


def advance_rng_step():
    """CPU path only; on CUDA the device step counter advances inside the
    (graph-captured) step so replays draw fresh masks."""
    _RNG["step"] += 1


def dropout(x, p_drop, training, layer_id=0):
    """Reference semantics (``layers2.py:885-891``): train → ``mask*x``;
    eval → ``(1-p)*x`` (no inverted scaling)."""
    if not training:
        return x * (1.0 - p_drop)
    if p_drop <= 0.0:
        return x
    return _DropoutFn.apply(x, p_drop, layer_id)


# --------------------------------------------------------------------------- softmax + NLL
class _SoftmaxXentFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, label_smoothing, mix):
        # under gradient accumulation over n micro-batches dlogits carries 1/n (in fp32, inside the kernel); the loss does not
        loss, err1, err5, dlogits = _impl(logits).softmax_xent(logits, labels, grad_scale=accum.grad_scale(),
                                                               label_smoothing=label_smoothing, mix=mix)
        ctx.save_for_backward(dlogits)
        ctx.in_dtype = logits.dtype
        ctx.mark_non_differentiable(err1, err5)
        return loss, err1, err5

    @staticmethod
    def backward(ctx, gl, g1, g5):
        (dlogits,) = ctx.saved_tensors
        # gl is a 0-dim tensor on the same device: no host sync, graph-capturable
        return (dlogits * gl.to(dlogits.dtype)).to(ctx.in_dtype), None, None, None


def softmax_xent(logits, labels, label_smoothing=0.0, mix=None):
    """Returns (mean NLL, top-1 error, top-5 error) — fused on CUDA.  ``label_smoothing`` ε > 0: the loss (and its gradient) is the
    cross-entropy against the soft target (1 − ε)·onehot + ε / C, as ``F.cross_entropy(..., label_smoothing=ε)``.  ``mix``: the
    step's Mixup / CutMix record (ops/mixup.py); the target is then λ·s(y_i) + (1 − λ)·s(y_j) with j = B − 1 − i, and the errors count
    against the label with the larger weight."""
    return _SoftmaxXentFn.apply(logits, labels, float(label_smoothing), mix)


class _SoftmaxXentKdFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, labels, teacher, alpha, temperature, label_smoothing, mix):
        # the teacher's logits carry no gradient; under gradient accumulation dlogits carries 1/n, as in _SoftmaxXentFn
        loss, err1, err5, dlogits = _impl(logits).softmax_xent_kd(logits, labels, teacher, alpha, temperature,
                                                                  grad_scale=accum.grad_scale(), label_smoothing=label_smoothing, mix=mix)
        ctx.save_for_backward(dlogits)
        ctx.in_dtype = logits.dtype
        ctx.mark_non_differentiable(err1, err5)
        return loss, err1, err5

    @staticmethod
    def backward(ctx, gl, g1, g5):
        (dlogits,) = ctx.saved_tensors
        return (dlogits * gl.to(dlogits.dtype)).to(ctx.in_dtype), None, None, None, None, None, None


def softmax_xent_kd(logits, labels, teacher, alpha, temperature, label_smoothing=0.0, mix=None):
    """Returns (mean L, top-1 error, top-5 error) of knowledge distillation, fused on CUDA: L = (1 − α)·CE_q(z) +
    α·T²·KL(softmax(t/T) ‖ softmax(z/T)) per row, with ``teacher`` the teacher's logits t of the same batch (no gradient) and q the
    target :func:`softmax_xent` takes with ``label_smoothing`` and ``mix``.  The errors are the student's."""
    return _SoftmaxXentKdFn.apply(logits, labels, teacher.detach(), float(alpha), float(temperature), float(label_smoothing), mix)


def mix_draw(cfg, rank, hw, out):
    """This step's Mixup / CutMix record (``cfg`` a validated ``config['mixup']``, ``hw`` the image size at the mix point) into
    ``out``, a uint8 tensor of ops/mixup.py's 64 bytes: on CUDA drawn by the kernel from the device step counter, on the CPU by
    :func:`reference.mix_draw` from the host one.  Returns ``out``."""
    if out.is_cuda:
        from . import cuda_impl
        return cuda_impl.mix_draw(cfg, rank, hw, cuda_impl.step_counter(out.device), out=out)
    from .mixup import encode
    return out.copy_(encode(ref.mix_draw(cfg, cfg["seed"], rank, _RNG["step"], hw)))


def drop_path_draw(dp, out):
    """This step's drop-path table for :class:`drop_path.DropPath` ``dp`` into ``out`` (fp32 [L, B]): on CUDA drawn by the kernel
    from the device step counter, on the CPU by :func:`reference.drop_path_draw` from the host one; both keyed by the dropout
    seed.  Returns ``out``."""
    if out.is_cuda:
        from . import cuda_impl
        return cuda_impl.drop_path_draw(dp, cuda_impl.step_counter(out.device), out)
    return out.copy_(ref.drop_path_draw(dp.rates, _RNG["seed"], dp.rank, _RNG["step"], dp.B))


def cifar_augment_draw(aug):
    """This step's offsets, flips and Cutout boxes for :class:`cifar_augment.CifarAugment` ``aug`` into its buffers: on CUDA drawn by
    the kernel from the device step counter, on the CPU by :func:`reference.cifar_augment_draw` from the host one.  Returns ``aug``."""
    if aug.offs.is_cuda:
        from . import cuda_impl
        cuda_impl.cifar_augment_draw(aug.cfg, aug.rank, cuda_impl.step_counter(aug.offs.device), aug.offs, aug.flips, aug.boxes)
        return aug
    for buf, v in zip((aug.offs, aug.flips, aug.boxes), ref.cifar_augment_draw(aug.cfg, aug.cfg["seed"], aug.rank, _RNG["step"], aug.B)):
        buf.copy_(v)
    return aug


def mix_batch(x, rec):
    """Mix the NHWC batch ``x`` in place (no autograd: it is an input) as the Mixup / CutMix record ``rec`` says; returns ``x``."""
    if x.is_cuda:
        from . import cuda_impl
        return cuda_impl.mix_batch(x, rec)
    with torch.no_grad():
        return x.copy_(ref.mix_batch(x, rec))


# --------------------------------------------------------------------------- GAN losses
class _GanLossFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, scores, kind, a):
        loss, d = _impl(scores).gan_loss(scores, kind, a)
        ctx.save_for_backward(d.view_as(scores))
        return loss

    @staticmethod
    def backward(ctx, gl):
        (d,) = ctx.saved_tensors
        return (d * gl.to(d.dtype)), None, None


def gan_loss(scores, kind, a):
    """WGAN (``kind="wgan"``: ``a * mean(scores)``) or least-squares (``"lsgan"``: ``0.5 * mean((scores - a)^2)``) loss as a
    device scalar; its gradient comes from the same launch (see :func:`reference.gan_loss`)."""
    return _GanLossFn.apply(scores, kind, a)


# --------------------------------------------------------------------------- data aug
def crop_mirror_normalize(x, mean, std_scale, crop_hw, offsets, flips, out_dtype=None, zero_fill=False):
    """Normalise, crop and mirror an NHWC batch: the native kernel on CUDA, :func:`reference.crop_mirror_normalize` on the CPU.
    ``zero_fill``: offsets may put a pixel outside the image, which is then 0 (cifar_augment's zero-padded crop)."""
    if x.is_cuda:
        from . import cuda_impl
        return cuda_impl.crop_mirror_normalize(x, mean, std_scale, crop_hw, offsets, flips, out_dtype, zero_fill=zero_fill)
    return ref.crop_mirror_normalize(x, mean, std_scale, crop_hw, offsets, flips,
                                     out_dtype or torch.float32, zero_fill=zero_fill)


def resized_crop_mirror_normalize(x, mean, std_scale, out_hw, boxes, flips, out_dtype=None):
    """Random-resized crop of a uint8 NHWC batch: the native kernel on CUDA, :func:`reference.resized_crop_mirror_normalize` on
    the CPU."""
    if x.is_cuda:
        from . import cuda_impl
        return cuda_impl.resized_crop_mirror_normalize(x, mean, std_scale, out_hw, boxes, flips, out_dtype)
    return ref.resized_crop_mirror_normalize(x, mean, std_scale, out_hw, boxes, flips, out_dtype or torch.float32)


def random_erase(x, boxes):
    """Random erasing of a normalised NHWC batch: the native kernel in place on CUDA (``boxes`` int32 on the device), a copy from
    :func:`reference.random_erase` on the CPU."""
    if x.is_cuda:
        from . import cuda_impl
        return cuda_impl.random_erase(x, boxes)
    return ref.random_erase(x, boxes)


def auto_augment_crop_normalize(x, mean, std_scale, out_hw, boxes, flips, records, out_dtype=None, weights=None):
    """TrivialAugmentWide / RandAugment / AutoAugment, or AugMix with ``weights``, on the crop of a uint8 NHWC batch, then
    normalisation: the native kernels on CUDA, :func:`reference.auto_augment_crop_normalize` on the CPU."""
    if x.is_cuda:
        from . import cuda_impl
        return cuda_impl.auto_augment_crop_normalize(x, mean, std_scale, out_hw, boxes, flips, records, out_dtype=out_dtype,
                                                     weights=weights)
    return ref.auto_augment_crop_normalize(x, mean, std_scale, out_hw, boxes, flips, records, out_dtype or torch.float32,
                                           weights=weights)
