"""Adapter for ``torch.nn.Module`` models (the reference's Lasagne / Keras / tutorial zoo:
ResNet50, Wide-ResNet, WGAN / LSGAN, LSTM — SURVEY §2.7 G9-G12, §2.6.3 O12-O14).

The module's parameters are bound into the same flat arena as the native-layer models
(``p.data`` and ``p.grad`` become views of W / G), so every rule, exchanger and fused
kernel works on them unchanged.  Two optimizer modes:

* ``flat_sgd`` — the framework's fused momentum-SGD (supports ``cdd`` and the fused
  exchange strategies; the reference's ResNet50 uses ``pre_model_iter_fn`` like this);
* a ``torch.optim`` optimizer (Adam for WRN ``wresnet.py:159``, RMSProp for the GANs
  ``wgan.py:18-59``, Adadelta for the LSTM ``lstm.py:284-342``) — self-contained updates,
  so only ``sync_type='avg'`` makes sense, exactly as in the reference (``wresnet.py:152-153``).

Compute is library code here (cuDNN / cuBLAS through torch, bf16 autocast, channels-last):
SURVEY §2.6.3 lists these ops as out of the headline metric.
"""
from __future__ import annotations

import torch

from .base import ModelBase


def tag_module_params(module):
    """Give parameters the names the arena's group rules understand (BN → gamma/beta)."""
    params, wtypes = [], []
    bn_types = (torch.nn.modules.batchnorm._BatchNorm, torch.nn.LayerNorm, torch.nn.GroupNorm)
    for mod in module.modules():
        for name, p in mod.named_parameters(recurse=False):
            if not p.requires_grad:
                continue
            if isinstance(mod, bn_types):
                p.pname = "gamma" if name == "weight" else "beta"
            else:
                p.pname = "W" if p.dim() > 1 else "b"
            params.append(p)
            wtypes.append("W" if p.dim() > 1 else "b")
    return params, wtypes


class TorchModelBase(ModelBase):
    optimizer_name = "flat_sgd"
    autocast = True
    supports_grad_accum = False    # torch autograd writes .grad: the native accumulate mode does not reach it
    supports_model_ema = False     # the library yardsticks: torch's own AveragedModel is their EMA
    supports_sam = False           # the library yardsticks train with torch's plain optimizers
    supports_lr_schedule = False   # the library yardsticks keep the per-epoch lr policies
    supports_mixup = False         # the library yardsticks train on the plain batch
    supports_grad_clip = False     # torch.optim or the flat SGD without a clipping pass: refused rather than trained unclipped

    def finalize_torch(self, module, input_shape, exchanged=None):
        self.module = module.to(self.device)
        if self.cuda and len(input_shape) == 4:
            self.module = self.module.to(memory_format=torch.channels_last)
        params, wtypes = tag_module_params(self.module)
        if exchanged is not None:
            params = [p for p in params if id(p) in exchanged]
            wtypes = ["W" if p.dim() > 1 else "b" for p in params]
        self.config.setdefault("_arena_shadow", False)
        self.finalize(params, wtypes, input_shape)
        self.layers = None
        for p in self.params:
            p.grad = p.gbuf                    # AccumulateGrad then adds in place into the arena's G region
            p.shadow = None
        self.torch_opt = None

    def make_torch_optimizer(self, params):
        return None

    def forward(self, x):
        if x.dim() == 4:
            x = x.permute(0, 3, 1, 2)          # NHWC storage viewed as channels-last NCHW, no copy
        if self.cuda and self.autocast:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return self.module(x)
        return self.module(x.float())

    def loss(self, x, y, label_smoothing=0.0):
        logits = self.forward(x).float()
        cost = torch.nn.functional.cross_entropy(logits, y, label_smoothing=label_smoothing)
        with torch.no_grad():
            pred = logits.argmax(1)
            err = (pred != y).float().mean()
            k = min(5, logits.shape[1])
            err5 = 1.0 - (logits.topk(k, 1).indices == y[:, None]).any(1).float().mean()
        return cost, err, err5

    def _fwd_bwd_eager(self):
        self.arena.G.zero_()
        for p in self.params:
            if p.grad is None or p.grad.data_ptr() != p.gbuf.data_ptr():
                p.grad = p.gbuf
        self.module.train()
        cost, err, err5 = self.loss(self.x_in, self.y_in, self.label_smoothing)
        cost.backward()
        return cost.detach(), err.detach()

    def compile_val(self):
        def val_fn(subb_ind=0):
            B = self.batch_size
            self.module.eval()
            with torch.no_grad():
                c, e, e5 = self.loss(self.shared_x[subb_ind * B:(subb_ind + 1) * B], self.shared_y[subb_ind * B:(subb_ind + 1) * B])
            self.module.train()
            return c, e, e5

        def multi_view_val_fn(subb_ind=0):
            # val_crops = V > 1: the mean of softmax(logits.float()) over the V views, with the native path's clamp and rank rule
            from ..ops.reference import view_metrics
            B, V = self.batch_size, self.val_crops
            self.module.eval()
            with torch.no_grad():
                pbar = sum(torch.softmax(self.forward(self.val_x[v, subb_ind * B:(subb_ind + 1) * B]).float(), dim=1) for v in range(V)) / V
                c, e, e5 = view_metrics(pbar, self.shared_y[subb_ind * B:(subb_ind + 1) * B])
            self.module.train()
            return c, e, e5
        self.val_fn = val_fn if self.val_crops == 1 else multi_view_val_fn

    def compile_iter_fns(self, sync_type="avg", aggregate="momentum", fused_tail=None):
        self.torch_opt = self.make_torch_optimizer(self.params)
        if self.torch_opt is None:
            return super().compile_iter_fns(sync_type, aggregate, fused_tail)
        self.setup_train_options(fused_tail=fused_tail)
        if sync_type != "avg" and self.size > 1:
            raise ValueError("%s has a self-contained torch optimizer: only sync_type='avg' is supported "
                             "(as in the reference, wresnet.py:152-153)" % self.name)
        self.sync_type = "avg"
        opt = self.torch_opt

        def tail():
            for g in opt.param_groups:
                g["lr"] = self.shared_lr.get_value()
            opt.step()

        self.use_graph = False                     # torch.optim steps read host-side hyper-parameters
        self.set_step_tail(tail)
        self.get_vel = lambda subb=0: self.forward_backward(subb)
        self.descent_vel = lambda: None
        self.train_iter_fn = self.get_vel
        self.vels, self.vels2 = [], []
        self.compile_val()
        self.val_iter_fn = self.val_fn

    def extra_state(self):
        sd = {"module": {k: v.detach().cpu() for k, v in self.module.state_dict().items()}}
        if self.torch_opt is not None:
            sd["opt"] = self.torch_opt.state_dict()
        return sd

    def load_extra_state(self, sd):
        # parameters come from the arena; restore buffers (BN statistics) and optimizer moments
        own = self.module.state_dict()
        for k, v in sd.get("module", {}).items():
            if k in own and own[k].data_ptr() not in {p.data_ptr() for p in self.params}:
                own[k].copy_(v.to(own[k].device))
        if self.torch_opt is not None and "opt" in sd:
            self.torch_opt.load_state_dict(sd["opt"])
