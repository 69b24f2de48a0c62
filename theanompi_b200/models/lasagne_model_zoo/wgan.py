"""Wasserstein GAN / LSGAN on MNIST (ref ``lasagne_model_zoo/wgan.py``, ``lsgan.py``).

Contract quirks kept from the reference: the exchanged ``params`` are the **critic**
parameters only (``wgan.py:142``); ``train_iter`` runs 50 (first 5 and every 100th
generator update) or 2 critic steps with weight clipping ±0.01, then one generator step,
and *returns the advanced count* (``:240-270``); ``val_iter`` records (critic score,
generator score, 0); ``print_info`` plots samples + score curves (``:287-312``); own
``save/load`` (npz); lr decays linearly to zero over the second half (``:314-320``).
RMSProp as in the reference (``wgan.py:18-59``).  DCGAN-style generator / critic
(``:61-110``) built from torch modules.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

from ... import ops
from ..base import ModelBase
from ..torch_base import TorchModelBase, tag_module_params

num_epochs = 100
epochsize = 100
batchsize = 64
initial_eta = 5e-5
clip = 0.01


def build_generator(nz=100, out_ch=1, size=28):
    s4 = size // 4
    return nn.Sequential(nn.Linear(nz, 1024), nn.BatchNorm1d(1024), nn.ReLU(True),
                         nn.Linear(1024, 128 * s4 * s4), nn.BatchNorm1d(128 * s4 * s4), nn.ReLU(True),
                         nn.Unflatten(1, (128, s4, s4)),
                         nn.ConvTranspose2d(128, 64, 5, 2, 2, output_padding=1), nn.BatchNorm2d(64), nn.ReLU(True),
                         nn.ConvTranspose2d(64, out_ch, 5, 2, 2, output_padding=1), nn.Sigmoid())


def build_critic(in_ch=1, size=28):
    s4 = size // 4
    return nn.Sequential(nn.Conv2d(in_ch, 64, 5, 2, 2), nn.LeakyReLU(0.2, True),
                         nn.Conv2d(64, 128, 5, 2, 2), nn.BatchNorm2d(128), nn.LeakyReLU(0.2, True),
                         nn.Flatten(), nn.Linear(128 * s4 * s4, 1024), nn.BatchNorm1d(1024), nn.LeakyReLU(0.2, True),
                         nn.Linear(1024, 1))


class WGAN(TorchModelBase):
    supports_label_smoothing = False   # no classifier head
    supports_mixup = False             # no classifier head
    loss_kind = "wgan"
    n_epochs = num_epochs
    batch_size = file_batch_size = batchsize
    learning_rate = initial_eta
    image_size, image_ch = 28, 1

    def __init__(self, config):
        super().__init__(config)
        self.name = "Wasserstein_GAN" if self.loss_kind == "wgan" else "LSGAN"
        torch.manual_seed(1234)
        self.n_epochs = config.get("n_epochs", self.n_epochs)
        self.epochsize = config.get("epochsize", epochsize)
        self.data = self.make_data(config)
        self.n_subb = 1
        self.generator = build_generator(100, self.image_ch, self.image_size).to(self.device)
        self.critic = build_critic(self.image_ch, self.image_size).to(self.device)
        self.config["_arena_shadow"] = False
        cparams, ctypes = tag_module_params(self.critic)
        for p in cparams:                       # GAN critics: everything (BN included) follows the same rule
            p.pname = "W" if p.dim() > 1 else "b"
        self.finalize(cparams, ctypes, (self.batch_size, self.image_size, self.image_size, self.image_ch))
        for p in self.params:
            p.grad, p.shadow = p.gbuf, None
        self.critic_params = self.params
        self.generator_params = [p for p in self.generator.parameters()]
        self.generator_updates = 0
        self.critic_scores, self.generator_scores, self.c_list, self.g_list = [], [], [], []
        self.current_info = None
        self.init_view = False
        self._train_gen = self.data.iterate("train", seed=1234 + self.rank)
        self._val_gen = self.data.iterate("val", shuffle=False)
        self.data.n_batch_train = self.epochsize
        self.data.n_batch_val = 1

    def make_data(self, config):
        from ..data.mnist import MNIST_data
        d = MNIST_data(self.verbose, **config.get("data_kwargs", {}))
        d.batch_data(self.batch_size)
        return d

    # ---- losses
    def _critic_loss(self, real, fake):
        if self.loss_kind == "wgan":
            return self.critic(fake).mean() - self.critic(real).mean()
        return 0.5 * ((self.critic(real) - 1) ** 2).mean() + 0.5 * (self.critic(fake) ** 2).mean()

    def _gen_loss(self, fake):
        if self.loss_kind == "wgan":
            return -self.critic(fake).mean()
        return 0.5 * ((self.critic(fake) - 1) ** 2).mean()

    def compile_iter_fns(self, sync_type="avg", **kw):
        self.setup_train_options()
        self.sync_type = "avg"
        self.opt_c = torch.optim.RMSprop(self.critic_params, lr=self.learning_rate)
        self.opt_g = torch.optim.RMSprop(self.generator_params, lr=self.learning_rate)
        self.vels, self.vels2 = [], []
        self.train_iter_fn = self.val_iter_fn = None

    def _batch(self, gen):
        x, _ = next(gen)
        return torch.from_numpy(np.ascontiguousarray(x)).to(self.device).permute(0, 3, 1, 2).float()

    def _noise(self, n):
        return torch.rand(n, 100, device=self.device)

    def critic_train_fn(self, real):
        for p in self.critic_params:
            p.grad = p.gbuf
        self.arena.G.zero_()
        with torch.no_grad():
            fake = self.generator(self._noise(real.shape[0]))
        loss = self._critic_loss(real, fake)
        loss.backward()
        self.opt_c.step()
        return -loss.detach() if self.loss_kind == "wgan" else loss.detach()

    def critic_clip_fn(self):
        if self.loss_kind == "wgan":
            with torch.no_grad():
                self.arena.W.clamp_(-clip, clip)

    def generator_train_fn(self):
        self.opt_g.zero_grad(set_to_none=True)
        loss = self._gen_loss(self.generator(self._noise(self.batch_size)))
        loss.backward()
        self.opt_g.step()
        self.arena.G.zero_()
        return loss.detach()

    def train_iter(self, count, recorder):
        if self.loss_kind == "wgan":
            critic_runs = 50 if (self.generator_updates < 5 or self.generator_updates % 100 == 0) else 2
            critic_runs = self.config.get("critic_runs", critic_runs)
        else:
            critic_runs = 1
        scores = []
        recorder.start()
        self.critic.train(); self.generator.train()
        for _ in range(critic_runs):
            scores.append(self.critic_train_fn(self._batch(self._train_gen)))
            self.critic_clip_fn()
            count += 1
        g_score = self.generator_train_fn()
        self.critic_scores.extend(float(s) for s in scores)
        self.generator_scores.append(float(g_score))
        self.generator_updates += 1
        recorder.train_error(count, sum(scores) / len(scores), g_score)
        recorder.end("calc")
        return count

    def val_iter(self, count, recorder):
        self.critic.eval(); self.generator.eval()
        with torch.no_grad():
            real = self._batch(self._val_gen)
            fake = self.generator(self._noise(real.shape[0]))
            c, g = self._critic_loss(real, fake), self._gen_loss(fake)
        recorder.val_error(count, -c if self.loss_kind == "wgan" else c, g, 0)

    def reset_iter(self, *args, **kwargs):
        pass

    def print_info(self, recorder, verbose=True):
        if not self.generator_scores:
            return
        g_, c_ = float(np.mean(self.generator_scores)), float(np.mean(self.critic_scores))
        self.g_list.append(g_); self.c_list.append(c_)
        if verbose:
            print("\nEpoch %d\n  generator score:\t\t%s\n  %s:\t\t%s" % (self.epoch, g_, "Wasserstein distance" if self.loss_kind == "wgan" else "critic loss", c_))
        self.critic_scores[:] = []; self.generator_scores[:] = []
        if verbose and self.config.get("plot", False):
            with torch.no_grad():
                self.generator.eval()
                s = self.generator(self._noise(42)).float().cpu().numpy()
            img = s[:, 0].reshape(6, 7, self.image_size, self.image_size).transpose(0, 2, 1, 3).reshape(6 * self.image_size, 7 * self.image_size)
            if not self.init_view:
                self.init_view = True
                recorder.plot_init(name="scores", save=True); recorder.plot_init(name="sample", save=True)
            recorder.plot(name="sample", image=img, cmap="gray")
            recorder.plot(name="scores", lines=[(list(range(len(self.c_list))), self.c_list, "critic"),
                                                (list(range(len(self.g_list))), self.g_list, "generator")])

    def adjust_hyperp(self, epoch):
        if epoch >= self.n_epochs // 2:
            progress = float(epoch) / self.n_epochs
            lr = self.learning_rate * 2 * (1 - progress)
            self.shared_lr.set_value(lr)
            for opt in (self.opt_c, self.opt_g):
                for g in opt.param_groups:
                    g["lr"] = lr

    def cleanup(self):
        pass

    def save(self, path):
        import os
        os.makedirs(path, exist_ok=True)
        np.savez(os.path.join(path, "%s_gen_%d.npz" % (self.name, self.epoch)), *[p.detach().cpu().numpy() for p in self.generator_params])
        np.savez(os.path.join(path, "%s_crit_%d.npz" % (self.name, self.epoch)), *[p.detach().cpu().numpy() for p in self.critic_params])

    def load(self, path, epoch):
        import os
        for params, tag in ((self.generator_params, "gen"), (self.critic_params, "crit")):
            with np.load(os.path.join(path, "%s_%s_%d.npz" % (self.name, tag, epoch))) as f:
                with torch.no_grad():
                    for p, k in zip(params, sorted(f.files, key=lambda s: int(s.split("_")[1]))):
                        p.copy_(torch.from_numpy(f[k]).to(p.device))


# ---------------------------------------------------------------------------------------------------------------- native
class NativeWGAN(ModelBase):
    """The same GAN on the hand-written sm_90a kernels (CPU: the reference ops), NHWC, with the contract of :class:`WGAN`.

    Generator: FC 100→1024, BN, ReLU; FC →128·s4·s4, BN, ReLU; transposed conv 5×5/2 →64, BN, ReLU; transposed conv 5×5/2 →image,
    sigmoid.  Critic: conv 5×5/2 →64, leaky ReLU; conv 5×5/2 →128, BN, leaky ReLU; FC →1024, BN, leaky ReLU; FC →1.  The image
    layer is padded to 16-byte channels (8 in bf16, 4 in fp32) with zero weights; its padded channels are stored as zeros, so the
    critic's padded input weights get zero gradient and stay zero.  The critic parameters are the exchanged arena (``params``);
    the generator has its own local arena.  Both train with :class:`FlatRMSProp` (the critic's ±0.01 clip in the same pass).
    On the GPU the critic step and the generator step are two captured CUDA graphs; ``train_iter`` copies each real batch into
    a static buffer and replays the critic graph ``critic_runs`` times, then the generator graph.  Noise is Philox keyed by a
    device step counter the graphs advance.

    ``grad_clip=5`` gives the reference MNIST GANs' gradient rescaling, g·5 / max(5, ‖g‖) (``wgan.py:18-59``, ``lsgan.py:14-55``),
    with the critic's and the generator's gradients clipped separately, each by the norm of its own arena.  It differs from the
    reference in two ways.  The reference takes the square root twice (``wgan.py:29-31``), so its threshold is effectively on
    ‖g‖^½; here it is on the true norm.  On a non-finite norm the reference substitutes g = 0.1·W; here the step is skipped and
    ``opt_c.skipped`` / ``opt_g.skipped`` count it.  The reference's CIFAR-10 LSGAN uses plain RMSProp without rescaling, so there
    ``grad_clip`` is simply available."""
    supports_grad_accum = False    # its critic / generator steps keep their own gaccum accumulation
    supports_model_ema = False     # two arenas, critic and generator
    supports_sam = False           # two arenas and an adversarial step, not one loss to flatten
    supports_lr_schedule = False   # two arenas and critic / generator step ratios: the reference's per-epoch decay
    supports_label_smoothing = False   # no classifier head
    supports_mixup = False             # no classifier head
    loss_kind = "wgan"
    n_epochs = num_epochs
    batch_size = file_batch_size = batchsize
    learning_rate = initial_eta
    image_size, image_ch = 28, 1
    bias_lr_mult = 1.0
    nz = 100

    def __init__(self, config):
        super().__init__(config)
        from ...ops import cuda_impl, functional as F_
        from ...parallel.arena import FlatArena
        from ...utils.opt import FlatRMSProp
        self.F = F_
        self.name = "Wasserstein_GAN" if self.loss_kind == "wgan" else "LSGAN"
        self.n_epochs = config.get("n_epochs", self.n_epochs)
        self.epochsize = config.get("epochsize", epochsize)
        self.data = self.make_data(config)
        self.n_subb = 1
        self.cp = cp = 4 if self.precision == "tf32" else 8              # 16-byte channel padding of the image
        self.seed = int(config.get("seed", 1234))
        g = torch.Generator().manual_seed(self.seed)
        S, s4, C = self.image_size, self.image_size // 4, self.image_ch

        def u(*shape, fan_in, cols=None):
            t = (torch.rand(*shape, generator=g) * 2 - 1) / fan_in ** 0.5
            if cols is not None:
                t[..., cols:] = 0
            return t

        def named(ts, names):
            for t, n in zip(ts, names):
                t.pname = n
                t.requires_grad_(True)
            return ts

        ones, zeros = torch.ones, torch.zeros
        gen = [u(1024, self.nz, fan_in=self.nz), zeros(1024), ones(1024), zeros(1024),
               u(s4 * s4 * 128, 1024, fan_in=1024), zeros(s4 * s4 * 128), ones(s4 * s4 * 128), zeros(s4 * s4 * 128),
               u(128, 5, 5, 64, fan_in=128 * 25), zeros(64), ones(64), zeros(64),
               u(64, 5, 5, cp, fan_in=64 * 25, cols=C), zeros(cp)]
        crit = [u(64, 5, 5, cp, fan_in=C * 25, cols=C), zeros(64),
                u(128, 5, 5, 64, fan_in=64 * 25), zeros(128), ones(128), zeros(128),
                u(1024, s4 * s4 * 128, fan_in=s4 * s4 * 128), zeros(1024), ones(1024), zeros(1024),
                u(1, 1024, fan_in=1024), zeros(1)]
        # GAN critics / generators: every parameter (BN included) follows the same rule, as in the torch twin
        named(gen, ["W" if t.dim() > 1 else "b" for t in gen]); named(crit, ["W" if t.dim() > 1 else "b" for t in crit])
        self.finalize(crit, [t.pname for t in crit], (self.batch_size, S, S, cp))
        self.critic_params = self.params
        for p in self.critic_params:
            p.gaccum = True                  # the critic loss sums a real and a fake pass
        self.gen_arena = FlatArena(gen, [t.pname for t in gen], self.device, bias_lr_mult=1.0,
                                   shadow=False if self.precision == "tf32" else None)
        self.generator_params = gen
        self.gen_lr = self.gen_arena.hyper
        self.gen_arena.hyper[0] = float(self.base_lr)
        self.opt_c = FlatRMSProp(self.arena, clip=clip if self.loss_kind == "wgan" else 0.0)
        self.opt_g = FlatRMSProp(self.gen_arena)
        if self.grad_clip is not None:                   # each arena by its own gradient norm, as the reference's MNIST GANs
            self.opt_c.set_grad_clip(self.grad_clip)
            self.opt_g.set_grad_clip(self.grad_clip)
        dev = self.device
        self.bn_stats = {k: (torch.zeros(n, device=dev), torch.ones(n, device=dev))
                         for k, n in (("g1", 1024), ("g2", s4 * s4 * 128), ("g3", 64), ("c2", 128), ("c3", 1024))}
        self.step = torch.zeros(1, dtype=torch.int64, device=dev)          # noise counter, advanced by every step
        self.real_raw = torch.zeros((self.batch_size, S, S, C), dtype=torch.float32, device=dev)
        self.generator_updates = 0
        self.critic_scores, self.generator_scores, self.c_list, self.g_list = [], [], [], []
        self.current_info = None
        self.init_view = False
        self._train_gen = self.data.iterate("train", seed=1234 + self.rank)
        self._val_gen = self.data.iterate("val", shuffle=False)
        self.data.n_batch_train = self.epochsize
        self.data.n_batch_val = 1
        self._cuda_impl = cuda_impl if self.cuda else None

    make_data = WGAN.make_data

    # ---- network
    def _bn(self, x, gamma, beta, key, training, act):
        m, v = self.bn_stats[key]
        return self.F.batch_norm(x, gamma, beta, m, v, training=training, relu=act)

    def generator(self, z, training=True):
        F_, p = self.F, self.generator_params
        s4 = self.image_size // 4
        h = self._bn(F_.linear_bias_act(z, p[0], p[1], relu=False), p[2], p[3], "g1", training, True)
        h = self._bn(F_.linear_bias_act(h, p[4], p[5], relu=False), p[6], p[7], "g2", training, True)
        h = h.reshape(z.shape[0], s4, s4, 128)
        h = self._bn(F_.conv_transpose2d_bias_act(h, p[8], p[9], 2, 2, 1, "none"), p[10], p[11], "g3", training, True)
        return F_.conv_transpose2d_bias_act(h, p[12], p[13], 2, 2, 1, "sigmoid", c_real=self.image_ch)

    def critic(self, x, training=True):
        F_, p = self.F, self.critic_params
        h = F_.conv2d_bias_act(x, p[0], p[1], 2, 2, 1, relu="leaky")
        h = self._bn(F_.conv2d_bias_act(h, p[2], p[3], 2, 2, 1, relu=False), p[4], p[5], "c2", training, "leaky")
        h = h.reshape(x.shape[0], -1)
        h = self._bn(F_.linear_bias_act(h, p[6], p[7], relu=False), p[8], p[9], "c3", training, "leaky")
        return F_.linear_bias_act(h, p[10], p[11], relu=False)

    def _noise(self, n, stream):
        if self.cuda:
            return self._cuda_impl.uniform_noise((n, self.nz), self.seed, stream, self.step)
        return ops.reference.uniform_noise((n, self.nz), self.seed, stream, int(self.step))

    def _advance(self):
        if self.cuda:
            ci = self._cuda_impl
            ci.L().advance_step(self.step.data_ptr(), ci._st(self.step))
        else:
            self.step += 1

    def _stage_real(self):
        """The static real batch in the critic's padded channel layout (a native normalise/pad pass on the GPU)."""
        B, S = self.batch_size, self.image_size
        if self.cuda:
            z = torch.zeros((B, 2), dtype=torch.int32, device=self.device)
            return self._cuda_impl.crop_mirror_normalize(self.real_raw, torch.zeros(1, device=self.device), 1.0, (S, S), z,
                                                         z[:, 0].to(torch.uint8), c_out=self.cp)
        x = torch.zeros((B, S, S, self.cp))
        x[..., :self.image_ch] = self.real_raw
        return x

    def _losses(self, real, fake):
        gl = self.F.gan_loss
        if self.loss_kind == "wgan":
            return gl(self.critic(fake), "wgan", 1.0) + gl(self.critic(real), "wgan", -1.0)
        return gl(self.critic(real), "lsgan", 1.0) + gl(self.critic(fake), "lsgan", 0.0)

    def _critic_body(self):
        self.arena.G.zero_()
        with torch.no_grad():
            fake = self.generator(self._noise(self.batch_size, 0))
        loss = self._losses(self._stage_real(), fake)
        loss.backward()
        with torch.no_grad():
            self.opt_c.step()
        self._advance()
        return (-loss if self.loss_kind == "wgan" else loss).detach()

    def _gen_body(self):
        o = self.critic(self.generator(self._noise(self.batch_size, 1)))
        loss = self.F.gan_loss(o, self.loss_kind, -1.0 if self.loss_kind == "wgan" else 1.0)
        loss.backward()
        with torch.no_grad():
            self.opt_g.step()
        self._advance()
        return loss.detach()

    def _run(self, kind):
        """Eager on the CPU / without graphs; on the GPU one captured graph per step kind (:meth:`ModelBase.run_keyed_step`)."""
        return self.run_keyed_step(kind, self._critic_body if kind == "critic" else self._gen_body)

    # ---- contract
    def compile_iter_fns(self, sync_type="avg", **kw):
        self.setup_train_options(optimizer="rmsprop")
        self.sync_type = "avg"
        self.vels, self.vels2 = [], []
        self.train_iter_fn = self.val_iter_fn = None

    def _load_real(self, gen):
        x, _ = next(gen)
        self.real_raw.copy_(torch.from_numpy(np.ascontiguousarray(x, dtype=np.float32)).reshape(self.real_raw.shape))

    def train_iter(self, count, recorder):
        if self.loss_kind == "wgan":
            critic_runs = 50 if (self.generator_updates < 5 or self.generator_updates % 100 == 0) else 2
            critic_runs = self.config.get("critic_runs", critic_runs)
        else:
            critic_runs = 1
        scores = []
        recorder.start()
        for _ in range(critic_runs):
            self._load_real(self._train_gen)
            scores.append(self._run("critic"))
            count += 1
        g_score = self._run("gen")
        self.critic_scores.extend(scores)
        self.generator_scores.append(g_score)
        self.generator_updates += 1
        recorder.train_error(count, sum(scores) / len(scores), g_score)
        recorder.end("calc")
        return count

    def val_iter(self, count, recorder):
        self._load_real(self._val_gen)
        with torch.no_grad():
            fake = self.generator(self._noise(self.batch_size, 2), training=False)
            o_real, o_fake = self.critic(self._stage_real(), training=False), self.critic(fake, training=False)
            if self.loss_kind == "wgan":
                c, g = o_fake.float().mean() - o_real.float().mean(), -o_fake.float().mean()
            else:
                c = 0.5 * ((o_real.float() - 1) ** 2).mean() + 0.5 * (o_fake.float() ** 2).mean()
                g = 0.5 * ((o_fake.float() - 1) ** 2).mean()
        recorder.val_error(count, -c if self.loss_kind == "wgan" else c, g, 0)

    def reset_iter(self, *args, **kwargs):
        pass

    def print_info(self, recorder, verbose=True):
        if not self.generator_scores:
            return
        g_ = float(torch.stack([s.float() for s in self.generator_scores]).mean())
        c_ = float(torch.stack([s.float() for s in self.critic_scores]).mean())
        self.g_list.append(g_); self.c_list.append(c_)
        if verbose:
            print("\nEpoch %d\n  generator score:\t\t%s\n  %s:\t\t%s" % (self.epoch, g_, "Wasserstein distance" if self.loss_kind == "wgan" else "critic loss", c_))
        self.critic_scores[:] = []; self.generator_scores[:] = []
        if verbose and self.config.get("plot", False):
            with torch.no_grad():
                s = self.generator(self._noise(42, 3), training=False)[..., 0].float().cpu().numpy()
            S = self.image_size
            img = s.reshape(6, 7, S, S).transpose(0, 2, 1, 3).reshape(6 * S, 7 * S)
            if not self.init_view:
                self.init_view = True
                recorder.plot_init(name="scores", save=True); recorder.plot_init(name="sample", save=True)
            recorder.plot(name="sample", image=img, cmap="gray")
            recorder.plot(name="scores", lines=[(list(range(len(self.c_list))), self.c_list, "critic"),
                                                (list(range(len(self.g_list))), self.g_list, "generator")])

    def adjust_hyperp(self, epoch):
        if epoch >= self.n_epochs // 2:
            lr = self.learning_rate * 2 * (1 - float(epoch) / self.n_epochs)
            self.shared_lr.set_value(lr)
            self.gen_arena.hyper[0] = lr

    save = WGAN.save

    def load(self, path, epoch):
        WGAN.load(self, path, epoch)
        self.arena.refresh_shadow(); self.gen_arena.refresh_shadow()

    def extra_state(self):
        """Batch-norm running statistics, the generator arena, both RMSProp averages, the noise step and the schedule."""
        return {"bn": {k: (m.detach().cpu(), v.detach().cpu()) for k, (m, v) in self.bn_stats.items()},
                "gen_arena": self.gen_arena.state_dict(), "rms_c": self.opt_c.state_dict(), "rms_g": self.opt_g.state_dict(),
                "step": int(self.step), "generator_updates": self.generator_updates}

    def load_extra_state(self, sd):
        for k, (m, v) in sd["bn"].items():
            self.bn_stats[k][0].copy_(m); self.bn_stats[k][1].copy_(v)
        self.gen_arena.load_state_dict(sd["gen_arena"])
        self.opt_c.load_state_dict(sd["rms_c"]); self.opt_g.load_state_dict(sd["rms_g"])
        self.step.fill_(int(sd["step"]))
        self.generator_updates = int(sd["generator_updates"])
