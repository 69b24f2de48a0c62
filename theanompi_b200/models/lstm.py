"""LSTM sentiment classifier on IMDB (ref ``theanompi/models/lstm.py`` — the Theano tutorial
LSTM: 128 units, maxlen 500, batch 16, mean-pooling over time, Adadelta ``:284-342`` — and
its model-contract adapter ``lstm_theanompi_outdated.py`` with rank-sharded ``IMDB_Data``
``:75-94`` and early stopping through ``val_iter`` returning ``'stop'``).

``LSTM`` runs on the hand-written kernels: embedding gather / scatter, the input projection of all time steps as one
wgmma GEMM, the masked recurrence as ONE autograd node (per step: one small GEMM + one fused cell kernel; the recurrent
weight gradient of the whole sequence is a single GEMM), masked mean pooling, dropout, softmax head (``ops/rnn.py``,
``csrc/rnn_kernels.cu``), and the update as one flat optimizer launch (Adadelta, the reference's centred RMSProp or SGD,
``config['optimizer']``); on the GPU each step is a CUDA graph per sequence-length bucket.  ``LSTMTorch`` is the same model on
``torch.nn.LSTM`` (cuDNN), kept as the library yardstick.  Sequences are never split across devices (the reference has no
sequence parallelism, SURVEY §5.7).  Without the IMDB pickle a synthetic corpus with class-dependent token statistics is
generated, with lengths drawn from ``data_kwargs['seq_len'] = (lo, hi)``.
"""
from __future__ import annotations

import os

import numpy as np
import torch
import torch.nn as nn

from .base import ModelBase
from .torch_base import TorchModelBase

dim_proj = 128
maxlen = 500
n_words = 10000
batch_size = 16
patience = 10
max_epochs = 100


class IMDB_Data(object):
    def __init__(self, rank=0, size=1, n_synthetic=512, seed=0, maxlen=maxlen, n_words=n_words, seq_len=(20, 80)):
        path = os.environ.get("TMPI_IMDB_PATH", "./imdb.pkl")
        rs = np.random.RandomState(seed)
        if os.path.exists(path):
            import pickle
            with open(path, "rb") as f:
                tr = pickle.load(f); te = pickle.load(f)
            xs = [np.asarray([min(w, n_words - 1) for w in s][:maxlen]) for s in tr[0]]
            ys = np.asarray(tr[1])
        else:
            ys = rs.randint(0, 2, n_synthetic)
            xs = []
            for y in ys:
                L = min(rs.randint(*seq_len), maxlen)                           # lengths drawn from [lo, hi)
                base = rs.randint(2, n_words, L)
                marks = rs.rand(L) < 0.3
                base[marks] = (2 + y * 50 + rs.randint(0, 50, marks.sum()))        # sentiment-bearing tokens
                xs.append(base)
        n = len(xs)
        nv = max(1, n // 10)
        self.train = (xs[nv:][rank::size], ys[nv:][rank::size])        # shard by rank (ref :75-94)
        self.valid = (xs[:nv], ys[:nv])
        self.n_words, self.maxlen = n_words, maxlen

    def batches(self, split, bs, shuffle, seed=None):
        xs, ys = self.train if split == "train" else self.valid
        idx = np.random.RandomState(seed).permutation(len(xs)) if shuffle else np.arange(len(xs))
        for s in range(0, len(xs) - bs + 1, bs):
            sel = idx[s:s + bs]
            L = max(len(xs[i]) for i in sel)
            x = np.zeros((bs, L), dtype=np.int64); m = np.zeros((bs, L), dtype=np.float32)
            for j, i in enumerate(sel):
                x[j, :len(xs[i])] = xs[i]; m[j, :len(xs[i])] = 1
            yield x, m, np.asarray([ys[i] for i in sel], dtype=np.int64)


class LSTMNet(nn.Module):
    def __init__(self, n_words, dim, n_out=2):
        super().__init__()
        self.emb = nn.Embedding(n_words, dim)
        self.lstm = nn.LSTM(dim, dim, batch_first=True)
        self.drop = nn.Dropout(0.5)
        self.out = nn.Linear(dim, n_out)

    def forward(self, x, mask):
        h, _ = self.lstm(self.emb(x))
        pooled = (h * mask[..., None]).sum(1) / mask.sum(1, keepdim=True).clamp_min(1)    # mean pooling (ref :217-253)
        return self.out(self.drop(pooled))


BUCKET = 16                 # graph buckets: the time length of a batch is padded up to a multiple of this


def bucket_len(T, maxlen):
    """Time length of the graph bucket that holds a batch of ``T`` steps: ``T`` rounded up to a multiple of :data:`BUCKET`, capped at
    the bucket that holds ``maxlen``."""
    cap = -(-maxlen // BUCKET) * BUCKET
    if T > cap:
        raise ValueError("batch of %d time steps is longer than maxlen %d" % (T, maxlen))
    return min(-(-T // BUCKET) * BUCKET, cap)


def pad_batch(x, m, T):
    """Pad a ``[B, t]`` batch to ``T`` steps with token id 0 and mask 0 (the masked carry makes padded steps no-ops)."""
    xp, mp = np.zeros((x.shape[0], T), dtype=x.dtype), np.zeros((m.shape[0], T), dtype=m.dtype)
    xp[:, :x.shape[1]], mp[:, :m.shape[1]] = x, m
    return xp, mp


class LSTM(ModelBase):
    """``config['optimizer']``: ``'adadelta'`` (default, lr 1.0), ``'rmsprop'`` (the reference's centred RMSProp with momentum,
    lr 1e-4) or ``'sgd'`` (``p - lr·g``, lr 1e-4), the three optimizers of the reference's ``train_lstm``; ``learning_rate``
    overrides the lr.  Each is one flat native launch over the arena; ``grad_clip`` (a maximum global gradient norm, the usual
    control for recurrent nets) adds the two norm launches before it.  On the GPU every training step is one CUDA graph per
    sequence-length bucket (:func:`bucket_len`): the batch is padded to its bucket, copied into the bucket's static buffers and
    the bucket's graph (forward, backward, update) is replayed.  ``cuda_graph=False`` and the CPU run the step eagerly on the
    unpadded batch; validation is always eager."""
    supports_mixup = False         # token input: nothing to mix
    supports_grad_accum = False    # one graph per sequence-length bucket, each with its own update
    supports_model_ema = False     # one graph per sequence-length bucket
    supports_sam = False           # its step has its own forward and backward per bucket
    n_epochs = max_epochs
    batch_size = file_batch_size = batch_size
    learning_rate = 1.0
    weight_decay = 0.0
    bias_lr_mult = 1.0
    optimizers = {"adadelta": 1.0, "rmsprop": 1e-4, "sgd": 1e-4}        # default lr per optimizer (ref train_lstm)

    def __init__(self, config):
        super().__init__(config)
        self.name = "LSTM"
        self.opt_name = config.get("optimizer", "adadelta")
        if self.opt_name not in self.optimizers:
            raise ValueError("LSTM optimizer must be one of %s, not %r" % (sorted(self.optimizers), self.opt_name))
        self.learning_rate = float(config.get("learning_rate", self.optimizers[self.opt_name]))
        self.base_lr = np.float32(self.learning_rate)
        self.opt = None
        from . import layers2
        from .layers2 import Constant, Normal, _tag
        layers2.reseed(123)
        self.n_epochs = config.get("n_epochs", self.n_epochs)
        self.data = IMDB_Data(self.rank, self.size, **config.get("data_kwargs", {}))
        self.n_subb = 1
        D = H = int(config.get("dim_proj", dim_proj))
        self.dim = D
        V = self.data.n_words
        ortho = lambda n: np.linalg.svd(layers2.rng.randn(n, n))[0].astype(np.float32)      # noqa: E731  (ref ortho_weight :104-107)
        self.emb = Normal((V, D), std=0.01)
        self.W = Constant((4 * H, D)); self.W._set(np.concatenate([ortho(D) for _ in range(4)], 0))
        self.U = Constant((4 * H, H)); self.U._set(np.concatenate([ortho(H) for _ in range(4)], 0))
        self.b = Constant((4 * H,), 0.0)
        self.Wo = Normal((2, H), std=0.01)
        self.bo = Constant((2,), 0.0)
        for t, n_, wt in ((self.emb, "Wemb", "W"), (self.W, "W", "W"), (self.b, "b", "b"), (self.U, "U", "W"), (self.Wo, "Wout", "W"),
                          (self.bo, "bout", "b")):
            _tag(t.val, n_, wt)
        params = [self.emb.val, self.W.val, self.b.val, self.U.val, self.Wo.val, self.bo.val]
        self.layers = None
        self.finalize(params, ["W", "W", "b", "W", "W", "b"], (self.batch_size, 1))
        self.data.n_batch_train = len(self.data.train[0]) // self.batch_size
        self.data.n_batch_val = max(1, len(self.data.valid[0]) // self.batch_size)
        self.best_err, self.bad_counter, self.patience = 1.0, 0, config.get("patience", patience)
        self._train_it = None
        self.training = True
        self._buckets = {}

    def forward_logits(self, x, mask):
        """x: int64 [B, T] token ids, mask: float [B, T]."""
        from .. import ops
        from ..ops import rnn
        B, T = x.shape
        ids = x.t().contiguous()                                   # time-major like the reference's scan
        m = mask.t().contiguous()
        e = rnn.embedding(ids, self.emb.val)                       # [T, B, D]
        gx = ops.linear_bias_act(e.reshape(T * B, self.dim), self.W.val, self.b.val, False).view(T, B, 4 * self.dim)
        h = rnn.lstm_sequence(gx, self.U.val, m)                   # [T, B, H]
        pooled = rnn.masked_mean(h, m)                             # mean pooling over the valid steps (ref :217-253)
        pooled = ops.dropout(pooled, 0.5, self.training, layer_id=0)
        return ops.linear_bias_act(pooled, self.Wo.val, self.bo.val, False)

    def _make_opt(self):
        if self.opt is None:
            from ..utils.opt import FlatAdadelta, FlatCenteredRMSProp, FlatSGD
            if self.opt_name == "adadelta":
                self.opt = FlatAdadelta(self.arena)                    # ref :284-342
            elif self.opt_name == "rmsprop":
                self.opt = FlatCenteredRMSProp(self.arena)             # ref :376-402
            else:
                self.opt = FlatSGD(self.arena, mu=0.0, use_momentum=False)       # ref :256-281: p - lr·g
            if self.grad_clip is not None:
                self.opt.set_grad_clip(self.grad_clip)                 # inside each bucket's captured step
        return self.opt

    def compile_iter_fns(self, sync_type="avg", **kw):
        self.setup_train_options()
        self.sync_type = "avg"
        self._make_opt()
        self.vels, self.vels2 = [], []

    def _to(self, x, m, y):
        d = self.device
        return torch.from_numpy(x).to(d), torch.from_numpy(m).to(d), torch.from_numpy(y).to(d)

    def _train_body(self, x, m, y):
        """Forward, backward and the flat update of one batch (device tensors); returns device scalars (cost, error)."""
        from .. import ops
        self._schedule_lr()                                        # one model-wide update counter for every bucket's graph
        self.arena.G.zero_()
        cost, err, _ = ops.softmax_xent(self.forward_logits(x, m), y, self.label_smoothing)
        cost.backward()                                            # the kernels write the gradients into the arena's G views
        with torch.no_grad():
            self.opt.step()                                        # lr from arena.hyper[0] (= shared_lr)
        self._after_step()
        return cost.detach(), err.detach()

    def _stage(self, x, m, y):
        """Copy a batch, padded to its bucket, into the bucket's static device buffers (one H2D copy from pinned staging).
        Returns the bucket length and the static ``(x, mask, y)``."""
        Tb = bucket_len(x.shape[1], self.data.maxlen)
        b = self._buckets.get(Tb)
        if b is None:
            B = self.batch_size
            nx, nm = B * Tb * 8, B * Tb * 4

            def views(raw):
                return (raw[:nx].view(torch.int64).view(B, Tb), raw[nx:nx + nm].view(torch.float32).view(B, Tb),
                        raw[nx + nm:].view(torch.int64))
            pin = torch.zeros(nx + nm + B * 8, dtype=torch.uint8, pin_memory=True)
            dev = torch.zeros(nx + nm + B * 8, dtype=torch.uint8, device=self.device)
            b = self._buckets[Tb] = {"pin": pin, "dev": dev, "host": views(pin), "static": views(dev), "event": None}
        if b["event"] is not None:
            b["event"].synchronize()          # the host runs ahead of the device: the last copy out of this staging buffer has run
        xp, mp = pad_batch(x, m, Tb)
        hx, hm, hy = b["host"]
        hx.numpy()[:] = xp; hm.numpy()[:] = mp; hy.numpy()[:] = y
        b["dev"].copy_(b["pin"], non_blocking=True)
        if b["event"] is None:
            b["event"] = torch.cuda.Event()
        b["event"].record(torch.cuda.current_stream(self.device))
        return Tb, b["static"]

    def train_iter(self, count, recorder):
        if self._train_it is None:
            self._train_it = self.data.batches("train", self.batch_size, True, seed=self.epoch)
        try:
            x, m, y = next(self._train_it)
        except StopIteration:
            self._train_it = self.data.batches("train", self.batch_size, True, seed=self.epoch + 1000)
            x, m, y = next(self._train_it)
        recorder.start()
        self.training = True
        if self.use_graph:
            Tb, (xs, ms, ys) = self._stage(x, m, y)
            cost, err = self.run_keyed_step(Tb, lambda: self._train_body(xs, ms, ys))
        else:
            cost, err = self._train_body(*self._to(x, m, y))
        recorder.train_error(count, cost, err)
        recorder.end("calc")

    def val_iter(self, count, recorder):
        """One full validation pass; returns ``'stop'`` when patience runs out (the early-stop
        protocol ``BSP_run`` understands, ``worker.py:118-126``)."""
        from .. import ops
        self.training = False
        errs, costs = [], []
        with torch.no_grad():
            for x, m, y in self.data.batches("valid", min(self.batch_size, len(self.data.valid[0])), False):
                x, m, y = self._to(x, m, y)
                c, e, _ = ops.softmax_xent(self.forward_logits(x, m), y)
                costs.append(float(c)); errs.append(float(e))
        self.training = True
        e, c = float(np.mean(errs)), float(np.mean(costs))
        recorder.val_error(count, c, e, 0)
        if e < self.best_err:
            self.best_err, self.bad_counter = e, 0
        else:
            self.bad_counter += 1
            if self.bad_counter > self.patience:
                return "stop"
        return self.data.n_batch_val            # one call covers the whole validation set

    def extra_state(self):
        """The optimizer's extra buffers (its U-region state travels with the arena), its name and the early-stopping state."""
        opt = self._make_opt()
        sd = {"optimizer": self.opt_name, "opt": opt.state_dict(), "best_err": self.best_err, "bad_counter": self.bad_counter}
        if self.lr_sched is not None:
            sd["lr_schedule"] = self.lr_sched.state_dict()
        return sd

    def load_extra_state(self, sd):
        if sd.get("optimizer") != self.opt_name:
            raise ValueError("checkpoint was written by an LSTM trained with optimizer %r; this model uses %r"
                             % (sd.get("optimizer"), self.opt_name))
        self._make_opt().load_state_dict(sd["opt"])
        self.best_err, self.bad_counter = float(sd["best_err"]), int(sd["bad_counter"])
        if "lr_schedule" in sd and self.lr_sched is not None:
            self.lr_sched.load_state_dict(sd["lr_schedule"])

    def reset_iter(self, mode):
        if mode == "train":
            self._train_it = None
            self._report_lr()

    def adjust_hyperp(self, epoch):
        pass

    def cleanup(self):
        pass


class LSTMTorch(TorchModelBase):
    n_epochs = max_epochs
    batch_size = file_batch_size = batch_size
    learning_rate = 1.0
    autocast = False

    def __init__(self, config):
        super().__init__(config)
        self.name = "LSTMTorch"
        torch.manual_seed(123)
        self.n_epochs = config.get("n_epochs", self.n_epochs)
        self.data = IMDB_Data(self.rank, self.size, **config.get("data_kwargs", {}))
        self.n_subb = 1
        self.config["_arena_shadow"] = False
        self.finalize_torch(LSTMNet(self.data.n_words, config.get("dim_proj", dim_proj)), (self.batch_size, 1))
        self.data.n_batch_train = len(self.data.train[0]) // self.batch_size
        self.data.n_batch_val = max(1, len(self.data.valid[0]) // self.batch_size)
        self.best_err, self.bad_counter, self.patience = 1.0, 0, config.get("patience", patience)
        self._val_errs = []
        self._train_it = None

    def make_torch_optimizer(self, params):
        return torch.optim.Adadelta(params, lr=1.0, rho=0.95, eps=1e-6)

    def compile_iter_fns(self, sync_type="avg", **kw):
        self.setup_train_options()
        self.sync_type = "avg"
        self.torch_opt = self.make_torch_optimizer(self.params)
        self.vels, self.vels2 = [], []

    def _to(self, x, m, y):
        d = self.device
        return torch.from_numpy(x).to(d), torch.from_numpy(m).to(d), torch.from_numpy(y).to(d)

    def train_iter(self, count, recorder):
        if self._train_it is None:
            self._train_it = self.data.batches("train", self.batch_size, True, seed=self.epoch)
        try:
            x, m, y = next(self._train_it)
        except StopIteration:
            self._train_it = self.data.batches("train", self.batch_size, True, seed=self.epoch + 1000)
            x, m, y = next(self._train_it)
        recorder.start()
        x, m, y = self._to(x, m, y)
        self.module.train()
        self.arena.G.zero_()
        for p in self.params:
            p.grad = p.gbuf
        logits = self.module(x, m)
        cost = nn.functional.cross_entropy(logits, y, label_smoothing=self.label_smoothing)
        cost.backward()
        self.torch_opt.step()
        err = (logits.argmax(1) != y).float().mean()
        recorder.train_error(count, cost.detach(), err)
        recorder.end("calc")

    def val_iter(self, count, recorder):
        """One full validation pass; returns ``'stop'`` when patience runs out (the early-stop
        protocol ``BSP_run`` understands, ``worker.py:118-126``)."""
        self.module.eval()
        errs, costs = [], []
        with torch.no_grad():
            for x, m, y in self.data.batches("valid", min(self.batch_size, len(self.data.valid[0])), False):
                x, m, y = self._to(x, m, y)
                lg = self.module(x, m)
                costs.append(float(nn.functional.cross_entropy(lg, y)))
                errs.append(float((lg.argmax(1) != y).float().mean()))
        e, c = float(np.mean(errs)), float(np.mean(costs))
        recorder.val_error(count, c, e, 0)
        if e < self.best_err:
            self.best_err, self.bad_counter = e, 0
        else:
            self.bad_counter += 1
            if self.bad_counter > self.patience:
                return "stop"
        return self.data.n_batch_val            # one call covers the whole validation set

    def reset_iter(self, mode):
        if mode == "train":
            self._train_it = None

    def adjust_hyperp(self, epoch):
        pass

    def cleanup(self):
        pass
