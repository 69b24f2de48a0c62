"""Training/validation/time recorder.

Same schema and API as the reference (``theanompi/lib/recorder.py``):
``start()/end(mode)`` with the four buckets calc / sync / comm / wait (``:54-62``),
``train_error/val_error``, ``print_train_info`` every ``printFreq`` file batches
(= 5120 images for printFreq 40 × 128-image files, ``:90-124``),
``gather_val_info`` (``:137-150``), ``save/load/cut`` (``:181-224``), plotting
(``:226-473``).

H100-native differences:

* Timing is **device time**: ``start()`` / ``end(mode)`` record CUDA events on the
  current stream; durations are resolved lazily (one ``synchronize`` per print
  period instead of the reference's ``.sync()`` of every param after every
  iteration, ``alex_net.py:455-460``).  On CPU it falls back to ``time.time()``.
* The printed time split is the **max over ranks** (the reference printed rank
  0's wall clock only).
* Costs/errors may be 0-dim device tensors; they are only converted to floats
  at print time, so recording never stalls the stream.
"""
from __future__ import annotations

import contextlib
import os
import pickle
import time

import numpy as np
import torch


def _tofloat(v):
    if isinstance(v, torch.Tensor):
        return float(v.detach().float().cpu())
    return float(v)


class Recorder(object):
    MODES = ("calc", "sync", "comm", "wait")

    def __init__(self, comm, printFreq, modelname, verbose, device=None):
        self.t_start = None
        self.info_dict = {"train_info": [], "val_info": [], "epoch_time": [], "all_time": [], "lr": []}
        self.train_info = {"cost": [], "error": []}
        self.val_info = {"cost": [], "error": [], "error_top5": []}
        # the second validation channel: the same validation on the moving average of the model (config['model_ema']), logged as
        # info_dict['val_info_ema'] once a pass has recorded into it (ema_channel)
        self.val_info_ema = {"cost": [], "error": [], "error_top5": []}
        self._ema = False
        self.all_time = {m: [] for m in self.MODES}
        self._pending = {m: [] for m in self.MODES}     # (start_event, end_event)
        self.epoch_time = None
        self.verbose = verbose
        self.comm, self.printFreq, self.modelname = comm, printFreq, modelname
        self.use_cuda = torch.cuda.is_available() and (device is None or torch.device(device).type == "cuda")
        self.fig = None
        self.figsaxe = {}
        self.save_counter = 0
        self.last_period = None

    # ------------------------------------------------------------------ timers
    def start(self):
        if self.use_cuda:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self.t_start = ev
        else:
            self.t_start = time.time()

    def end(self, mode):
        if self.t_start is None:
            return
        if self.use_cuda:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            self._pending[mode].append((self.t_start, ev))
        else:
            self.all_time[mode].append(time.time() - self.t_start)
        self.t_start = None

    def add_time(self, mode, seconds):
        self.all_time[mode].append(float(seconds))

    def add_event_pair(self, mode, ev0, ev1):
        self._pending[mode].append((ev0, ev1))

    def _resolve(self):
        if not self.use_cuda:
            return
        any_pending = any(self._pending[m] for m in self.MODES)
        if any_pending:
            torch.cuda.synchronize()
        for m in self.MODES:
            for e0, e1 in self._pending[m]:
                self.all_time[m].append(e0.elapsed_time(e1) / 1000.0)
            self._pending[m] = []

    def start_epoch(self):
        self.epoch_time = time.time()

    def end_epoch(self, count, uepoch):
        duration = time.time() - self.epoch_time
        self.info_dict["epoch_time"].append([count, duration])
        if self.verbose:
            print("global epoch %d took %.4f h\n" % (uepoch, duration / 3600.0))
        self.epoch_time = None

    # ------------------------------------------------------------------ curves
    def train_error(self, count, cost, error):
        self.train_info["cost"].append(cost)
        self.train_info["error"].append(error)

    def val_error(self, count, cost, error, error_top5):
        info = self.val_info_ema if self._ema else self.val_info
        info["cost"].append(cost)
        info["error"].append(error)
        info["error_top5"].append(error_top5)

    @contextlib.contextmanager
    def ema_channel(self):
        """Inside the block :meth:`val_error` records into the EMA channel (``val_info_ema``)."""
        self._ema = True
        try:
            yield
        finally:
            self._ema = False

    def _max_over_ranks(self, vals):
        comm = self.comm
        if comm is None or getattr(comm, "size", 1) == 1:
            return vals
        allv = comm.allgather(list(vals))
        return [max(v[i] for v in allv) for i in range(len(vals))]

    def print_train_info(self, count):
        printFreq = self.printFreq
        if count % printFreq != 0 or not self.train_info["cost"]:
            return
        self._resolve()
        cost = sum(_tofloat(c) for c in self.train_info["cost"]) / len(self.train_info["cost"])
        error = sum(_tofloat(e) for e in self.train_info["error"]) / len(self.train_info["error"])
        self.info_dict["train_info"].append([count, cost, error])
        if self.verbose:
            print("")
            print("%d %f %f" % (count, cost, error))
        self.train_info["cost"][:] = []
        self.train_info["error"][:] = []
        calc, sync, comm, wait = self._max_over_ranks([sum(self.all_time[m]) for m in self.MODES])
        t_all = calc + sync + comm + wait
        self.info_dict["all_time"].append([count, t_all, calc, sync, comm, wait])
        self.last_period = dict(count=count, total=t_all, calc=calc, sync=sync, comm=comm, wait=wait)
        if self.verbose:
            print("time per %d batches: %.4f (train %.4f sync %.4f comm %.4f wait %.4f)"
                  % (printFreq, t_all, calc, sync, comm, wait))
        for m in self.MODES:
            self.all_time[m][:] = []

    def clear_train_info(self):
        self._resolve()
        self.train_info["cost"][:] = []
        self.train_info["error"][:] = []
        for m in self.MODES:
            self.all_time[m][:] = []

    def gather_val_info(self):
        """Gather both validation channels over the ranks; the EMA channel only when this epoch recorded into it (on every rank)."""
        for info in (self.val_info, self.val_info_ema):
            if info is self.val_info_ema and not info["cost"]:
                continue
            for k in ("cost", "error", "error_top5"):
                local = [_tofloat(v) for v in info[k]]
                if self.comm is not None and getattr(self.comm, "size", 1) > 1:
                    parts = self.comm.allgather(local)
                    local = [x for p in parts for x in p]
                info[k] = local

    def print_val_info(self, count, comment=None):
        for key, info, label in (("val_info", self.val_info, "validation"), ("val_info_ema", self.val_info_ema, "EMA validation")):
            if info is self.val_info_ema and not info["cost"]:
                continue
            n = max(1, len(info["cost"]))
            cost = sum(_tofloat(v) for v in info["cost"]) / n
            error = sum(_tofloat(v) for v in info["error"]) / n
            error_top5 = sum(_tofloat(v) for v in info["error_top5"]) / n
            self.info_dict.setdefault(key, []).append([count, cost, error, error_top5])
            if self.verbose:
                if comment is not None and info is self.val_info:
                    print(comment)
                print("\n%s cost:%.4f" % (label, cost))
                print("%s error:%.4f" % (label, error))
                print("%s top_5_error:%.4f" % (label, error_top5))
            for k in info:
                info[k][:] = []

    def get_latest_val_info(self):
        return self.info_dict["val_info"][-1] if self.info_dict["val_info"] else None

    # ------------------------------------------------------------------ persistence
    def save(self, count, lr, filepath="./inforec/"):
        os.makedirs(filepath, exist_ok=True)
        self.info_dict["lr"].append([count, float(lr)])
        with open(os.path.join(filepath, "inforec.pkl"), "wb") as f:
            pickle.dump(self.info_dict, f, protocol=pickle.HIGHEST_PROTOCOL)

    def load(self, filepath="./inforec/inforec.pkl"):
        with open(filepath, "rb") as f:
            d = pickle.load(f)
        for k in ("train_info", "val_info", "epoch_time", "all_time", "lr"):
            self.info_dict[k].extend(d.get(k, []))
        if "val_info_ema" in d:
            self.info_dict.setdefault("val_info_ema", []).extend(d["val_info_ema"])

    def cut(self, load_epoch):
        """Truncate curves to ``load_epoch`` entries when resuming (ref ``:212-224``)."""
        for k in ("train_info", "val_info", "val_info_ema", "epoch_time", "all_time", "lr"):
            if k in self.info_dict:
                self.info_dict[k] = self.info_dict[k][0:load_epoch]

    # ------------------------------------------------------------------ plotting (matplotlib optional)
    def plot_init(self, name, fig_specs=None, save=False):
        try:
            import matplotlib
            if save:
                matplotlib.use("Agg")
            import matplotlib.pyplot as plt
        except Exception:
            self.fig = None
            return False
        if self.fig is None:
            self.fig = plt.figure()
        idx = len(self.figsaxe) + 1
        ax = self.fig.add_subplot(1, max(idx, 1), idx)
        if fig_specs:
            ax.set_xlabel(fig_specs.get("xlabel", "")); ax.set_ylabel(fig_specs.get("ylabel", ""))
        self.figsaxe[name] = ax
        self._plot_save = save
        return True

    def plot(self, name, image=None, cmap="gray", lines=None, show=False):
        if self.fig is None or name not in self.figsaxe:
            return
        ax = self.figsaxe[name]
        ax.clear()
        if image is not None:
            ax.imshow(image, cmap=cmap)
        if lines is not None:
            for xs, ys, label in lines:
                ax.plot(xs, ys, label=label)
            ax.legend()
        if getattr(self, "_plot_save", False):
            os.makedirs("./inforec/", exist_ok=True)
            self.fig.savefig("./inforec/%s_%d.png" % (name.strip(), self.save_counter))
            self.save_counter += 1

    def show(self, label="", color_id=0, show=True, save=None):
        """Offline five-panel report: train cost/error, val cost/error/top-5 and the
        'time per 5120 images' split (ref ``recorder.py:328-473``)."""
        try:
            import matplotlib
            if not show:
                matplotlib.use("Agg")
            import matplotlib.pyplot as plt
        except Exception:
            print("matplotlib unavailable; summary only")
            return self.summary()
        d = self.info_dict
        fig, axs = plt.subplots(1, 5, figsize=(22, 4))
        if d["train_info"]:
            t = np.array(d["train_info"]); axs[0].plot(t[:, 0], t[:, 1], label=label); axs[0].set_title("train cost")
            axs[1].plot(t[:, 0], t[:, 2], label=label); axs[1].set_title("train error")
        if d["val_info"]:
            v = np.array(d["val_info"]); axs[2].plot(v[:, 0], v[:, 1], label=label); axs[2].set_title("val cost")
            axs[3].plot(v[:, 0], v[:, 2], label="top1"); axs[3].plot(v[:, 0], v[:, 3], label="top5")
            axs[3].set_title("val error"); axs[3].legend()
        if d["all_time"]:
            a = np.array(d["all_time"])
            for i, m in enumerate(("total", "calc", "sync", "comm", "wait")):
                axs[4].plot(a[:, 0], a[:, 1 + i], label=m)
            axs[4].set_title("time per %d images" % (self.printFreq * 128)); axs[4].legend()
        if save:
            fig.savefig(save)
        if show:
            plt.show()
        return self.summary()

    def summary(self):
        d = self.info_dict
        out = {"n_train_points": len(d["train_info"]), "n_val_points": len(d["val_info"])}
        if d["all_time"]:
            a = np.array(d["all_time"])
            out["mean_time_per_period"] = dict(zip(("total", "calc", "sync", "comm", "wait"),
                                                    a[:, 1:].mean(0).tolist()))
        if d["val_info"]:
            out["last_val"] = d["val_info"][-1]
        return out
