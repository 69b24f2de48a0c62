"""BSP worker runtime — one OS process per GPU (ref ``theanompi/worker.py``).

    python -u -m theanompi_b200.worker <device> <sync_type> <exch_strategy> <modelfile> <modelclass> [cpulist]

Same loop as the reference's ``BSP_run`` (``worker.py:66-150``): Barrier; per epoch:
lr warm-up (``:34-63``), ``while batch_i < n_batch_train: for subb in n_subb: train_iter;
exchange``, print every 40 global file batches (5120 images), validation with the
early-``'stop'`` protocol, ``gather_val_info``, rank-0 recorder save + snapshot every 5
epochs, ``adjust_hyperp``, optional ``print_info``.

Differences: rendezvous via ``torch.distributed`` env vars instead of ``mpirun``; the
model gets an allocator for the peer-mapped symmetric arena; with a ``fused*`` strategy
the exchange + optimizer update is part of the (CUDA-graph-captured) step; an optional
``resume`` checkpoint restores weights + momentum + lr + epoch (SURVEY §5.4).
"""
from __future__ import annotations

import os
import sys

import numpy as np

from .parallel.base import MPI_GPU_Process
from .parallel.exchanger import FUSED


class BSP_Worker(MPI_GPU_Process):
    def __init__(self, device, sync_type="cdd", exch_strategy="fused"):
        MPI_GPU_Process.__init__(self, device)
        self.get_intranode_comm()
        self.sync_type = sync_type
        self.exch_strategy = exch_strategy
        self.verbose = (self.rank == 0)
        if self.size == 1:
            self.sync_type = "avg"                         # tmlauncher does the same (``bin/tmlauncher:335-338``)
        self.needs_arena = (self.kind == "cuda" and self.size > 1 and
                            (exch_strategy in FUSED or exch_strategy == "p2p32"))

    def arena_allocator(self):
        """Allocator for the model's flat arena inside peer-mapped symmetric memory."""
        if not self.needs_arena:
            return None
        from .parallel.symmetric import SymmetricComm
        self.gpucomm = SymmetricComm(self.comm, self.ctx, None, local_ranks=self.local_ranks)
        return self.gpucomm.alloc

    def model_config(self, modelclass, **extra):
        cfg = dict(verbose=self.verbose, rank=self.rank, size=self.size, mname=modelclass,
                   device=str(self.ctx), arena_allocator=self.arena_allocator())
        cfg.update(extra)
        return cfg

    def build(self, model, config):
        from .utils.helper_funcs import check_model
        from .utils.recorder import Recorder
        from .parallel.exchanger import BSP_Exchanger
        check_model(model)
        self.recorder = Recorder(self.comm, printFreq=config.get("printFreq", 40), modelname=config["mname"],
                                 verbose=self.verbose, device=self.ctx)
        fused = self.size > 1 and self.exch_strategy in FUSED
        if fused:
            # the exchanger supplies the step tail (allreduce + SGD kernels) → needs the arena only
            self.exchanger = BSP_Exchanger(self.comm, self.gpucomm, self.exch_strategy, self.sync_type, self.ctx, model,
                                           nccl_group=None, overlap=config.get("overlap", True),
                                           bucket_bytes=config.get("bucket_bytes"), comm_blocks=config.get("comm_blocks"))
            model.compile_iter_fns(sync_type=self.sync_type, fused_tail=self.exchanger.fused_step)
        else:
            model.compile_iter_fns(sync_type=self.sync_type)
            self.exchanger = BSP_Exchanger(self.comm, self.gpucomm, self.exch_strategy, self.sync_type, self.ctx, model,
                                           nccl_group=self.nccl() if self.kind == "cuda" else None)
        model.exchanger = self.exchanger
        if config.get("resume"):
            from .utils.helper_funcs import load_checkpoint
            self.start_epoch = load_checkpoint(model, config["resume"], self.recorder)
            if self.verbose:
                print("resumed from %s at epoch %d" % (config["resume"], self.start_epoch))
        else:
            self.start_epoch = 0

    def lr_warmup(self, model, epoch):
        """Geometric warm-up lr → lr·size over 5 epochs (ref ``worker.py:34-63``).  A model with a per-update ``lr_schedule`` states
        the peak lr for the global batch itself: the schedule owns lr and nothing is scaled here."""
        if getattr(model, "lr_sched", None) is not None:
            if self.verbose:
                print("per-update lr schedule: lr %f at the last update before epoch %d" % (model.shared_lr.get_value(), epoch))
            return
        if epoch == 0:
            self.warmup_epochs = 5.0
            self.power_base = pow(self.size, 1.0 / self.warmup_epochs)
            if self.verbose:
                print("calculating lr warming up power base: %.3f" % self.power_base)
        elif epoch <= self.warmup_epochs:
            current_lr = model.shared_lr.get_value()
            if self.verbose:
                print("warming up lr from %f to %f" % (current_lr, current_lr * self.power_base))
            model.shared_lr.set_value(np.float32(current_lr * self.power_base))
        if self.verbose:
            print("learning rate %f will be used for epoch %d" % (model.shared_lr.get_value(), epoch))

    def _validate(self, model, recorder, n_val, count):
        """One pass over the first ``n_val`` validation files (the early-'stop' protocol sets ``self.stop``)."""
        batch_j = 0
        while batch_j < n_val:
            for subb_i in range(model.n_subb):
                out = model.val_iter(count, recorder)
                if out == "stop":
                    self.stop = True
                    break
                elif out is not None:
                    batch_j = out
                else:
                    batch_j += 1
            if self.stop:
                break
        model.reset_iter("val")

    def BSP_run(self, model, snapshot_freq=5, snapshot_path="./snapshots/", max_batches=None):
        from .utils.helper_funcs import save_model
        self.comm.Barrier()
        exchange_freq = 1
        recorder, exchanger = self.recorder, self.exchanger
        self.stop = False
        if not hasattr(self, "warmup_epochs"):
            self.warmup_epochs, self.power_base = 5.0, pow(self.size, 1.0 / 5.0)
        for epoch in range(self.start_epoch, model.n_epochs):
            model.epoch = epoch
            recorder.start_epoch()
            self.lr_warmup(model, epoch)
            self.comm.Barrier()
            exch_iteration = 0
            batch_i = 0
            n_train = model.data.n_batch_train if max_batches is None else min(max_batches, model.data.n_batch_train)
            while batch_i < n_train:
                for subb_i in range(model.n_subb):
                    model.train_iter(batch_i, recorder)
                    if exch_iteration % exchange_freq == 0:
                        exchanger.exchange(recorder)
                    exch_iteration += 1
                batch_i += 1
                recorder.print_train_info(batch_i * self.size)
            recorder.clear_train_info()
            model.reset_iter("train")

            self.comm.Barrier()
            n_val = model.data.n_batch_val if max_batches is None else min(max_batches, model.data.n_batch_val)
            self._validate(model, recorder, n_val, batch_i * self.size)
            if getattr(model, "ema", None) is not None and not self.stop:
                # config['model_ema']: the same validation files again on the averaged weights, into the recorder's EMA channel
                with model.ema_weights(), recorder.ema_channel():
                    self._validate(model, recorder, n_val, batch_i * self.size)
            recorder.gather_val_info()
            recorder.print_val_info(batch_i * self.size)
            model.current_info = recorder.get_latest_val_info()
            if self.rank == 0:
                recorder.save(batch_i * self.size, model.shared_lr.get_value() if hasattr(model, "shared_lr") else 0)
            # lr schedule BEFORE the snapshot: ckpt_<epoch> must carry the lr epoch+1 will train with (every lr_step of the
            # zoo is a multiple of snapshot_freq — saving first would lose that decay on resume)
            model.adjust_hyperp(epoch)
            if epoch % snapshot_freq == 0:
                if hasattr(exchanger, "sync_master"):
                    exchanger.sync_master()               # owner-keeps-master: rank 0 is about to read every fp32 weight
                if self.rank == 0:
                    save_model(model, snapshot_path, verbose=self.verbose, recorder=recorder)
            # rank 0 may have spent seconds writing files: park everybody on the HOST here — the next fused step spins in a
            # device-side flag barrier, which is the wrong place to wait for a slow disk
            self.comm.Barrier()
            if hasattr(model, "print_info"):
                model.print_info(recorder, verbose=self.verbose)
            recorder.end_epoch(batch_i * self.size, epoch)
            if self.stop:
                break
        if hasattr(exchanger, "sync_master"):
            exchanger.sync_master()
        model.cleanup()


def load_model_class(modelfile, modelclass):
    import importlib
    mod = importlib.import_module(modelfile)
    return getattr(mod, modelclass)


def main(argv=None):
    argv = list(sys.argv[1:] if argv is None else argv)
    device, sync_type, exch_strategy, modelfile, modelclass = argv[:5]
    if len(argv) > 5 and argv[5]:
        from .parallel.hwloc_utils import bind_to_socket_mem, detect_socket_num
        bind_to_socket_mem(argv[5], label="train")
        detect_socket_num(debug=True, label="train")
    worker = BSP_Worker(device, sync_type, exch_strategy)
    extra = {}
    if os.environ.get("TMPI_MODEL_CONFIG"):
        import json
        extra = json.loads(os.environ["TMPI_MODEL_CONFIG"])
    config = worker.model_config(modelclass, **extra)
    model = load_model_class(modelfile, modelclass)(config)
    worker.build(model, config)
    worker.BSP_run(model, max_batches=config.get("max_batches"))
    worker.finalize()


if __name__ == "__main__":
    main()
