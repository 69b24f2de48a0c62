"""Two-GPU check of the per-update lr schedule over the fused BSP exchange, launched by tests/test_gpu_lr_schedule.py as

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 ... tests/mp_lr_schedule_gpu.py <sched | oracle> <out dir>

``sched``: Cifar10_model with a warm-up + multistep schedule (bit-exact on the device); ``oracle``: the schedule off and lr_at(u)
written with set_value before each step.  Every rank saves its lr sequence and its weights to <out dir>/<mode>_<rank>.pt.
"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SCHED = dict(warmup_steps=4, warmup_start=0.1, decay="multistep", milestones=[6, 8], gamma=0.5, total_steps=20)


def main():
    mode, out = sys.argv[1], sys.argv[2]
    local = int(os.environ.get("LOCAL_RANK", os.environ["RANK"]))
    from theanompi_b200.models import layers2
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.ops.reference import lr_at
    from theanompi_b200.worker import BSP_Worker
    worker = BSP_Worker("cuda%d" % local, "cdd", "fused")
    layers2.reseed()
    cfg = worker.model_config("Cifar10_model", batch_size=64, file_batch_size=64, learning_rate=0.01,
                              lr_schedule=SCHED if mode == "sched" else None, data_kwargs=dict(n_synthetic=2048, synthetic=True))
    model = Cifar10_model(cfg)
    layers2.Dropout.SetDropoutOff(); layers2.Crop.SetRandCropOff()
    worker.build(model, cfg)
    assert getattr(worker.exchanger, "fused", False), "not the fused exchange"
    lrs = []
    for u in range(10):
        if mode == "oracle":
            model.shared_lr.set_value(lr_at(u, 0.01, **SCHED))
        model.train_iter(u, worker.recorder)
        worker.exchanger.exchange(worker.recorder)
        lrs.append(float(model.arena.hyper[0]))
    torch.cuda.synchronize()
    want = [float(lr_at(u, 0.01, **SCHED)) for u in range(10)]
    assert lrs == want, (lrs, want)
    if hasattr(worker.exchanger, "sync_master"):
        worker.exchanger.sync_master()
    torch.cuda.synchronize()
    torch.save({"lrs": lrs, "W": model.arena.W.detach().cpu()}, os.path.join(out, "%s_%d.pt" % (mode, worker.rank)))
    worker.comm.Barrier()
    print("OK rank", worker.rank)
    worker.finalize()


if __name__ == "__main__":
    main()
