"""Multi-process CPU (gloo) checks of the per-update lr schedule, launched by tests/test_lr_schedule_cpu.py with RANK/WORLD_SIZE set.

    python tests/mp_lr_schedule_checks.py <case>
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from mp_cpu_checks import _proc  # noqa: E402

SCHED = dict(warmup_steps=3, decay="cosine", total_steps=10, final_lr=0.001)


def case_bsp_cdd():
    """2 ranks, BSP ``sync_type='cdd'`` over the split 'ar' strategy for both aggregations (momentum: the scheduled lr enters in
    ``post``; gradient: also in ``post``) and without momentum (in ``pre``): every update's lr equals lr_at(u) on both ranks, the
    arena equals a schedule-off model that sets lr_at(u) by hand before each update, and the replicas agree."""
    from theanompi_b200.models import layers2
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.layers2 import Crop, Dropout
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    from theanompi_b200.utils.recorder import Recorder
    p = _proc()
    for aggregate, momentum in (("momentum", True), ("gradient", True), ("momentum", False)):
        arenas = []
        for sched in (SCHED, None):
            layers2.reseed()
            m = Cifar10_model(dict(verbose=False, rank=p.rank, size=p.size, device="cpu", batch_size=16, file_batch_size=16,
                                   learning_rate=0.05, lr_schedule=sched, data_kwargs=dict(n_synthetic=640, synthetic=True)))
            m.use_momentum = momentum
            Dropout.SetDropoutOff(); Crop.SetRandCropOff()
            m.compile_iter_fns("cdd", aggregate=aggregate)
            if sched is not None:
                oracle = m.lr_sched.lr_at
            ex = BSP_Exchanger(p.comm, None, "ar", "cdd", p.ctx, m)
            rec = Recorder(p.comm, 1000, "t", False, device="cpu")
            lrs = []
            for u in range(8):
                if sched is None:
                    m.shared_lr.set_value(oracle(u))
                m.train_iter(u, rec)
                ex.exchange(rec)
                lrs.append(float(m.arena.hyper[0]))
            want = [float(oracle(u)) for u in range(8)]
            assert lrs == want, (aggregate, momentum, lrs, want)
            arenas.append(m.arena.W.clone())
        assert torch.equal(arenas[0], arenas[1]), "scheduled run differs from the set_value oracle (%s, %s)" % (aggregate, momentum)
        ws = p.comm.allgather(arenas[0])
        assert torch.equal(ws[0], ws[1]), "replicas diverged"
    p.comm.Barrier()
    print("OK lr schedule rank", p.rank)


if __name__ == "__main__":
    globals()["case_" + sys.argv[1]]()
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
