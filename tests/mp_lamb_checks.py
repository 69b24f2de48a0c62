"""Multi-process CPU (gloo) checks of the LAMB optimizer, launched by tests/test_lamb_cpu.py with RANK/WORLD_SIZE set.

    python tests/mp_lamb_checks.py <case>
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from mp_cpu_checks import _proc  # noqa: E402

LR = 0.01


def case_bsp_lamb():
    """2 ranks × batch 16, BSP cdd over 'ar' with optimizer='lamb': rank 0 saves the final weights for the single-process
    comparison in test_lamb_cpu.py."""
    from theanompi_b200.models import layers2
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.layers2 import Crop, Dropout
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    from theanompi_b200.utils.recorder import Recorder
    p = _proc()
    layers2.reseed()
    m = Cifar10_model(dict(verbose=False, rank=p.rank, size=p.size, device="cpu", batch_size=16, file_batch_size=16, learning_rate=LR,
                           optimizer="lamb", data_kwargs=dict(n_synthetic=640, synthetic=True)))
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    m.compile_iter_fns("cdd")
    ex = BSP_Exchanger(p.comm, None, "ar", "cdd", p.ctx, m)
    rec = Recorder(p.comm, 1000, "t", False, device="cpu")
    for i in range(6):
        m.train_iter(i, rec)
        ex.exchange(rec)
    ws = p.comm.allgather(m.arena.W.clone())
    assert torch.equal(ws[0], ws[1]), "replicas diverged"
    if p.rank == 0:
        torch.save({"W": m.arena.W.clone(), "trust": m.lamb.trust.clone(), "t": int(m.lamb.t)},
                   os.path.join(os.environ["TMPI_TEST_OUT"], "bsp_lamb.pt"))
    p.comm.Barrier()
    print("OK bsp lamb rank", p.rank)


if __name__ == "__main__":
    globals()["case_" + sys.argv[1]]()
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
