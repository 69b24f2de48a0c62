"""Multi-process CPU (gloo) checks of gradient-norm clipping, launched by tests/test_grad_clip_cpu.py with RANK/WORLD_SIZE set.

    python tests/mp_grad_clip_checks.py <case>
"""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from mp_cpu_checks import _proc  # noqa: E402


def case_cdd_refused_avg_clips():
    """2 ranks: BSP ``sync_type='cdd'`` with ``grad_clip`` is refused at compile time; ``'avg'`` over the split 'ar' strategy takes
    clipped local steps, and the replicas agree after the weight exchange."""
    from theanompi_b200.models import layers2
    from theanompi_b200.models.cifar10 import Cifar10_model
    from theanompi_b200.models.layers2 import Crop, Dropout
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    from theanompi_b200.utils.recorder import Recorder
    p = _proc()
    cfg = dict(verbose=False, rank=p.rank, size=p.size, device="cpu", batch_size=16, file_batch_size=16, learning_rate=0.01,
               grad_clip=0.5, data_kwargs=dict(n_synthetic=640, synthetic=True))
    layers2.reseed()
    m = Cifar10_model(cfg)
    try:
        m.compile_iter_fns("cdd")
    except ValueError as e:
        assert "sync_type='cdd' with 2 workers" in str(e) and "sync_type='avg'" in str(e), str(e)
    else:
        raise AssertionError("sync_type='cdd' with grad_clip was not refused")
    Dropout.SetDropoutOff(); Crop.SetRandCropOff()
    m.compile_iter_fns("avg")
    ex = BSP_Exchanger(p.comm, None, "ar", "avg", p.ctx, m)
    rec = Recorder(p.comm, 1000, "t", False, device="cpu")
    for i in range(3):
        m.train_iter(i, rec)
        ex.exchange(rec)
    assert m.clip_opt is not None and float(m.clip_opt.grad_norm) > 0.5      # the threshold is active
    ws = p.comm.allgather(m.arena.W.clone())
    assert torch.equal(ws[0], ws[1]), "replicas diverged"
    p.comm.Barrier()
    print("OK grad clip rank", p.rank)


if __name__ == "__main__":
    globals()["case_" + sys.argv[1]]()
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
