"""Rank processes of the native-GAN world-size-2 check (launched by tests/test_native_gan_cpu.py)."""
import sys

import torch
import torch.distributed as dist

from mp_cpu_checks import _proc


def case_native_gan_bsp():
    """Two ranks train NativeWGAN (critic_runs=2) and NativeLSGAN for 2 steps with the BSP weight-averaging exchange: the
    exchanged critic arenas end identical, the local generator arenas differ (each rank drew its own batches)."""
    from theanompi_b200.models.lasagne_model_zoo.lsgan import NativeLSGAN
    from theanompi_b200.models.lasagne_model_zoo.wgan import NativeWGAN
    from theanompi_b200.parallel.exchanger import BSP_Exchanger
    from theanompi_b200.utils.recorder import Recorder
    p = _proc()
    for cls, cfg in ((NativeWGAN, dict(critic_runs=2)), (NativeLSGAN, {})):
        m = cls(dict(verbose=False, rank=p.rank, size=p.size, device="cpu", data_kwargs=dict(n_synthetic=128), **cfg))
        m.compile_iter_fns("avg")
        ex = BSP_Exchanger(p.comm, None, "ar", "avg", p.ctx, m)
        rec = Recorder(p.comm, 1000, "t", False, device="cpu")
        c = 0
        for _ in range(2):
            c = m.train_iter(c, rec)
            ex.exchange(rec)
        ws = p.comm.allgather(m.arena.W.clone())
        assert torch.equal(ws[0], ws[1]), "critic replicas diverged (%s)" % cls.__name__
        gs = p.comm.allgather(m.gen_arena.W.clone())
        assert not torch.equal(gs[0], gs[1]), "generator arenas must stay local (%s)" % cls.__name__
    p.comm.Barrier()
    print("OK native gan rank", p.rank)


if __name__ == "__main__":
    globals()["case_" + sys.argv[1]]()
    if dist.is_initialized():
        dist.barrier()
        dist.destroy_process_group()
