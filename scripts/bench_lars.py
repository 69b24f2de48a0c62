"""What LARS costs over momentum SGD on AlexNet (bf16).

    python scripts/bench_lars.py [--iters 200] [--steps 50] [--rounds 3]

1. The optimizer passes alone, on the AlexNet arena (sizes from building the model; no data is read): ``sgd_flat`` over the whole
   arena against a LARS step (per-block sums of squares, per-tensor finalize, the LARS update pass), CUDA events over ``--iters``
   back-to-back calls after a warm-up.  Bytes are what each must move at least, from the arena size n (padded elements) and the
   block count: sgd_flat reads W, U, G and writes W, U and the bf16 shadow (22 B per element); LARS adds a read of W and G (8 B per
   element) and 8 B per block of partial sums written and read.
2. AlexNet-128b training steps (``train_iter_fn`` on a device-resident batch, CUDA graph on) with ``optimizer='sgd'`` against
   ``'lars'``: two models in one process, ``--rounds`` alternating windows of ``--steps`` steps each.  The SGD model runs its FC
   weight update in the weight-gradient GEMM epilogue; LARS cannot.

The card's name, power limit and SM clock are printed by the same run, before and after the measurements.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def timed(fn, iters, warmup=10):
    for _ in range(warmup):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def alexnet(optimizer):
    from theanompi_b200.models import layers2
    from theanompi_b200.models.alex_net import AlexNet
    layers2.reseed()
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, optimizer=optimizer,
                     cuda_graph=True, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x = torch.randn(tuple(m.shared_x.shape), device="cuda:0").to(m.act_dtype)
    m.shared_y.copy_(torch.randint(0, 1000, (m.shared_x.shape[0],), device="cuda:0"))
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lars.py needs a CUDA device")
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.opt import FlatLARS
    print(json.dumps({"card": card()}))

    # ---- 1. the optimizer passes on the AlexNet arena
    m = alexnet("lars")
    a = m.arena
    a.hyper[0] = 0.01
    a.G.normal_(0, 1e-3)
    lars = FlatLARS(a, 0.9, False, 0.001)
    t_sgd = timed(lambda: cuda_impl.sgd_flat(a, a.G, 0.01, 0.9, False, 1.0, 0, a.numel), args.iters)
    t_lars = timed(lambda: lars.step(), args.iters)
    t_norms = timed(lambda: cuda_impl.lars_trust(a, a.G, 1.0, 0.001, lars._partial, lars.norms, lars.trust), args.iters)
    n, nb = a.numel, a.n_blocks
    b_sgd, b_norms = 22 * n, 8 * n + 16 * nb
    print(json.dumps({"arena_elements": n, "params": a.n_real, "tensors": len(a.sizes),
                      "sgd_flat_us": round(t_sgd * 1e3, 1), "sgd_flat_GBps": round(b_sgd / t_sgd / 1e6, 1),
                      "lars_step_us": round(t_lars * 1e3, 1), "lars_step_GBps": round((b_sgd + b_norms) / t_lars / 1e6, 1),
                      "lars_norms_us": round(t_norms * 1e3, 1), "lars_norms_GBps": round(b_norms / t_norms / 1e6, 1)}))
    del m, a, lars

    # ---- 2. AlexNet-128b steps, SGD against LARS, alternating
    models = {o: alexnet(o) for o in ("sgd", "lars")}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    res = {o: [] for o in models}
    for _ in range(args.rounds):
        for o, mm in models.items():
            res[o].append(round(timed(lambda: mm.train_iter_fn(0), args.steps, warmup=3), 3))
    print(json.dumps({"alexnet128_ms_per_step": res, "armed_fc_weights_sgd": sum(getattr(p, "sgd_epilogue", None) is not None
                                                                                  for p in models["sgd"].arena.params)}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
