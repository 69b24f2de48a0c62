"""What LAMB costs over Adam: the optimizer passes on the Wide-ResNet and AlexNet arenas, and Wide-ResNet training steps (bf16).

    python scripts/bench_lamb.py [--iters 200] [--steps 50] [--rounds 3]

1. The optimizer passes alone, on the arenas of WRN-28-4 and AlexNet (sizes from building the models; no data is read): Adam
   (``adam_flat``, the update and the counter launch) against a LAMB step (moments and per-block sums of squares, per-tensor
   finalize, the LAMB update pass, the counter launch) and against its first two launches alone, CUDA events over ``--iters``
   back-to-back calls after a warm-up.  Bytes are what each must move at least, from the arena size n (padded elements) and the
   block count: Adam reads W, G, M, V and writes W, M, V and the bf16 shadow (30 B per element); LAMB's first pass reads W, G, M, V
   and writes M, V (24 B), its update pass reads W, M, V and writes W and the shadow (18 B), and the partial sums add 16 B per
   1024-element block.
2. WRN-28-4 training steps at batch 128 (``train_iter_fn`` on a device-resident batch, CUDA graph on) with the default Adam against
   ``optimizer='lamb'``: two models in one process, ``--rounds`` alternating windows of ``--steps`` steps each.

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


def wide_resnet(optimizer):
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    cfg = dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, cuda_graph=True,
               data_kwargs=dict(n_synthetic=256, synthetic=True))
    if optimizer != "adam":
        cfg["optimizer"] = optimizer
    m = Wide_ResNet(cfg)
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 10, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


def alexnet():
    from theanompi_b200.models.alex_net import AlexNet
    return AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128,
                        data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))


def passes(name, a, iters):
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.utils.opt import FlatAdam, FlatLAMB
    a.hyper[0] = 1e-3
    a.G.normal_(0, 1e-3)
    adam, lamb = FlatAdam(a), FlatLAMB(a)
    t_adam = timed(lambda: adam.step(), iters)
    t_lamb = timed(lambda: lamb.step(), iters)
    t_trust = timed(lambda: cuda_impl.lamb_trust(a, a.G, a.U, lamb.V, lamb.t, *lamb.hyper(), 1.0, 0, lamb._partial, lamb.norms,
                                                 lamb.trust), iters)
    n, nb = a.numel, a.n_blocks
    b_adam, b_trust, b_update = 30 * n, 24 * n + 16 * nb, 18 * n
    print(json.dumps({"arena": name, "arena_elements": n, "params": a.n_real, "tensors": len(a.sizes),
                      "adam_flat_us": round(t_adam * 1e3, 1), "adam_flat_GBps": round(b_adam / t_adam / 1e6, 1),
                      "lamb_step_us": round(t_lamb * 1e3, 1), "lamb_step_GBps": round((b_trust + b_update) / t_lamb / 1e6, 1),
                      "lamb_trust_us": round(t_trust * 1e3, 1), "lamb_trust_GBps": round(b_trust / t_trust / 1e6, 1)}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lamb.py needs a CUDA device")
    print(json.dumps({"card": card()}))

    # ---- 1. the optimizer passes on the Wide-ResNet and AlexNet arenas
    for name, build in (("wide_resnet_28_4", lambda: wide_resnet("lamb")), ("alexnet", alexnet)):
        m = build()
        passes(name, m.arena, args.iters)
        m.cleanup()
        del m
        torch.cuda.empty_cache()

    # ---- 2. WRN-28-4 batch-128 steps, Adam against LAMB, alternating
    models = {o: wide_resnet(o) for o in ("adam", "lamb")}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
    res = {o: [] for o in models}
    for _ in range(args.rounds):
        for o, mm in models.items():
            res[o].append(round(timed(lambda: mm.train_iter_fn(0), args.steps, warmup=3), 3))
    print(json.dumps({"wide_resnet_28_4_b128_ms_per_step": res}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
