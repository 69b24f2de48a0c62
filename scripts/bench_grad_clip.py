"""What global gradient-norm clipping (``grad_clip``) costs: the norm launches alone, AlexNet-128b training steps and LSTM steps.

    python scripts/bench_grad_clip.py [--iters 200] [--steps 50] [--rounds 3]

1. The two norm launches alone (``cuda_impl.grad_clip_norm``: per-block sums of squares of G, one-CTA fp64 finalize) on the AlexNet
   and LSTM arenas (sizes from building the models; no data is read), CUDA events over ``--iters`` back-to-back calls after a
   warm-up.  Bytes are what they must move at least: 4 B per arena element (G) and 8 B per 1024-element block (the partial sum,
   written and read back).
2. AlexNet-128b training steps (``train_iter_fn`` on a device-resident batch, CUDA graph on) with the default SGD against SGD with
   ``grad_clip``: two models in one process, ``--rounds`` alternating windows of ``--steps`` steps each.  The clipped model also
   loses the FC weight-gradient GEMM epilogue (its FC weights are updated by the flat pass instead).
3. LSTM steps (the default Adadelta, dim 128, batch 16, one 64-step bucket graph) without and with ``grad_clip``, alternating.

The card's name, power limit and SM clock are printed by the same run, before and after the measurements.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_lamb import card, timed  # noqa: E402

CLIP = 1.0


def alexnet(**kw):
    from theanompi_b200.models.alex_net import AlexNet
    m = AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, cuda_graph=True,
                     data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True), **kw))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 16, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


def lstm(**kw):
    """An LSTM with one staged 64-step batch; returns the model and its captured-step callable."""
    from theanompi_b200.models.lstm import LSTM
    m = LSTM(dict(verbose=False, rank=0, size=1, device="cuda:0", cuda_graph=True, data_kwargs=dict(n_synthetic=512, n_words=10000),
                  **kw))
    m.compile_iter_fns("avg")
    rs = np.random.RandomState(0)
    x = rs.randint(2, 10000, (m.batch_size, 64)).astype(np.int64)
    mk = np.ones((m.batch_size, 64), dtype=np.float32)
    y = rs.randint(0, 2, m.batch_size).astype(np.int64)
    Tb, (xs, ms, ys) = m._stage(x, mk, y)
    torch.cuda.synchronize()
    return m, lambda: m.run_keyed_step(Tb, lambda: m._train_body(xs, ms, ys))


def norm_launches(name, a, iters):
    from theanompi_b200.ops import cuda_impl
    a.G.normal_(0, 1e-3)
    partial = torch.zeros(a.n_blocks, device="cuda:0")
    rec = torch.zeros(4, device="cuda:0")
    skipped = torch.zeros(1, dtype=torch.int64, device="cuda:0")
    t = timed(lambda: cuda_impl.grad_clip_norm(a, a.G, CLIP, partial, rec, skipped), iters)
    n, nb = a.numel, a.n_blocks
    print(json.dumps({"arena": name, "arena_elements": n, "blocks": nb, "params": a.n_real, "grad_clip_norm_us": round(t * 1e3, 1),
                      "grad_clip_norm_GBps": round((4 * n + 8 * nb) / t / 1e6, 1)}))


def alternate(fns, rounds, steps):
    res = {k: [] for k in fns}
    for _ in range(rounds):
        for k, fn in fns.items():
            res[k].append(round(timed(fn, steps, warmup=3), 3))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grad_clip.py needs a CUDA device")
    print(json.dumps({"card": card()}))

    # ---- 1. the norm launches on the AlexNet and LSTM arenas
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lstm import LSTM
    for name, build in (("alexnet", lambda: AlexNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128,
                                                          file_batch_size=128, data_kwargs=dict(n_train_files=2, n_val_files=1,
                                                                                                synthetic=True)))),
                        ("lstm", lambda: LSTM(dict(verbose=False, rank=0, size=1, device="cuda:0",
                                                   data_kwargs=dict(n_synthetic=64, n_words=10000))))):
        m = build()
        norm_launches(name, m.arena, args.iters)
        m.cleanup()
        del m
        torch.cuda.empty_cache()

    # ---- 2. AlexNet-128b steps, SGD against SGD + grad_clip, alternating
    models = {"sgd": alexnet(), "sgd_grad_clip": alexnet(grad_clip=CLIP)}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
    armed = {k: sum(getattr(p, "sgd_epilogue", None) is not None for p in mm.arena.params) for k, mm in models.items()}
    res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
    print(json.dumps({"alexnet_b128_ms_per_step": res, "fc_epilogue_weights": armed,
                      "grad_norm_last_step": float(models["sgd_grad_clip"].clip_opt.grad_norm)}))
    for mm in models.values():
        mm.cleanup()
    del models
    torch.cuda.empty_cache()

    # ---- 3. LSTM steps (one bucket graph) without and with grad_clip, alternating
    (m0, f0), (m1, f1) = lstm(), lstm(grad_clip=CLIP)
    for f in (f0, f1):
        for _ in range(4):                            # two eager warm-ups, the capture, a replay
            f()
    torch.cuda.synchronize()
    res = alternate({"adadelta": f0, "adadelta_grad_clip": f1}, args.rounds, args.steps)
    print(json.dumps({"lstm_b16_t64_ms_per_step": res, "grad_norm_last_step": float(m1.opt.grad_norm)}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
