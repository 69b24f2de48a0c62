"""What gradient accumulation (``grad_accum``) costs: training windows of n micro-steps against single steps.

    python scripts/bench_grad_accum.py [--windows 20] [--rounds 3]

Rows (CUDA graphs on, device-resident synthetic batches; every model is built once and the rows are timed in ``--rounds`` alternating
rounds of ``--windows`` windows each, CUDA events around each round):

  a. AlexNet bf16, grad_accum = 1, batch 128 (the default path: FC weights updated in their wgrad GEMM epilogue)
  b. AlexNet bf16, grad_accum = 4, batch 32
  c. AlexNet bf16, grad_accum = 4, batch 128
  d. (c) through the library route: on the mid and last micro-steps every parameter is flagged ``gaccum``, so each gradient is
     stored into a fresh, uninitialised scratch buffer and added into G by a library ``add_``; the first micro-step stores into G
     as in (c).  It computes what (c) computes (tests/test_gpu_grad_accum.py checks it bit for bit in deterministic mode).
  e. ResNet50, grad_accum = 4, batch 64, LARS
  f. Wide_ResNet (28-4), grad_accum = 4, batch 128, Adam

With grad_accum > 1 the FC epilogue is never armed, so (c) is also "(c) with the FC epilogue disarmed".  Printed per row: ms per
micro-step and per update (the best round), images per second, and the peak of ``torch.cuda.max_memory_allocated`` while the row's
model was built, warmed up and captured (its three micro-step graphs share one pool).  The card's name, power limit and SM clock are
printed by the same run, before and after the measurements; one JSON line per row.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_lamb import card  # noqa: E402

IMNET = dict(n_class=1000, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True))


def build(name, mod, cls, n, B, library=False, **cfg):
    import importlib
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    m = getattr(importlib.import_module(mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=B,
                                                        file_batch_size=n * B, cuda_graph=True, grad_accum=n, **cfg))
    m.compile_iter_fns("avg")
    if library:
        body = m._step_body

        def library_body(kind):
            # the flag is read when each micro-step kind's graph is captured
            for p in m.arena.params:
                p.gaccum = kind != "first"
            try:
                return body(kind)
            finally:
                for p in m.arena.params:
                    p.gaccum = False

        m._step_body = library_body
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 10, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))

    def window():
        for i in range(n):
            m.train_iter_fn(i % m.n_subb)

    for _ in range(4):                                   # eager warm-up of every micro-step kind, then the captures
        window()
    torch.cuda.synchronize()
    peak = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    return dict(name=name, model=m, window=window, n=n, B=B, peak_gib=peak, ms=[])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--windows", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    print("card before:", card())
    alex = ("theanompi_b200.models.alex_net", "AlexNet")
    rows = [build("a AlexNet n=1 B=128", *alex, 1, 128, **IMNET),
            build("b AlexNet n=4 B=32", *alex, 4, 32, **IMNET),
            build("c AlexNet n=4 B=128", *alex, 4, 128, **IMNET),
            build("d AlexNet n=4 B=128 library add_", *alex, 4, 128, library=True, **IMNET),
            build("e ResNet50 n=4 B=64 LARS", "theanompi_b200.models.lasagne_model_zoo.resnet50", "ResNet50", 4, 64, optimizer="lars",
                  no_paraload=True, **IMNET),
            build("f Wide_ResNet n=4 B=128 Adam", "theanompi_b200.models.keras_model_zoo.wresnet", "Wide_ResNet", 4, 128,
                  data_kwargs=dict(n_synthetic=1024, synthetic=True))]
    for r in rows:
        assert r["model"].use_graph, r["name"] + ": the micro-step graphs were not captured"
    for _ in range(args.rounds):
        for r in rows:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.windows):
                r["window"]()
            e1.record()
            torch.cuda.synchronize()
            r["ms"].append(e0.elapsed_time(e1) / args.windows)
    for r in rows:
        best = min(r["ms"])
        print(json.dumps(dict(row=r["name"], ms_per_update=round(best, 3), ms_per_micro_step=round(best / r["n"], 3),
                              images_per_s=round(r["n"] * r["B"] * 1000.0 / best, 1), rounds_ms=[round(v, 3) for v in r["ms"]],
                              peak_gib=round(r["peak_gib"], 2), n_updates=r["model"].n_updates)))
    print("card after:", card())


if __name__ == "__main__":
    main()
