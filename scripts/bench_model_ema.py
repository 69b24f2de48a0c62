"""What the model EMA (``model_ema``) costs: the ``ema_update`` pass alone on AlexNet's and ResNet50's arenas, in average and skip mode,
and AlexNet-128b and ResNet50 training steps with the key off, averaging every update and every 32 updates.

    python scripts/bench_model_ema.py [--iters 200] [--steps 50] [--rounds 3]

1. ``ema_update`` over each arena (CUDA events over ``--iters`` launches, after 10 warm-up launches); the achieved bandwidth counts
   12 B per arena element (read W and E, write E) in average mode.  A skip launch returns before it touches memory.
2. ``train_iter_fn`` on a device-resident batch with the CUDA graph on, the three variants of a model in one process, ``--rounds``
   alternating windows of ``--steps`` steps each (``scripts/bench_grad_clip.py: alternate``).

Needs a CUDA device.  The card's name, power limit and SM clock are printed by the same run, before and after the measurements.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_grad_clip import alexnet, alternate  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402

VARIANTS = {"off": None, "every1": dict(decay=0.9999, every=1), "every32": dict(decay=0.99998, every=32)}


def resnet50(**kw):
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    m = ResNet50(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=64, file_batch_size=64, cuda_graph=True,
                      data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True), **kw))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 16, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


def update_pass(build, iters):
    """``ema_update`` alone over the model's arena: ms per launch and TB/s in average and skip mode."""
    from theanompi_b200.ops import cuda_impl, reference as ref
    m = build(model_ema=dict(decay=0.99998))
    e, a = m.ema, m.arena
    e._ensure_table()
    out = {"arena_elements": a.numel, "bn_elements": int(e.E_bn.numel())}
    for name, mode in (("average", ref.EMA_AVERAGE), ("skip", ref.EMA_SKIP)):
        e.state[2] = mode
        ms = timed(lambda: cuda_impl.ema_update(a, e.E, e.state, e._table, e.decay, e.one_minus_decay), iters)
        out[name + "_ms"] = round(ms, 4)
        if mode == ref.EMA_AVERAGE:
            out["average_TBps"] = round(12.0 * (a.numel + e.E_bn.numel()) / (ms * 1e-3) / 1e12, 3)
    m.cleanup()
    return out


def steps(build, args):
    models = {k: build(model_ema=v) for k, v in VARIANTS.items()}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
    res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
    for mm in models.values():
        mm.cleanup()
    del models
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_model_ema.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for name, build in (("alexnet_b128", alexnet), ("resnet50_b64", resnet50)):
        print(json.dumps({name + "_ema_update": update_pass(build, args.iters)}))
    for name, build in (("alexnet_b128", alexnet), ("resnet50_b64", resnet50)):
        print(json.dumps({name + "_ms_per_step": steps(build, args)}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
