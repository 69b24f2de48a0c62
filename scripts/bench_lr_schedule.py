"""What a per-update learning-rate schedule (``lr_schedule``) costs: AlexNet-128b bf16 training steps with SGD, schedule off against
warm-up + cosine, and the native launches of one step of each.

    python scripts/bench_lr_schedule.py [--steps 50] [--rounds 3]

Two models in one process (``train_iter_fn`` on a device-resident batch, CUDA graph on), ``--rounds`` alternating windows of
``--steps`` steps each, timed with CUDA events (``scripts/bench_lamb.py: timed``).  The scheduled step adds one single-thread launch
(``lr_schedule_kernel``) to the captured graph; the launch counts are taken from one eager step of each model.  The card's name,
power limit and SM clock are printed by the same run, before and after the measurements.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_grad_clip import alexnet, alternate  # noqa: E402
from scripts.bench_lamb import card  # noqa: E402

SCHED = dict(warmup_steps=500, decay="cosine", total_steps=10000)


def launches(**kw):
    """Native launches of one eager AlexNet-128b step."""
    from theanompi_b200.ops import native
    m = alexnet(**kw)
    m.use_graph = False                               # count the launches one by one
    m.train_iter_fn(0)
    torch.cuda.synchronize()
    native.reset_launch_count()
    m.train_iter_fn(0)
    torch.cuda.synchronize()
    n = native.launch_count()
    m.cleanup()
    return n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_lr_schedule.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    models = {"sgd": alexnet(), "sgd_warmup_cosine": alexnet(lr_schedule=SCHED)}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
    res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
    sched = models["sgd_warmup_cosine"].lr_sched
    print(json.dumps({"alexnet_b128_ms_per_step": res, "schedule": SCHED, "updates": int(sched.u), "lr_last": sched.value()}))
    for mm in models.values():
        mm.cleanup()
    del models
    torch.cuda.empty_cache()
    print(json.dumps({"native_launches_per_step": {"sgd": launches(), "sgd_warmup_cosine": launches(lr_schedule=SCHED)}}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
