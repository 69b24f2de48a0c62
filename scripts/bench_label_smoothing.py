"""What label smoothing (``label_smoothing``) costs: the fused softmax / NLL kernel alone at ε = 0 against ε = 0.1, and AlexNet-128b bf16
training steps with and without it.

    python scripts/bench_label_smoothing.py [--calls 400] [--steps 50] [--rounds 3]

1. The native ``softmax_xent`` (the row kernel + the batch mean, two launches per call) at (B, C) in (32, 1000), (128, 1000),
   (256, 1000) and (16, 2), bf16 and fp32 logits, ε = 0 and ε = 0.1.  ``--calls`` calls on preallocated buffers are captured in one
   CUDA graph per ε, so the time is the device's and not the Python enqueue's; the graphs replay alternately in ``--rounds``
   windows of 25 replays, timed with CUDA events.  GB/s counts the minimum bytes: B·C logits read, B·C dlogits written, B int64 labels read.
2. AlexNet-128b models in one process (``train_iter_fn`` on a device-resident batch, CUDA graph on): ε = 0, ε = 0.1 and a second
   ε = 0 instance as a control for the spread between two models of the same configuration, in ``--rounds`` alternating windows of
   ``--steps`` steps, and the native launches of one eager step of each ε.
3. The card's name, power limit and SM clock, printed by the same run before and after the measurements.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_grad_clip import alexnet, alternate  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402
from scripts.bench_lr_schedule import launches  # noqa: E402

SHAPES = [(32, 1000), (128, 1000), (256, 1000), (16, 2)]
EPS = 0.1


def captured_calls(lg, lab, eps, calls):
    """One CUDA graph of ``calls`` native softmax_xent launches on static buffers."""
    from theanompi_b200.ops import cuda_impl
    B, C = lg.shape
    dl = torch.empty_like(lg)
    rowstat = torch.empty((B, 3), dtype=torch.float32, device=lg.device)
    out3 = torch.empty(3, dtype=torch.float32, device=lg.device)
    f32 = int(lg.dtype == torch.float32)

    def call():
        cuda_impl.L().softmax_xent(lg.data_ptr(), lab.data_ptr(), dl.data_ptr(), rowstat.data_ptr(), out3.data_ptr(), B, C, 1.0, 1.0,
                                   eps, f32, torch.cuda.current_stream().cuda_stream)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        call()                                        # load the module before the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            call()
    return g


def kernel_rows(calls, rounds):
    from theanompi_b200.ops import precision
    rows = []
    for mode in ("bf16", "tf32"):
        precision.set_precision(mode)
        dt = precision.act_dtype()
        for B, C in SHAPES:
            torch.manual_seed(0)
            lg = (torch.randn(B, C, device="cuda:0") * 3).to(dt)
            lab = torch.randint(0, C, (B,), device="cuda:0")
            graphs = {eps: captured_calls(lg, lab, eps, calls) for eps in (0.0, EPS)}
            us = {eps: [] for eps in graphs}
            for _ in range(rounds):
                for eps, g in graphs.items():
                    us[eps].append(round(1e3 * timed(g.replay, 25, warmup=2) / calls, 3))     # 25 replays per window
            nbytes = 2 * B * C * lg.element_size() + 8 * B
            rows.append({"dtype": "bf16" if mode == "bf16" else "fp32", "B": B, "C": C, "min_bytes": nbytes,
                         "us_per_call": {str(k): v for k, v in us.items()},
                         "GB_per_s_best": {str(k): round(nbytes / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    precision.set_precision("bf16")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=400)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_label_smoothing.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"softmax_xent": row}))
    models = {"eps0": alexnet(), "eps0.1": alexnet(label_smoothing=EPS), "eps0_control": alexnet()}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
    res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
    print(json.dumps({"alexnet_b128_ms_per_step": res}))
    for mm in models.values():
        mm.cleanup()
    del models
    torch.cuda.empty_cache()
    print(json.dumps({"native_launches_per_step": {"eps0": launches(), "eps0.1": launches(label_smoothing=EPS)}}))
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
