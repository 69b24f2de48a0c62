"""What Mixup / CutMix (``mixup``) cost: the in-place mix kernel alone, the mixing softmax / NLL instantiation against the plain and
label-smoothing ones, and AlexNet-128b and WRN-28-4 training steps with Mixup and CutMix against steps without the key.

    python scripts/bench_mixup.py [--calls 200] [--steps 30] [--rounds 3]

1. ``mix_batch`` on a [128, 227, 227, 3] bf16 batch (the scalar path: 309,174-byte rows) and on [128, 32, 32, 3] bf16 and fp32
   batches (16-byte vectors), for a Mixup record (λ = 0.6), a CutMix record (a 136×136 box on 227², a 20×20 box on 32²) and an
   unmixed one.  ``--calls`` launches on a static batch are captured in one CUDA graph per record and replayed in ``--rounds``
   alternating windows of 10 replays, timed with CUDA events.  GB/s counts the minimum bytes: Mixup reads and writes the whole batch,
   CutMix reads and writes the box of both samples of every pair (4 · box bytes per pair).
2. The native ``softmax_xent`` at (B, C) = (128, 1000) and (256, 1000) in bf16: plain, label smoothing ε = 0.1 and mixing (ε = 0.1),
   ``--calls`` calls per CUDA graph, alternating windows as above.
3. AlexNet-128b bf16 and WRN-28-4 batch-128 ``train_iter_fn`` with the CUDA graph: off, Mixup (α = 0.2) and CutMix (α = 1.0) in
   ``--rounds`` alternating windows of ``--steps`` steps, and the native launches of one eager AlexNet step of each.
4. The card's name, power limit and SM clock, printed by the same run before and after the measurements.
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_grad_clip import alexnet, alternate  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402
from scripts.bench_lr_schedule import launches  # noqa: E402

MIX = {"off": None, "mixup": dict(alpha=0.2), "cutmix": dict(cutmix_alpha=1.0)}


def _graph(fn, calls):
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        fn()                                          # load the module before the capture
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(calls):
            fn()
    return g


def _record(mode, lam, box, hw):
    from theanompi_b200.ops import mixup
    r = np.zeros((), dtype=mixup.RECORD)
    r["mode"], r["lam"], r["lam_raw"], r["H"], r["W"] = mode, lam, lam, hw[0], hw[1]
    r["y0"], r["y1"], r["x0"], r["x1"] = box
    return mixup.encode(r).cuda()


def mix_rows(calls, rounds):
    from theanompi_b200.ops import cuda_impl, mixup
    rows = []
    for shape, dt, side in (((128, 227, 227, 3), torch.bfloat16, 136), ((128, 32, 32, 3), torch.bfloat16, 20),
                            ((128, 32, 32, 3), torch.float32, 20)):
        B, H, W, C = shape
        torch.manual_seed(0)
        x = torch.randn(shape, device="cuda:0").to(dt)
        y0, x0 = (H - side) // 2 + 3, (W - side) // 2 - 2
        recs = {"mixup": _record(mixup.MIX_MIXUP, 0.6, (0, 0, 0, 0), (H, W)),
                "cutmix": _record(mixup.MIX_CUTMIX, 1 - side * side / (H * W), (y0, y0 + side, x0, x0 + side), (H, W)),
                "none": _record(mixup.MIX_NONE, 1.0, (0, 0, 0, 0), (H, W))}
        graphs = {k: _graph(lambda r=r: cuda_impl.mix_batch(x, r), calls) for k, r in recs.items()}
        us = {k: [] for k in graphs}
        for _ in range(rounds):
            for k, g in graphs.items():
                us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
        esz = x.element_size()
        nbytes = {"mixup": 2 * x.numel() * esz, "cutmix": 4 * (B // 2) * side * side * C * esz, "none": 0}
        rows.append({"shape": list(shape), "dtype": str(dt).replace("torch.", ""),
                     "path": "vector" if (H * W * C * esz) % 16 == 0 else "scalar", "us_per_call": us, "min_bytes": nbytes,
                     "GB_per_s_best": {k: round(nbytes[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items() if nbytes[k]}})
    return rows


def softmax_rows(calls, rounds):
    from theanompi_b200.ops import cuda_impl, mixup
    rows = []
    rec = _record(mixup.MIX_MIXUP, 0.6, (0, 0, 0, 0), (32, 32))
    for B, C in ((128, 1000), (256, 1000)):
        torch.manual_seed(0)
        lg = (torch.randn(B, C, device="cuda:0") * 3).to(torch.bfloat16)
        lab = torch.randint(0, C, (B,), device="cuda:0")
        dl = torch.empty_like(lg)
        rowstat = torch.empty((B, 3), dtype=torch.float32, device="cuda:0")
        out3 = torch.empty(3, dtype=torch.float32, device="cuda:0")
        L, st = cuda_impl.L(), lambda: torch.cuda.current_stream().cuda_stream
        fns = {"plain": lambda: L.softmax_xent(lg.data_ptr(), lab.data_ptr(), dl.data_ptr(), rowstat.data_ptr(), out3.data_ptr(), B, C,
                                               1.0, 1.0, 0.0, 0, st()),
               "smooth0.1": lambda: L.softmax_xent(lg.data_ptr(), lab.data_ptr(), dl.data_ptr(), rowstat.data_ptr(), out3.data_ptr(), B,
                                                   C, 1.0, 1.0, 0.1, 0, st()),
               "mix_smooth0.1": lambda: L.softmax_xent_mix(lg.data_ptr(), lab.data_ptr(), rec.data_ptr(), dl.data_ptr(),
                                                           rowstat.data_ptr(), out3.data_ptr(), B, C, 1.0, 1.0, 0.1, 0, st())}
        graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
        us = {k: [] for k in graphs}
        for _ in range(rounds):
            for k, g in graphs.items():
                us[k].append(round(1e3 * timed(g.replay, 25, warmup=2) / calls, 3))
        rows.append({"dtype": "bf16", "B": B, "C": C, "us_per_call": us})
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mixup.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in mix_rows(args.calls, args.rounds):
        print(json.dumps({"mix_batch": row}))
    for row in softmax_rows(args.calls, args.rounds):
        print(json.dumps({"softmax_xent": row}))
    for name, build in (("alexnet_b128", lambda mx: alexnet(**({} if mx is None else dict(mixup=mx)))),
                        ("wrn28_4_b128_adam", wrn)):
        models = {k: build(mx) for k, mx in MIX.items()}
        for mm in models.values():
            for _ in range(5):                        # eager warm-up and the CUDA-graph capture
                mm.train_iter_fn(0)
        torch.cuda.synchronize()
        assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
        res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
        print(json.dumps({name + "_ms_per_step": res}))
        for mm in models.values():
            mm.cleanup()
        del models
        torch.cuda.empty_cache()
    print(json.dumps({"alexnet_native_launches_per_step": {k: launches(**({} if mx is None else dict(mixup=mx))) for k, mx in MIX.items()}}))
    print(json.dumps({"card_after": card()}))


def wrn(mx):
    """WRN-28-4, batch 128, Adam (bench_lamb.py's model), with ``config['mixup']`` = ``mx``."""
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    m = Wide_ResNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, cuda_graph=True, mixup=mx,
                         data_kwargs=dict(n_synthetic=256, synthetic=True)))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 10, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


if __name__ == "__main__":
    main()
