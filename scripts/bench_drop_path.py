"""What stochastic depth (``drop_path_rate``) costs: the batch-norm kernels and the WRN merge kernels with and without a drop row, ResNet50
and WRN-28-4 training steps with drop-path against steps without it, and ``bench.py`` against another checkout.

    python scripts/bench_drop_path.py [--calls 100] [--steps 20] [--rounds 3] [--parent DIR]

1. ``bn_forward`` + ``bn_backward`` (training, ReLU, residual) in bf16 at ResNet50's bottleneck outputs for batch 64: (R, C) =
   (64·56², 256), (64·28², 512), (64·14², 1024), (64·7², 2048), with and without a drop row.  ``--calls`` pairs are captured in one
   CUDA graph per variant and replayed in ``--rounds`` alternating windows, timed with CUDA events.  GB/s counts the minimum bytes:
   forward reads x twice and the residual, writes y (4·R·C·2); backward reads x, dy, y twice and writes dx and dres (8·R·C·2); the
   row adds 3·4·B bytes.  The WRN-28-4 merges at batch 128 the same way: the plain ``add``, the scaled add y = s·a + b and the branch
   gradient s·dy (minimum bytes 3, 3 and 2 times the tensor).
2. ResNet50 batch 64 bf16 (p = 0 / 0.05 / 0.1) and WRN-28-4 batch 128 Adam (p = 0 / 0.1) ``train_iter_fn`` with the CUDA graph, in
   ``--rounds`` alternating windows of ``--steps`` steps, and the native launches of one eager step of each.
3. With ``--parent DIR`` (a built checkout): ResNet50 batch 64 bf16 graph steps without the key (one process per window of
   4·``--steps`` steps) and ``bench.py --gpus 1 --steps 50 --warmup 10``, each run from this checkout and from DIR, alternating,
   ``--rounds`` times each.
4. The card's name, power limit and SM clock, printed by the same run before and after the measurements.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_grad_clip import alternate  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402
from scripts.bench_mixup import _graph  # noqa: E402

BN_SHAPES = [(64 * 56 * 56, 256), (64 * 28 * 28, 512), (64 * 14 * 14, 1024), (64 * 7 * 7, 2048)]
WRN_SHAPES = [(128, 32, 32, 64), (128, 16, 16, 128), (128, 8, 8, 256)]


def _windows(fns, calls, rounds, reps=10):
    graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
    us = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            us[k].append(round(1e3 * timed(g.replay, reps, warmup=2) / calls, 2))
    return us


def bn_rows(calls, rounds, B=64):
    from theanompi_b200.ops import cuda_impl
    L, st = cuda_impl.L(), lambda: torch.cuda.current_stream().cuda_stream
    rows = []
    for R, C in BN_SHAPES:
        torch.manual_seed(0)
        t = lambda: torch.randn(R, C, device="cuda:0").to(torch.bfloat16)      # noqa: E731
        x, res, dy = t(), t(), t()
        y, dx, dres = torch.empty_like(x), torch.empty_like(x), torch.empty_like(x)
        f = lambda n: torch.zeros(n, device="cuda:0")                           # noqa: E731
        gam, bet, mean, rstd, scr, dg, db, k = f(C) + 1, f(C), f(C), f(C), f(2 * C), f(C), f(C), f(3 * C)
        row = torch.where(torch.rand(B, device="cuda:0") < 0.1, 0.0, 1.0 / 0.9).float()

        def pair(drop):
            L.bn_forward(x.data_ptr(), res.data_ptr(), y.data_ptr(), gam.data_ptr(), bet.data_ptr(), mean.data_ptr(), rstd.data_ptr(), 0, 0,
                         scr.data_ptr(), R, C, 0.1, 1e-5, 1, 1, 0.0, drop, B, 0, st())
            L.bn_backward(x.data_ptr(), dy.data_ptr(), y.data_ptr(), dx.data_ptr(), dres.data_ptr(), gam.data_ptr(), mean.data_ptr(),
                          rstd.data_ptr(), dg.data_ptr(), db.data_ptr(), k.data_ptr(), R, C, 1, 0.0, 0, drop, B, 0, st())
        us = _windows({"no_row": lambda: pair(0), "row": lambda: pair(row.data_ptr())}, calls, rounds)
        nb = {"no_row": 12 * R * C * 2, "row": 12 * R * C * 2 + 3 * 4 * B}
        rows.append({"R": R, "C": C, "dtype": "bf16", "us_fwd_plus_bwd": us, "min_bytes": nb,
                     "GB_per_s_best": {k2: round(nb[k2] / (min(v) * 1e-6) / 1e9, 1) for k2, v in us.items()}})
    return rows


def add_rows(calls, rounds):
    from theanompi_b200.ops import cuda_impl
    L, st = cuda_impl.L(), lambda: torch.cuda.current_stream().cuda_stream
    rows = []
    for shape in WRN_SHAPES:
        torch.manual_seed(0)
        a, b = (torch.randn(shape, device="cuda:0").to(torch.bfloat16) for _ in range(2))
        y = torch.empty_like(a)
        B, n = shape[0], a.numel()
        s = torch.where(torch.rand(B, device="cuda:0") < 0.1, 0.0, 1.0 / 0.9).float()
        us = _windows({"add": lambda: L.add_tensors(a.data_ptr(), b.data_ptr(), y.data_ptr(), n, 0, st()),
                       "add_scaled": lambda: L.add_scaled(a.data_ptr(), b.data_ptr(), s.data_ptr(), y.data_ptr(), n, B, 0, st()),
                       "row_scale": lambda: L.add_scaled(a.data_ptr(), 0, s.data_ptr(), y.data_ptr(), n, B, 0, st())}, calls, rounds, reps=25)
        nb = {"add": 3 * n * 2, "add_scaled": 3 * n * 2 + 4 * B, "row_scale": 2 * n * 2 + 4 * B}
        rows.append({"shape": list(shape), "dtype": "bf16", "us_per_call": us, "min_bytes": nb,
                     "GB_per_s_best": {k: round(nb[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    return rows


def resnet50(p):
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    m = ResNet50(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=64, file_batch_size=64, cuda_graph=True, no_paraload=True,
                      n_class=1000, drop_path_rate=p, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randn(tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 1000, (m.shared_y.shape[0],), device="cuda:0"))
    return m


def wrn(p):
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    m = Wide_ResNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, cuda_graph=True,
                         drop_path_rate=p, data_kwargs=dict(n_synthetic=256, synthetic=True)))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 10, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


def model_steps(name, build, rates, rounds, steps):
    from theanompi_b200.ops import native
    models, launches = {}, {}
    for p in rates:
        m = models["p=%g" % p] = build(p)
        torch.cuda.synchronize()
        native.reset_launch_count()
        m.train_iter_fn(0)                            # the first step is an eager warm-up: its launches are one step's
        torch.cuda.synchronize()
        launches["p=%g" % p] = native.launch_count()
        for _ in range(4):                            # the second warm-up and the CUDA-graph capture
            m.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in m.captured_steps() for m in models.values()), "a step was not captured"
    res = alternate({k: (lambda m=m: m.train_iter_fn(0)) for k, m in models.items()}, rounds, steps)
    print(json.dumps({name + "_ms_per_step": res, name + "_native_launches_per_step": launches}))
    for m in models.values():
        m.cleanup()
    del models
    torch.cuda.empty_cache()


# one process per window: a ResNet50 batch-64 bf16 CUDA-graph step without the key, from the checkout in the working directory (so it
# also runs against a checkout that predates drop-path)
RESNET_P0 = """
import json, sys, torch
sys.path.insert(0, '.')
from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
m = ResNet50(dict(verbose=False, rank=0, size=1, device='cuda:0', batch_size=64, file_batch_size=64, cuda_graph=True, no_paraload=True,
                  n_class=1000, data_kwargs=dict(n_train_files=2, n_val_files=1, synthetic=True)))
m.compile_iter_fns('avg')
for _ in range(8):
    m.train_iter_fn(0)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
torch.cuda.synchronize(); e0.record()
for _ in range(%d):
    m.train_iter_fn(0)
e1.record(); torch.cuda.synchronize()
print(json.dumps({'ms_per_step': e0.elapsed_time(e1) / %d}))
"""


def resnet50_p0_vs(parent, rounds, steps):
    out = {"this": [], "parent": []}
    for _ in range(rounds):
        for k, d in (("this", ROOT), ("parent", parent)):
            r = subprocess.run([sys.executable, "-c", RESNET_P0 % (steps, steps)], cwd=d, stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                               text=True, timeout=900)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            out[k].append(round(json.loads(line[-1])["ms_per_step"], 3) if r.returncode == 0 and line else r.stdout[-300:])
    print(json.dumps({"resnet50_b64_bf16_no_key_ms_per_step": out}))


def bench_py(parent, rounds):
    cmd = [sys.executable, "bench.py", "--gpus", "1", "--steps", "50", "--warmup", "10"]
    out = {"this": [], "parent": []}
    for _ in range(rounds):
        for k, d in (("this", ROOT), ("parent", parent)):
            r = subprocess.run(cmd, cwd=d, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=1200)
            line = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
            out[k].append(json.loads(line[-1]) if r.returncode == 0 and line else {"error": r.stdout[-500:]})
    print(json.dumps({"bench_py": out}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=100)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_drop_path.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in bn_rows(args.calls, args.rounds):
        print(json.dumps({"batch_norm": row}))
    for row in add_rows(args.calls, args.rounds):
        print(json.dumps({"wrn_merge": row}))
    model_steps("resnet50_b64_bf16", resnet50, (0.0, 0.05, 0.1), args.rounds, args.steps)
    model_steps("wrn28_4_b128_adam", wrn, (0.0, 0.1), args.rounds, args.steps)
    if args.parent:
        resnet50_p0_vs(args.parent, args.rounds, 4 * args.steps)
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
