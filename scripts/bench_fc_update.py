"""FC weight update at AlexNet's fc6 / fc7 / fc8 shapes (batch 128): "wgrad GEMM into G, then sgd_flat over that tensor" against
the wgrad GEMM with the momentum-SGD epilogue (``cuda_impl.gemm_sgd``), bf16 and tf32.

    python scripts/bench_fc_update.py [--iters 200]

CUDA events over ``--iters`` back-to-back launches after a warm-up.  Bytes are what each route must move at least: the GEMM's
operands (dy, x) plus, per weight element, 4 B of G written + 22 B for sgd_flat (W, U, G read; W, U written; bf16 shadow
written) on the two-kernel route, 18 B (W, U read and written, shadow written) on the fused one.  The card's name, power
limit and SM clock are printed by the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

SHAPES = {"fc6": (4096, 9216), "fc7": (4096, 4096), "fc8": (1000, 4096)}


def card():
    try:
        return subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], stdout=subprocess.PIPE, text=True).stdout.strip()
    except OSError:
        return torch.cuda.get_device_name()


def timed(fn, iters):
    for _ in range(5):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1000.0 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--batch", type=int, default=128)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fc_update.py needs a CUDA device")
    from theanompi_b200.ops import cuda_impl
    from theanompi_b200.parallel.arena import FlatArena
    from theanompi_b200.utils.opt import FlatSGD
    print(json.dumps({"card": card()}))
    B = args.batch
    for dtype, adt in (("bf16", torch.bfloat16), ("tf32", torch.float32)):
        for name, (O, I) in SHAPES.items():
            w = torch.nn.Parameter(torch.randn(O, I) * 0.005)
            w.pname = "W"
            a = FlatArena([w], device="cuda:0", weight_decay=5e-4)
            a.hyper[0] = 0.01
            sgd = FlatSGD(a, 0.9, False)
            w.sgd_epilogue, w.arena_group = sgd, a.group_of[0]
            dy = torch.randn(B, O, device="cuda").to(adt)
            x = torch.randn(B, I, device="cuda").to(adt)

            def two_kernels():
                cuda_impl.gemm(dy, x, O, I, B, a_mn=True, b_mn=True, out=w.gbuf, lda=O, ldb=I, ldc=I)
                cuda_impl.sgd_flat(a, a.G, 0.01, 0.9, False, 1.0, 0, a.numel)

            def gemm_only():
                cuda_impl.gemm(dy, x, O, I, B, a_mn=True, b_mn=True, out=w.gbuf, lda=O, ldb=I, ldc=I)

            def sgd_only():
                cuda_impl.sgd_flat(a, a.G, 0.01, 0.9, False, 1.0, 0, a.numel)

            def fused():
                cuda_impl.gemm_sgd(dy, x, w, O, I, B, lda=O, ldb=I)

            n = O * I
            ops = B * (O + I) * dy.element_size()
            t2, tg, ts, tf = (timed(f, args.iters) for f in (two_kernels, gemm_only, sgd_only, fused))
            b2, bs, bf = ops + 26 * n, 22 * a.numel, ops + 18 * n
            print(json.dumps({"dtype": dtype, "shape": name, "O": O, "I": I, "B": B,
                              "gemm_then_sgd_flat_us": round(t2, 2), "gemm_us": round(tg, 2), "sgd_flat_us": round(ts, 2),
                              "sgd_flat_GBps": round(bs / ts / 1e3, 1), "fused_us": round(tf, 2),
                              "fused_bytes": bf, "fused_GBps": round(bf / tf / 1e3, 1), "two_kernel_bytes": b2,
                              "speedup": round(t2 / tf, 3)}))


if __name__ == "__main__":
    main()
