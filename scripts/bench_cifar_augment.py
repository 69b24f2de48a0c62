"""What CIFAR augmentation (``cifar_augment``) costs: its kernels on a CIFAR batch, WRN-28-4 training steps with the key against steps
without it, and ``bench.py`` against another checkout.

    python scripts/bench_cifar_augment.py [--calls 200] [--steps 20] [--rounds 3] [--parent DIR]

1. On a [128, 32, 32, 3] batch in bf16 and fp32 (input and output in the same dtype): the plain normalise (``crop_mirror_normalize``
   with zero offsets, the launch a Wide_ResNet step makes without the key), the zero-filled crop with drawn offsets and flips, the draw
   (``cifar_augment_draw``) and the Cutout (``random_erase``, L = 16).  ``--calls`` launches are captured in one CUDA graph per kernel
   and replayed in ``--rounds`` alternating windows, timed with CUDA events: µs per launch.
2. WRN-28-4 batch 128 Adam ``train_iter_fn`` with the CUDA graph, without the key, with ``{}`` and with ``{"cutout": 16}``, in
   ``--rounds`` alternating windows of ``--steps`` steps, and the native launches of one eager step of each.
3. With ``--parent DIR`` (a built checkout): ``bench.py --gpus 1 --steps 50 --warmup 10`` from this checkout and from DIR, alternating,
   ``--rounds`` times each.
4. The card's name, power limit and SM clock, printed by the same run before and after the measurements.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from scripts.bench_drop_path import _windows, bench_py  # noqa: E402
from scripts.bench_grad_clip import alternate  # noqa: E402
from scripts.bench_lamb import card  # noqa: E402


def kernel_rows(calls, rounds, B=128):
    from theanompi_b200.ops import cifar_augment as ca
    from theanompi_b200.ops import cuda_impl
    rows = []
    for dt in (torch.bfloat16, torch.float32):
        torch.manual_seed(0)
        x = torch.randint(0, 256, (B, 32, 32, 3), device="cuda:0").to(dt)
        mean = torch.rand(32, 32, 3, device="cuda:0") * 255
        out = torch.empty_like(x)
        aug = ca.CifarAugment(dict(cutout=16), 0, B, "cuda:0")
        step = torch.full((1,), 7, dtype=torch.int64, device="cuda:0")
        cuda_impl.cifar_augment_draw(aug.cfg, 0, step, aug.offs, aug.flips, aug.boxes)
        zo, zf = torch.zeros_like(aug.offs), torch.zeros_like(aug.flips)
        fns = {
            "normalise": lambda: cuda_impl.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), zo, zf, dt, out=out),
            "zero_fill_crop": lambda: cuda_impl.crop_mirror_normalize(x, mean, 1.0 / 64.0, (32, 32), aug.offs, aug.flips, dt, out=out,
                                                                      zero_fill=True),
            "draw": lambda: cuda_impl.cifar_augment_draw(aug.cfg, 0, step, aug.offs, aug.flips, aug.boxes),
            "erase": lambda: cuda_impl.random_erase(out, aug.boxes),
        }
        us = _windows(fns, calls, rounds, reps=25)
        rows.append({"shape": [B, 32, 32, 3], "dtype": str(dt).replace("torch.", ""), "us_per_launch": us})
    return rows


def wrn(aug):
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    cfg = dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, cuda_graph=True,
               data_kwargs=dict(n_synthetic=256, synthetic=True))
    if aug != "off":
        cfg["cifar_augment"] = json.loads(aug)
    m = Wide_ResNet(cfg)
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 10, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


def wrn_steps(keys, rounds, steps):
    from theanompi_b200.ops import native
    models, launches = {}, {}
    for k in keys:
        m = models[k] = wrn(k)
        torch.cuda.synchronize()
        native.reset_launch_count()
        m.train_iter_fn(0)                            # the first step is an eager warm-up: its launches are one step's
        torch.cuda.synchronize()
        launches[k] = native.launch_count()
        for _ in range(4):                            # the second warm-up and the CUDA-graph capture
            m.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in m.captured_steps() for m in models.values()), "a step was not captured"
    res = alternate({k: (lambda m=m: m.train_iter_fn(0)) for k, m in models.items()}, rounds, steps)
    print(json.dumps({"wrn28_4_b128_adam_ms_per_step": res, "wrn28_4_b128_adam_native_launches_per_step": launches}))
    for m in models.values():
        m.cleanup()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cifar_augment.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"kernels": row}))
    wrn_steps(("off", "{}", '{"cutout": 16}'), args.rounds, args.steps)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
