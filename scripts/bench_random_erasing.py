"""What random erasing (``random_erasing``) costs: the erase kernel on its own and after the fixed crop, the host draw, and
AlexNet-128b / ResNet50-64b training through the loader with the key off and on.

    python scripts/bench_random_erasing.py [--calls 50] [--rounds 3] [--steps 30] [--parent DIR]

1. The erase kernel on a [128, 224, 224, 3] and a [128, 227, 227, 3] output slot, bf16 and fp32, with boxes drawn at the default
   scale and ratio with p = 0.5 and p = 1; and the fixed crop of a [128, 256, 256, 3] uint8 batch (per-pixel mean, per-channel scale)
   without and with the erase launch after it.  ``--calls`` launches per variant are captured in one CUDA graph and replayed in
   ``--rounds`` alternating windows of 10 replays, timed with CUDA events.  GB/s counts the minimum bytes: the erased elements' bytes
   (the kernel only stores), plus the crop's source and output bytes for the crop rows.
2. The host draw of one 128-image batch (``draw_erase_boxes``): mean µs of ``--rounds`` windows of 2,000 draws.
3. AlexNet-128b (fixed crops) and ResNet50-64b (random-resized crop, file batches of 128) bf16 ``train_iter`` through the thread loader
   on synthetic data with the CUDA graph: key off and on (p = 0.5) in ``--rounds`` alternating windows of ``--steps`` steps.
4. With ``--parent DIR`` (a built checkout): ``bench.py --gpus 1 --steps 50 --warmup 10`` alternating with it.
5. The card's name, power limit and SM clock, printed by the same run before and after the measurements.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_drop_path import bench_py  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402
from scripts.bench_mixup import _graph  # noqa: E402
from scripts.bench_resized_crop import model, train_steps  # noqa: E402

N, H, W = 128, 256, 256
STD = np.array([0.229, 0.224, 0.225], np.float32)


def kernel_rows(calls, rounds):
    from theanompi_b200.models.data.utils import check_random_erasing, draw_erase_boxes, random_erasing_rng
    from theanompi_b200.ops import cuda_impl
    torch.manual_seed(0)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device="cuda:0")
    mean = torch.rand(H, W, 3, device="cuda:0") * 255
    cs = torch.from_numpy(1.0 / 255.0 / STD).cuda()
    flips = (torch.arange(N, device="cuda:0") % 2).to(torch.uint8)
    rows = []
    for out_hw in ((224, 224), (227, 227)):
        ch, cw = out_hw
        offs = torch.tensor([[(H - ch) // 2, (W - cw) // 2]] * N, dtype=torch.int32, device="cuda:0")
        boxes = {}
        for p in (0.5, 1.0):
            c = check_random_erasing({"p": p})
            boxes[p] = torch.from_numpy(draw_erase_boxes(N, out_hw, c, random_erasing_rng(c, 0))).cuda()
        for dt in (torch.bfloat16, torch.float32):
            out = torch.empty((N, ch, cw, 3), dtype=dt, device="cuda:0")
            crop = lambda: cuda_impl.crop_mirror_normalize(x, mean, cs, out_hw, offs, flips, dt, out=out)  # noqa: E731

            def erase(b):
                return lambda: cuda_impl.random_erase(out, b)

            def crop_erase(b):
                def fn():
                    crop()
                    cuda_impl.random_erase(out, b)
                return fn
            fns = {"erase_p0.5": erase(boxes[0.5]), "erase_p1": erase(boxes[1.0]), "fixed_crop": crop,
                   "fixed_crop+erase_p0.5": crop_erase(boxes[0.5])}
            graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
            us = {k: [] for k in graphs}
            for _ in range(rounds):
                for k, g in graphs.items():
                    us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
            esz = out.element_size()
            erased = {p: int((b[:, 2].long() * b[:, 3].long()).sum()) * 3 * esz for p, b in boxes.items()}
            crop_bytes = N * ch * cw * 3 + out.numel() * esz
            nbytes = {"erase_p0.5": erased[0.5], "erase_p1": erased[1.0], "fixed_crop": crop_bytes,
                      "fixed_crop+erase_p0.5": crop_bytes + erased[0.5]}
            rows.append({"out": [N, ch, cw, 3], "dtype": str(dt).replace("torch.", ""), "images_erased": {str(p): int((b[:, 2] > 0).sum())
                                                                                                        for p, b in boxes.items()},
                         "us_per_call": us, "min_bytes": nbytes,
                         "GB_per_s_best": {k: round(nbytes[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    return rows


def draw_row(rounds, n=2000):
    from theanompi_b200.models.data.utils import check_random_erasing, draw_erase_boxes, random_erasing_rng
    cfg = check_random_erasing({})
    rng = random_erasing_rng(cfg, 0)
    us = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        for _ in range(n):
            draw_erase_boxes(N, (224, 224), cfg, rng)
        us.append(round((time.perf_counter() - t0) / n * 1e6, 1))
    return {"host_draw_us_per_128_image_batch": us}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_random_erasing.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"erase_kernel": row}))
    print(json.dumps(draw_row(args.rounds)))
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    re = {"p": 0.5}
    train_steps("alexnet_b128_bf16", lambda on: model(AlexNet, None, random_erasing=re if on is not None else None,
                                                       batch_size=128, file_batch_size=128), args.rounds, args.steps)
    train_steps("resnet50_b64_bf16", lambda on: model(ResNet50, {}, random_erasing=re if on is not None else None,
                                                       batch_size=64, file_batch_size=128), args.rounds, args.steps)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
