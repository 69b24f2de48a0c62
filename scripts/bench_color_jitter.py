"""What colour jitter and PCA lighting (``color_jitter``) cost: the loader kernels against the ones without the key, the host draw, and
AlexNet-128b / ResNet50-64b training through the loader with the key off and on.

    python scripts/bench_color_jitter.py [--calls 50] [--rounds 3] [--steps 30] [--parent DIR]

1. The loader kernels on a [128, 256, 256, 3] uint8 batch → [128, 224, 224, 3] and [128, 227, 227, 3], bf16 and fp32 outputs, with
   the loader's per-pixel mean and per-channel scale: the fixed crop off (``crop_mirror_norm``), with lighting only (the jitter path,
   no crop mean) and with all four strengths (``crop_mean`` + the jitter path); the resized crop (default-scale draw) off
   (``resized_crop_mirror_norm``) and with all four.  ``--calls`` launches per variant are captured in one CUDA graph and replayed in
   ``--rounds`` alternating windows of 10 replays, timed with CUDA events.  GB/s counts the minimum bytes: the source bytes of the
   boxes (read once more by the crop mean when it runs) plus the output bytes; the mean image and the 96-byte records are excluded.
2. The host draw of one 128-image batch (``color_jitter_records``, all four strengths): mean µs of ``--rounds`` windows of 2,000
   draws.
3. AlexNet-128b (fixed crops) and ResNet50-64b (random-resized crop, file batches of 128) bf16 ``train_iter`` through the thread loader
   on synthetic data with the CUDA graph: key off and on (all four strengths) in ``--rounds`` alternating windows of ``--steps``
   steps.  The loader kernels run on the copy stream next to the step, so this is the number that matters.
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
ALL4 = {"brightness": 0.4, "contrast": 0.4, "saturation": 0.4, "lighting": 0.1}


def kernel_rows(calls, rounds):
    from theanompi_b200.models.data.utils import (check_color_jitter, check_resized_crop, color_jitter_records, color_jitter_rng,
                                                  draw_resized_crops, resized_crop_rng)
    from theanompi_b200.ops import cuda_impl
    torch.manual_seed(0)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device="cuda:0")
    mean = torch.rand(H, W, 3, device="cuda:0") * 255
    cs = torch.from_numpy(1.0 / 255.0 / STD).cuda()
    flips = (torch.arange(N, device="cuda:0") % 2).to(torch.uint8)
    rcfg = check_resized_crop({})
    drawn = torch.from_numpy(draw_resized_crops(N, (H, W), rcfg["scale"], rcfg["ratio"], resized_crop_rng(rcfg, 0))[0]).cuda()
    recs = {}
    for name, c in (("lighting", {"lighting": 0.1}), ("all4", ALL4)):
        c = check_color_jitter(c)
        recs[name] = torch.from_numpy(color_jitter_records(N, c, color_jitter_rng(c, 0))[0]).cuda()
    mu = torch.empty((N, 4), dtype=torch.float32, device="cuda:0")
    rows = []
    for out_hw in ((224, 224), (227, 227)):
        ch, cw = out_hw
        offs = torch.tensor([[(H - ch) // 2, (W - cw) // 2]] * N, dtype=torch.int32, device="cuda:0")
        fixed = torch.cat([offs, torch.tensor([[ch, cw]] * N, dtype=torch.int32, device="cuda:0")], 1).contiguous()
        for dt in (torch.bfloat16, torch.float32):
            out = torch.empty((N, ch, cw, 3), dtype=dt, device="cuda:0")

            def jitter(boxes, rec, with_mean):
                def fn():
                    m = cuda_impl.crop_mean(x, boxes, out_hw, out=mu) if with_mean else None
                    cuda_impl.color_crop_mirror_normalize(x, mean, cs, out_hw, boxes, flips, rec, m, dt, out=out)
                return fn
            fns = {"fixed_off": lambda: cuda_impl.crop_mirror_normalize(x, mean, cs, out_hw, offs, flips, dt, out=out),
                   "fixed_lighting": jitter(fixed, recs["lighting"], False),
                   "fixed_all4": jitter(fixed, recs["all4"], True),
                   "resized_off": lambda: cuda_impl.resized_crop_mirror_normalize(x, mean, cs, out_hw, drawn, flips, dt, out=out),
                   "resized_all4": jitter(drawn, recs["all4"], True)}
            graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
            us = {k: [] for k in graphs}
            for _ in range(rounds):
                for k, g in graphs.items():
                    us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
            out_bytes = out.numel() * out.element_size()
            src_fixed = N * ch * cw * 3
            src_drawn = int((drawn[:, 2].long() * drawn[:, 3].long()).sum()) * 3
            nbytes = {"fixed_off": src_fixed + out_bytes, "fixed_lighting": src_fixed + out_bytes, "fixed_all4": 2 * src_fixed + out_bytes,
                      "resized_off": src_drawn + out_bytes, "resized_all4": 2 * src_drawn + out_bytes}
            rows.append({"in": [N, H, W, 3], "out": [N, ch, cw, 3], "dtype": str(dt).replace("torch.", ""), "mean": "per-pixel, excluded",
                         "us_per_call": us, "min_bytes": nbytes,
                         "GB_per_s_best": {k: round(nbytes[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    return rows


def draw_row(rounds, n=2000):
    from theanompi_b200.models.data.utils import check_color_jitter, color_jitter_records, color_jitter_rng
    cfg = check_color_jitter(ALL4)
    rng = color_jitter_rng(cfg, 0)
    us = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        for _ in range(n):
            color_jitter_records(N, cfg, rng)
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
        raise SystemExit("bench_color_jitter.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"loader_kernel": row}))
    print(json.dumps(draw_row(args.rounds)))
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    train_steps("alexnet_b128_bf16", lambda on: model(AlexNet, None, color_jitter=ALL4 if on is not None else None,
                                                       batch_size=128, file_batch_size=128), args.rounds, args.steps)
    train_steps("resnet50_b64_bf16", lambda on: model(ResNet50, {}, color_jitter=ALL4 if on is not None else None,
                                                       batch_size=64, file_batch_size=128), args.rounds, args.steps)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
