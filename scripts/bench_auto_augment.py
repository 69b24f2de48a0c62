"""What TrivialAugmentWide / RandAugment (``auto_augment``) cost: each loader kernel, the whole pipeline, the host draw, and
AlexNet-128b / ResNet50-64b training through the loader with the key off and on.

    python scripts/bench_auto_augment.py [--calls 20] [--rounds 3] [--steps 30] [--parent DIR]

1. On a [128, 256, 256, 3] uint8 batch → 224² and 227², bf16 and fp32 (per-pixel mean, per-channel scale): the fixed crop without the
   key (``crop_mirror_norm``), the uint8 crop, the LUT kernel of a slot whose images all draw Equalize, the apply kernel per op class
   (Identity, LUT, Color, Sharpness, the affine gather), the normalisation, and the whole pipeline for "trivial_wide" and for "rand"
   (2, 9).  ``--calls`` launches per variant are captured in one CUDA graph and replayed in ``--rounds`` alternating windows of 10
   replays, timed with CUDA events.  GB/s counts the minimum bytes (``min_bytes`` below): each kernel's uint8 input and output, the
   source box bytes of the crop, the output slot of the normalisation; records, LUTs and the mean image are excluded.
2. The host draw of one 128-image batch (``auto_augment_records``), both policies: mean µs of ``--rounds`` windows of 500 draws.
3. AlexNet-128b (fixed crops) and ResNet50-64b (random-resized crop) bf16 ``train_iter`` through the thread loader with the CUDA graph,
   key off and on ("trivial_wide") in ``--rounds`` alternating windows of ``--steps`` steps.
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
OP_CLASSES = {"identity": 0, "lut_brightness": 6, "color": 7, "sharpness": 9, "affine_rotate": 5}


def _records_of(op, out_hw):
    from theanompi_b200.models.data.utils import auto_augment_records, auto_augment_rng, check_auto_augment
    cfg = check_auto_augment({"seed": op})
    rng = auto_augment_rng(cfg, 0)
    rec = np.zeros((0, 1, 12), np.float32)
    while len(rec) < N:
        r, o, _ = auto_augment_records(4096, cfg, rng, out_hw)
        rec = np.concatenate([rec, r[o[:, 0] == op]])
    return torch.from_numpy(np.ascontiguousarray(rec[:N])).cuda()


def kernel_rows(calls, rounds):
    from theanompi_b200.models.data.utils import auto_augment_records, auto_augment_rng, check_auto_augment
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
        boxes = torch.cat([offs, torch.tensor([[ch, cw]] * N, dtype=torch.int32, device="cuda:0")], 1).contiguous()
        ping = torch.empty((N, ch, cw, 3), dtype=torch.uint8, device="cuda:0")
        pong, lut = torch.empty_like(ping), torch.zeros((N, 3, 256), dtype=torch.uint8, device="cuda:0")
        cuda_impl.aa_crop_u8(x, out_hw, boxes, flips, out=ping)
        recs = {k: _records_of(op, out_hw) for k, op in OP_CLASSES.items()}
        eq = _records_of(13, out_hw)
        pol = {}
        for name, c in (("trivial_wide", {}), ("rand_2_9", {"policy": "rand"})):
            c = check_auto_augment(c)
            r, o, _ = auto_augment_records(N, c, auto_augment_rng(c, 0), out_hw)
            pol[name] = (torch.from_numpy(r).cuda(), o)
        u8 = N * ch * cw * 3
        for dt in (torch.bfloat16, torch.float32):
            out = torch.empty((N, ch, cw, 3), dtype=dt, device="cuda:0")
            fns = {"fixed_crop_off": lambda: cuda_impl.crop_mirror_normalize(x, mean, cs, out_hw, offs, flips, dt, out=out),
                   "crop_u8": lambda: cuda_impl.aa_crop_u8(x, out_hw, boxes, flips, out=pong),
                   "lut_equalize": lambda: cuda_impl.aa_lut(ping, eq, 0, out=lut),
                   "normalize": lambda: cuda_impl.aa_normalize(ping, mean, cs, boxes, flips, (H, W), dt, out=out)}
            nbytes = {"fixed_crop_off": u8 + out.numel() * out.element_size(), "crop_u8": 2 * u8, "lut_equalize": u8,
                      "normalize": u8 + out.numel() * out.element_size()}
            for k, r in recs.items():
                fns["apply_" + k] = (lambda r=r: cuda_impl.aa_apply(ping, r, 0, lut, out=pong))
                nbytes["apply_" + k] = 2 * u8
            for k, (r, o) in pol.items():
                fns["pipeline_" + k] = (lambda r=r, o=o: cuda_impl.auto_augment_crop_normalize(
                    x, mean, cs, out_hw, boxes, flips, r, o, dt, out=out, ping=ping, pong=pong, lut=lut))
                nbytes["pipeline_" + k] = 2 * u8 + out.numel() * out.element_size()
            graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
            us = {k: [] for k in graphs}
            for _ in range(rounds):
                for k, g in graphs.items():
                    us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
            rows.append({"in": [N, H, W, 3], "out": [N, ch, cw, 3], "dtype": str(dt).replace("torch.", ""), "us_per_call": us,
                         "min_bytes": nbytes, "GB_per_s_best": {k: round(nbytes[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    return rows


def draw_row(rounds, n=500):
    from theanompi_b200.models.data.utils import auto_augment_records, auto_augment_rng, check_auto_augment
    out = {}
    for name, c in (("trivial_wide", {}), ("rand_2_9", {"policy": "rand"})):
        cfg = check_auto_augment(c)
        rng = auto_augment_rng(cfg, 0)
        us = []
        for _ in range(rounds):
            t0 = time.perf_counter()
            for _ in range(n):
                auto_augment_records(N, cfg, rng, (224, 224))
            us.append(round((time.perf_counter() - t0) / n * 1e6, 1))
        out[name] = us
    return {"host_draw_us_per_128_image_batch": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_auto_augment.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"loader_kernels": row}), flush=True)
    print(json.dumps(draw_row(args.rounds)), flush=True)
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    train_steps("alexnet_b128_bf16", lambda on: model(AlexNet, None, auto_augment={} if on is not None else None,
                                                       batch_size=128, file_batch_size=128), args.rounds, args.steps)
    train_steps("resnet50_b64_bf16", lambda on: model(ResNet50, {}, auto_augment={} if on is not None else None,
                                                       batch_size=64, file_batch_size=128), args.rounds, args.steps)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
