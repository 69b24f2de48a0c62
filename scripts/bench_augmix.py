"""What AutoAugment and AugMix (``auto_augment`` policies "autoaugment" and "augmix") cost: the whole loader pipeline per policy, bilinear
against nearest geometry, the mix kernel, the host draw, and AlexNet-128b / ResNet50-64b training through the loader with the key off
and on ("augmix").

    python scripts/bench_augmix.py [--calls 20] [--rounds 3] [--steps 30] [--parent DIR]

1. On a [128, 256, 256, 3] uint8 batch → 224² and 227², bf16 and fp32 (per-pixel mean, per-channel scale), fixed crops: the crop
   without the key (``crop_mirror_norm``), and the whole pipeline (crop, LUT and apply launches, mix, normalisation) for
   "trivial_wide", "trivial_wide" with bilinear geometry, "autoaugment", "augmix" at its defaults (width 3, depth uniform in 1…3,
   bilinear) and "augmix" with chain_depth 1; plus the apply kernel on a batch of Rotate records, nearest and bilinear, and the mix
   kernel alone.  Every variant replays one drawn batch: ``--calls`` calls are captured in one CUDA graph and replayed in ``--rounds``
   alternating windows of 10 replays, timed with CUDA events.  The launches per call are counted and reported with each time.
2. The host draw of one 128-image batch (``auto_augment_records`` / ``augmix_records``) per policy: mean µs of ``--rounds`` windows of
   500 draws.
3. AlexNet-128b (fixed crops) and ResNet50-64b (random-resized crop) bf16 ``train_iter`` through the thread loader with the CUDA graph,
   key off and "augmix" on, in ``--rounds`` alternating windows of ``--steps`` steps.
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
POLICIES = {"trivial_wide": {}, "trivial_wide_bilinear": {"interpolation": "bilinear"}, "autoaugment": {"policy": "autoaugment"},
            "augmix": {"policy": "augmix"}, "augmix_depth1": {"policy": "augmix", "chain_depth": 1}}


def _draw(c, out_hw):
    from theanompi_b200.models.data.utils import augmix_records, auto_augment_records, auto_augment_rng, check_auto_augment
    cfg = check_auto_augment(c)
    if cfg["policy"] == "augmix":
        r, w, o, _ = augmix_records(N, cfg, auto_augment_rng(cfg, 0), out_hw)
        return cfg, torch.from_numpy(r).cuda(), o, torch.from_numpy(w).cuda()
    r, o, _ = auto_augment_records(N, cfg, auto_augment_rng(cfg, 0), out_hw)
    return cfg, torch.from_numpy(r).cuda(), o, None


def kernel_rows(calls, rounds):
    from theanompi_b200.models.data.utils import aa_bilinear, aa_compose_records
    from theanompi_b200.ops import cuda_impl, native
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
        chains = torch.empty((3, 2) + tuple(ping.shape), dtype=torch.uint8, device="cuda:0")
        cuda_impl.aa_crop_u8(x, out_hw, boxes, flips, out=ping)
        draws = {k: _draw(c, out_hw) for k, c in POLICIES.items()}
        rot = torch.from_numpy(aa_compose_records(np.full((N, 1), 5), np.linspace(-30, 30, N)[:, None], out_hw)).cuda()
        rot_bil = rot.clone()
        rot_bil[..., 3] = 1
        mix = draws["augmix"]
        for dt in (torch.bfloat16, torch.float32):
            out = torch.empty((N, ch, cw, 3), dtype=dt, device="cuda:0")
            fns = {"fixed_crop_off": lambda: cuda_impl.crop_mirror_normalize(x, mean, cs, out_hw, offs, flips, dt, out=out),
                   "apply_rotate_nearest": lambda: cuda_impl.aa_apply(ping, rot, 0, lut, out=pong, bilinear=False),
                   "apply_rotate_bilinear": lambda: cuda_impl.aa_apply(ping, rot_bil, 0, lut, out=pong, bilinear=True),
                   "mix_width3": lambda: cuda_impl.aa_mix(pong, chains, mix[1], mix[3])}
            for k, (cfg, r, o, w) in draws.items():
                fns["pipeline_" + k] = (lambda cfg=cfg, r=r, o=o, w=w: cuda_impl.auto_augment_crop_normalize(
                    x, mean, cs, out_hw, boxes, flips, r, o, dt, out=out, ping=ping, pong=pong, lut=lut, bilinear=aa_bilinear(cfg),
                    weights=w, chains=chains[:r.shape[1] // 3] if w is not None else None))
            launches = {}
            for k, fn in fns.items():
                torch.cuda.synchronize()
                native.reset_launch_count()
                fn()
                torch.cuda.synchronize()
                launches[k] = native.launch_count()
            graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
            us = {k: [] for k in graphs}
            for _ in range(rounds):
                for k, g in graphs.items():
                    us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
            rows.append({"in": [N, H, W, 3], "out": [N, ch, cw, 3], "dtype": str(dt).replace("torch.", ""), "us_per_call": us,
                         "launches_per_call": launches})
    return rows


def draw_row(rounds, n=500):
    from theanompi_b200.models.data.utils import augmix_records, auto_augment_records, auto_augment_rng, check_auto_augment
    out = {}
    for name in ("trivial_wide", "autoaugment", "augmix", "augmix_depth1"):
        cfg = check_auto_augment(POLICIES[name])
        rng = auto_augment_rng(cfg, 0)
        fn = augmix_records if cfg["policy"] == "augmix" else auto_augment_records
        us = []
        for _ in range(rounds):
            t0 = time.perf_counter()
            for _ in range(n):
                fn(N, cfg, rng, (224, 224))
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
        raise SystemExit("bench_augmix.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"loader_kernels": row}), flush=True)
    print(json.dumps(draw_row(args.rounds)), flush=True)
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    augmix = {"policy": "augmix"}
    train_steps("alexnet_b128_bf16", lambda on: model(AlexNet, None, auto_augment=augmix if on is not None else None,
                                                       batch_size=128, file_batch_size=128), args.rounds, args.steps)
    train_steps("resnet50_b64_bf16", lambda on: model(ResNet50, {}, auto_augment=augmix if on is not None else None,
                                                       batch_size=64, file_batch_size=128), args.rounds, args.steps)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
