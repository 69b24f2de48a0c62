"""What random-resized crop (``random_resized_crop``) costs: the loader kernel against the fixed-crop one, the host draw, and
AlexNet-128b / ResNet50-64b training through the loader with the key off and on.

    python scripts/bench_resized_crop.py [--calls 50] [--rounds 3] [--steps 30] [--parent DIR]

1. ``resized_crop_mirror_norm`` against ``crop_mirror_norm`` on a [128, 256, 256, 3] uint8 batch → [128, 227, 227, 3] and
   [128, 224, 224, 3], bf16 and fp32 outputs, with the loader's per-pixel mean and per-channel scale.  Two box sets: the
   default-scale draw (scale [0.08, 1], ratio [3/4, 4/3], seed 0) and full-image boxes (every output pixel downscaled from 256²).
   ``--calls`` launches are captured in one CUDA graph per kernel and replayed in ``--rounds`` alternating windows of 10 replays
   (≥ 200 launches per window at the default), timed with CUDA events.  GB/s counts the minimum bytes: the source bytes of the
   boxes (of the fixed crop's window) plus the output bytes, mean excluded (786 KB, read by every image from L2).
2. The host draw of one 128-image batch (``draw_resized_crops``, all attempts vectorised), a host cost: mean / min / max µs of
   ``--rounds`` windows of 2,000 draws.
3. AlexNet-128b and ResNet50-64b (file batches of 128) bf16 ``train_iter`` through the thread loader on synthetic data, with the
   CUDA graph: key off and on in ``--rounds`` alternating windows of ``--steps`` steps (CUDA events around the window, which ends in
   a synchronise).  The loader kernel runs on the copy stream next to the step, so this is the number that matters.
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
from scripts.bench_grad_clip import alternate  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402
from scripts.bench_mixup import _graph  # noqa: E402

N, H, W = 128, 256, 256
STD = np.array([0.229, 0.224, 0.225], np.float32)


def kernel_rows(calls, rounds):
    from theanompi_b200.models.data.utils import check_resized_crop, draw_resized_crops, resized_crop_rng
    from theanompi_b200.ops import cuda_impl
    torch.manual_seed(0)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device="cuda:0")
    mean = torch.rand(H, W, 3, device="cuda:0") * 255
    cs = torch.from_numpy(1.0 / 255.0 / STD).cuda()
    flips = (torch.arange(N, device="cuda:0") % 2).to(torch.uint8)
    cfg = check_resized_crop({})
    drawn, _ = draw_resized_crops(N, (H, W), cfg["scale"], cfg["ratio"], resized_crop_rng(cfg, 0))
    box_sets = {"default_draw": torch.from_numpy(drawn).cuda(),
                "full_image": torch.tensor([[0, 0, H, W]] * N, dtype=torch.int32, device="cuda:0")}
    rows = []
    for out_hw in ((227, 227), (224, 224)):
        ch, cw = out_hw
        offs = torch.tensor([[(H - ch) // 2, (W - cw) // 2]] * N, dtype=torch.int32, device="cuda:0")
        for dt in (torch.bfloat16, torch.float32):
            out = torch.empty((N, ch, cw, 3), dtype=dt, device="cuda:0")
            fns = {"crop_mirror_norm": lambda: cuda_impl.crop_mirror_normalize(x, mean, cs, out_hw, offs, flips, dt, out=out)}
            for name, b in box_sets.items():
                fns["resized_" + name] = (lambda b=b: cuda_impl.resized_crop_mirror_normalize(x, mean, cs, out_hw, b, flips, dt, out=out))
            graphs = {k: _graph(fn, calls) for k, fn in fns.items()}
            us = {k: [] for k in graphs}
            for _ in range(rounds):
                for k, g in graphs.items():
                    us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
            out_bytes = out.numel() * out.element_size()
            nbytes = {"crop_mirror_norm": N * ch * cw * 3 + out_bytes}
            for name, b in box_sets.items():
                nbytes["resized_" + name] = int((b[:, 2].long() * b[:, 3].long()).sum()) * 3 + out_bytes
            rows.append({"in": [N, H, W, 3], "out": [N, ch, cw, 3], "dtype": str(dt).replace("torch.", ""), "mean": "per-pixel, excluded",
                         "us_per_call": us, "min_bytes": nbytes,
                         "GB_per_s_best": {k: round(nbytes[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    return rows


def draw_row(rounds, n=2000):
    from theanompi_b200.models.data.utils import check_resized_crop, draw_resized_crops, resized_crop_rng
    cfg = check_resized_crop({})
    rng = resized_crop_rng(cfg, 0)
    us = []
    for _ in range(rounds):
        t0 = time.perf_counter()
        for _ in range(n):
            draw_resized_crops(N, (H, W), cfg["scale"], cfg["ratio"], rng)
        us.append(round((time.perf_counter() - t0) / n * 1e6, 1))
    return {"host_draw_us_per_128_image_batch": us}


def model(cls, rrc, **kw):
    from theanompi_b200.models import layers2
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cuda:0", cuda_graph=True, n_class=1000,
               data_kwargs=dict(n_train_files=64, n_val_files=1, synthetic=True), random_resized_crop=rrc, **kw)
    m = cls(cfg)
    m.compile_iter_fns("avg")
    return m


def train_steps(name, build, rounds, steps):
    from theanompi_b200.utils.recorder import Recorder
    models = {"off": build(None), "on": build({})}
    recs = {k: Recorder(None, 10 ** 6, k, False, device="cuda:0") for k in models}
    count = {k: 0 for k in models}

    def window(k):
        m = models[k]
        m.reset_iter("train")                         # drain the look-ahead, start at file 0: a window never crosses an epoch

        def step():
            m.train_iter(count[k], recs[k])
            count[k] += 1
        return step

    for k, m in models.items():
        fn = window(k)
        for _ in range(6):                            # eager warm-up and the CUDA-graph capture
            fn()
        torch.cuda.synchronize()
        assert "step" in m.captured_steps(), "the step was not captured"
    res = {k: [] for k in models}
    for _ in range(rounds):
        for k in models:
            res[k].append(round(timed(window(k), steps, warmup=3), 3))
    print(json.dumps({name + "_train_iter_ms_per_step": res}))
    for m in models.values():
        m.cleanup()
    del models
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resized_crop.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"loader_kernel": row}))
    print(json.dumps(draw_row(args.rounds)))
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    train_steps("alexnet_b128_bf16", lambda rrc: model(AlexNet, rrc, batch_size=128, file_batch_size=128), args.rounds, args.steps)
    train_steps("resnet50_b64_bf16", lambda rrc: model(ResNet50, rrc, batch_size=64, file_batch_size=128), args.rounds, args.steps)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
