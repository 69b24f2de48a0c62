"""What ten-crop and mirrored validation (``val_crops``) costs: the loader's view kernel against the single crop, the view-accumulate
launches, and whole validation file batches of AlexNet-128b and ResNet50 at 1, 2 and 10 views.

    python scripts/bench_multi_crop.py [--calls 20] [--rounds 3] [--files 4] [--parent DIR]

1. The loader kernels on a [128, 256, 256, 3] uint8 batch → 224² and 227², bf16 and fp32, with the loader's per-pixel mean and
   per-channel scale: ``crop_mirror_norm`` (V = 1, the centre crop) and ``multi_crop_norm`` at V = 2 and V = 10.  ``--calls``
   launches per variant are captured in one CUDA graph and replayed in ``--rounds`` alternating windows of 10 replays, timed with
   CUDA events.  GB/s counts the minimum bytes: the source read once (N·H·W·3) plus the V outputs; the mean image is excluded.
2. ``view_softmax_accum`` at (B, C) = (128, 1000), bf16 and fp32 logits: one view that stores, one that adds, and the last view with
   its ``rowstat_mean``, timed the same way.
3. Validation file batches of 128 images through the thread loader on synthetic data, V = 1, 2 and 10: AlexNet-128b and ResNet50
   with sub-batches of 64, bf16; ms per file batch (the loader hand-off, the V forwards of every sub-batch and the score launches,
   ending in a device synchronise), mean over ``--files`` file batches in each of ``--rounds`` alternating windows.
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

N, H, W = 128, 256, 256
STD = np.array([0.229, 0.224, 0.225], np.float32)


def _windows(graphs, calls, rounds):
    us = {k: [] for k in graphs}
    for _ in range(rounds):
        for k, g in graphs.items():
            us[k].append(round(1e3 * timed(g.replay, 10, warmup=2) / calls, 2))
    return us


def crop_rows(calls, rounds):
    from theanompi_b200.ops import cuda_impl
    torch.manual_seed(0)
    x = torch.randint(0, 256, (N, H, W, 3), dtype=torch.uint8, device="cuda:0")
    mean = torch.rand(H, W, 3, device="cuda:0") * 255
    cs = torch.from_numpy(1.0 / 255.0 / STD).cuda()
    rows = []
    for ch in (224, 227):
        offs = torch.tensor([[(H - ch) // 2, (W - ch) // 2]] * N, dtype=torch.int32, device="cuda:0")
        flips = torch.zeros(N, dtype=torch.uint8, device="cuda:0")
        for dt in (torch.bfloat16, torch.float32):
            one = torch.empty((N, ch, ch, 3), dtype=dt, device="cuda:0")
            outs = {v: torch.empty((v, N, ch, ch, 3), dtype=dt, device="cuda:0") for v in (2, 10)}
            fns = {"V1_crop_mirror_norm": lambda: cuda_impl.crop_mirror_normalize(x, mean, cs, (ch, ch), offs, flips, dt, out=one)}
            for v in (2, 10):
                fns["V%d_multi_crop_norm" % v] = (lambda v=v: cuda_impl.multi_crop_normalize(x, mean, cs, (ch, ch), v, dt, out=outs[v]))
            us = _windows({k: _graph(fn, calls) for k, fn in fns.items()}, calls, rounds)
            V = {"V1_crop_mirror_norm": 1, "V2_multi_crop_norm": 2, "V10_multi_crop_norm": 10}
            nbytes = {k: N * H * W * 3 + V[k] * one.numel() * one.element_size() for k in us}
            rows.append({"in": [N, H, W, 3], "out": [N, ch, ch, 3], "dtype": str(dt).replace("torch.", ""), "mean": "per-pixel, excluded",
                         "us_per_call": us, "min_bytes": nbytes,
                         "GB_per_s_best": {k: round(nbytes[k] / (min(v) * 1e-6) / 1e9, 1) for k, v in us.items()}})
    return rows


def accum_rows(calls, rounds, B=128, C=1000):
    from theanompi_b200.ops import cuda_impl
    rows = []
    for dt in (torch.bfloat16, torch.float32):
        z = torch.randn((B, C), device="cuda:0").to(dt)
        y = torch.randint(0, C, (B,), device="cuda:0")
        acc = torch.empty((B, C), dtype=torch.float32, device="cuda:0")
        rs = torch.empty((B, 3), dtype=torch.float32, device="cuda:0")
        fns = {"first_view_store": lambda: cuda_impl.view_softmax_accum(z, y, acc, 0, 10, rowstat=rs),
               "mid_view_add": lambda: cuda_impl.view_softmax_accum(z, y, acc, 5, 10, rowstat=rs),
               "last_view_add_metrics_and_rowstat_mean": lambda: cuda_impl.view_softmax_accum(z, y, acc, 9, 10, rowstat=rs)}
        us = _windows({k: _graph(fn, calls) for k, fn in fns.items()}, calls, rounds)
        rows.append({"B": B, "C": C, "logits": str(dt).replace("torch.", ""), "us_per_call": us})
    return rows


def _model(cls, V, batch_size, files):
    from theanompi_b200.models import layers2
    layers2.reseed()
    cfg = dict(verbose=False, rank=0, size=1, device="cuda:0", cuda_graph=True, n_class=1000, val_crops=V, batch_size=batch_size,
               file_batch_size=128, data_kwargs=dict(n_train_files=2, n_val_files=files, synthetic=True))
    m = cls(cfg)
    m.compile_iter_fns("avg")
    return m


def val_rows(rounds, files):
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    from theanompi_b200.utils.recorder import Recorder
    for name, cls, bs in (("alexnet_b128_bf16", AlexNet, 128), ("resnet50_b64_bf16", ResNet50, 64)):
        models = {V: _model(cls, V, bs, files) for V in (1, 2, 10)}
        rec = Recorder(None, 10 ** 6, name, False, device="cuda:0")
        ms = {V: [] for V in models}

        def one_pass(m):
            m.reset_iter("val")
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i in range(files * m.n_subb):
                m.val_iter(i, rec)
            torch.cuda.synchronize()
            return (time.perf_counter() - t0) * 1e3 / files
        for m in models.values():
            one_pass(m)                                            # warm-up: module loads, allocator
        for _ in range(rounds):
            for V, m in models.items():
                ms[V].append(round(one_pass(m), 2))
        for m in models.values():
            m.cleanup()
        print(json.dumps({"validation_ms_per_file_batch": {"model": name, "sub_batch": bs, "files": files,
                                                           "ms": {"V%d" % V: v for V, v in ms.items()}}}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--files", type=int, default=4)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multi_crop.py needs a CUDA device")
    print(json.dumps({"card": card()}))
    for row in crop_rows(args.calls, args.rounds):
        print(json.dumps({"loader_kernel": row}))
    for row in accum_rows(args.calls, args.rounds):
        print(json.dumps({"view_softmax_accum": row}))
    val_rows(args.rounds, args.files)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
