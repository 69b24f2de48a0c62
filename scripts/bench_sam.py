"""What sharpness-aware minimization (``sam``) costs: the three SAM kernels alone on AlexNet's and ResNet50's arenas, and training steps
with the key off, SAM and ASAM.

    python scripts/bench_sam.py [--iters 200] [--steps 20] [--rounds 3] [--parent DIR]

1. ``sam_norm`` (two launches), ``sam_perturb`` and ``sam_restore`` over each arena, SAM and ASAM (CUDA events over ``--iters`` calls,
   after 10 warm-up calls).  GB/s count the minimum bytes per arena element: the norm reads G (4 B; ASAM also W: 8 B), the perturbation
   reads W and G and writes P, W and the bf16 shadow (18 B), the restore reads P and writes W and the shadow (10 B).
2. ``train_iter_fn`` on a device-resident batch with the CUDA graph on: AlexNet-128b bf16 with SGD, ResNet50-64b with SGD and
   WRN-28-4-128b with Adam, each with the key off, ``{"rho": 0.05}`` and ``{"rho": 1.0, "adaptive": true}`` in one process, ``--rounds``
   alternating windows of ``--steps`` steps (``scripts/bench_grad_clip.py: alternate``).
3. With ``--parent DIR`` (a built checkout): ``bench.py --gpus 1 --steps 50 --warmup 10`` from this checkout and from DIR, alternating.

Needs a CUDA device.  The card's name, power limit and SM clock are printed by the same run, before and after the measurements.
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_drop_path import bench_py  # noqa: E402
from scripts.bench_grad_clip import alexnet, alternate  # noqa: E402
from scripts.bench_lamb import card, timed  # noqa: E402
from scripts.bench_model_ema import resnet50  # noqa: E402

VARIANTS = {"off": None, "sam": dict(rho=0.05), "asam": dict(rho=1.0, adaptive=True)}


def kernels(build, iters):
    """The SAM launches alone over the model's arena: ms per call and GB/s on the minimum bytes."""
    from theanompi_b200.ops import cuda_impl
    m = build(sam=dict(rho=0.05))
    a, s = m.arena, m.sam_opt
    torch.manual_seed(0)
    a.G.copy_(torch.randn_like(a.G) * 1e-3)
    out = {"arena_elements": a.numel}
    for adaptive in (False, True):
        tag = "asam" if adaptive else "sam"
        ms = timed(lambda: cuda_impl.sam_norm(a, s.rho, adaptive, s._partial, s.rec), iters)
        out[tag + "_norm_us"] = round(ms * 1e3, 1)
        out[tag + "_norm_GBps"] = round((8 if adaptive else 4) * a.numel / (ms * 1e-3) / 1e9, 1)
        # every call moves W by e once more: the timing does not depend on the values
        ms = timed(lambda: cuda_impl.sam_perturb(a, s.P, s.rec, adaptive), iters)
        out[tag + "_perturb_us"] = round(ms * 1e3, 1)
        out[tag + "_perturb_GBps"] = round((18 if a.H is not None else 16) * a.numel / (ms * 1e-3) / 1e9, 1)
        cuda_impl.sam_restore(a, s.P)
    ms = timed(lambda: cuda_impl.sam_restore(a, s.P), iters)
    out["restore_us"] = round(ms * 1e3, 1)
    out["restore_GBps"] = round((10 if a.H is not None else 8) * a.numel / (ms * 1e-3) / 1e9, 1)
    m.cleanup()
    del m
    torch.cuda.empty_cache()
    return out


def steps(build, args):
    models = {k: build(sam=v) for k, v in VARIANTS.items()}
    for mm in models.values():
        for _ in range(5):                            # eager warm-up and the CUDA-graph capture
            mm.train_iter_fn(0)
    torch.cuda.synchronize()
    assert all("step" in mm.captured_steps() for mm in models.values()), "a step was not captured"
    res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
    for mm in models.values():
        mm.cleanup()
    del models
    torch.cuda.empty_cache()
    return res


def wrn_adam(**kw):
    from theanompi_b200.models.keras_model_zoo.wresnet import Wide_ResNet
    m = Wide_ResNet(dict(verbose=False, rank=0, size=1, device="cuda:0", batch_size=128, file_batch_size=128, cuda_graph=True,
                         data_kwargs=dict(n_synthetic=256, synthetic=True), **kw))
    m.compile_iter_fns("avg")
    torch.manual_seed(0)
    m.shared_x.copy_(torch.randint(0, 256, tuple(m.shared_x.shape), device="cuda:0").to(m.shared_x.dtype))
    m.shared_y.copy_(torch.randint(0, 10, (m.shared_y.shape[0],), device="cuda:0").to(m.shared_y.dtype))
    return m


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sam.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for name, build in (("alexnet_b128", alexnet), ("resnet50_b64", resnet50)):
        print(json.dumps({name + "_sam_kernels": kernels(build, args.iters)}), flush=True)
    for name, build in (("alexnet_b128", alexnet), ("resnet50_b64", resnet50), ("wrn28_4_b128_adam", wrn_adam)):
        print(json.dumps({name + "_ms_per_step": steps(build, args)}), flush=True)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
