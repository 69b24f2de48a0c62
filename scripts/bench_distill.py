"""What knowledge distillation (``distill``) costs: the fused loss kernel against the plain one, and training steps with the key off and
with a teacher.

    python scripts/bench_distill.py [--calls 200] [--steps 20] [--rounds 3] [--parent DIR]

1. ``softmax_xent_kd`` against ``softmax_xent`` (each with its ``rowstat_mean``) at (B, C) = (32 / 64 / 128 / 256, 1000), bf16 and fp32,
   with and without a mix record: one CUDA graph of ``--calls`` calls per arm, replayed in ``--rounds`` alternating windows and timed with
   CUDA events (µs per call).
2. ``train_iter_fn`` on a device-resident batch with the CUDA graph on, ``--rounds`` alternating windows of ``--steps`` steps: ResNet50-64b
   bf16 with the key off, with a ResNet152 teacher and with a ResNet50 teacher; AlexNet-128b bf16 with the key off and with an AlexNet
   teacher.  The teachers load checkpoints of freshly initialised models written to a temporary directory (the cost does not depend on
   the weights).  Per arm: the peak device memory the arm adds (its build, its teacher and its captured step) and the native launches of
   one eager step.
3. With ``--parent DIR`` (a built checkout): ``bench.py --gpus 1 --steps 50 --warmup 10`` from this checkout and from DIR, alternating.

Needs a CUDA device.  The card's name, power limit and SM clock are printed by the same run, before and after the measurements.
"""
import argparse
import json
import os
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from scripts.bench_drop_path import bench_py  # noqa: E402
from scripts.bench_grad_clip import alexnet  # noqa: E402
from scripts.bench_lamb import card  # noqa: E402
from scripts.bench_model_ema import resnet50  # noqa: E402


def graph_timed(fns, calls, rounds):
    """Per arm one CUDA graph of ``calls`` calls; µs per call over ``rounds`` alternating replays."""
    graphs = {}
    s = torch.cuda.Stream()
    for k, fn in fns.items():
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            for _ in range(3):
                fn()
        torch.cuda.current_stream().wait_stream(s)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            for _ in range(calls):
                fn()
        graphs[k] = g
    for g in graphs.values():
        g.replay()
    torch.cuda.synchronize()
    res = {k: [] for k in fns}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(rounds):
        for k, g in graphs.items():
            e0.record()
            g.replay()
            e1.record()
            torch.cuda.synchronize()
            res[k].append(round(e0.elapsed_time(e1) * 1e3 / calls, 2))
    return res


def kernel_rows(calls, rounds):
    from theanompi_b200.ops import cuda_impl, mixup, reference as ref  # noqa: F401
    import numpy as np
    r = np.zeros((), dtype=mixup.RECORD)
    r["mode"], r["lam"], r["lam_raw"], r["H"], r["W"] = mixup.MIX_MIXUP, 0.7, 0.7, 224, 224
    rec = mixup.encode(r).cuda()
    rows = []
    for dtype in (torch.bfloat16, torch.float32):
        for B in (32, 64, 128, 256):
            g = torch.Generator(device="cuda").manual_seed(B)
            z = (torch.randn(B, 1000, device="cuda", generator=g) * 4).to(dtype)
            t = (torch.randn(B, 1000, device="cuda", generator=g) * 4).to(dtype)
            y = torch.randint(0, 1000, (B,), device="cuda", generator=g)
            for mix in (None, rec):
                fns = {"xent": lambda mix=mix: cuda_impl.softmax_xent(z, y, label_smoothing=0.1, mix=mix),
                       "kd": lambda mix=mix: cuda_impl.softmax_xent_kd(z, y, t, 0.5, 2.0, label_smoothing=0.1, mix=mix)}
                res = graph_timed(fns, calls, rounds)
                rows.append(dict(dtype=str(dtype).split(".")[1], B=B, C=1000, mix=mix is not None, us_per_call=res))
    return rows


def teacher_ckpt(d, name, build):
    """A checkpoint of a freshly built model, written by save_checkpoint into ``d``."""
    from theanompi_b200.utils.helper_funcs import save_checkpoint
    m = build()
    path = save_checkpoint(m, os.path.join(d, "ckpt_%s.pt" % name))
    m.cleanup()
    del m
    torch.cuda.empty_cache()
    return path


def arm(build, dist, steps_warm=5):
    """Build one arm and warm it up (two eager steps, the capture, replays); the peak memory it added and one eager step's launches."""
    from theanompi_b200.ops import native
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    m = build(distill=dist)
    for i in range(steps_warm):
        if i == 1:
            native.reset_launch_count()
        m.train_iter_fn(0)
        if i == 1:
            torch.cuda.synchronize()
            launches = native.launch_count()
    torch.cuda.synchronize()
    assert "step" in m.captured_steps(), "the step was not captured"
    return m, dict(peak_MiB=round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1), launches_per_step=launches)


def model_steps(name, build, arms, args):
    from scripts.bench_grad_clip import alternate
    models, info = {}, {}
    for k, dist in arms.items():
        models[k], info[k] = arm(build, dist)
    res = alternate({k: (lambda mm=mm: mm.train_iter_fn(0)) for k, mm in models.items()}, args.rounds, args.steps)
    print(json.dumps({name + "_ms_per_step": res, name + "_arms": info}), flush=True)
    for mm in models.values():
        mm.cleanup()
    del models
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--parent", default=None, help="a built checkout to run bench.py from, alternating with this one")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_distill.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for row in kernel_rows(args.calls, args.rounds):
        print(json.dumps({"loss_kernel": row}), flush=True)
    from theanompi_b200.models.alex_net import AlexNet
    from theanompi_b200.models.lasagne_model_zoo.resnet152_outdated import ResNet152
    from theanompi_b200.models.lasagne_model_zoo.resnet50 import ResNet50
    data = dict(n_train_files=2, n_val_files=1, synthetic=True)
    with tempfile.TemporaryDirectory() as d:
        r152 = teacher_ckpt(d, "r152", lambda: ResNet152(dict(verbose=False, device="cuda:0", batch_size=64, file_batch_size=64,
                                                              no_paraload=True, data_kwargs=data)))
        r50 = teacher_ckpt(d, "r50", lambda: ResNet50(dict(verbose=False, device="cuda:0", batch_size=64, file_batch_size=64,
                                                           no_paraload=True, data_kwargs=data)))
        alex = teacher_ckpt(d, "alex", lambda: AlexNet(dict(verbose=False, device="cuda:0", batch_size=128, file_batch_size=128,
                                                            no_paraload=True, data_kwargs=data)))
        mod = "theanompi_b200.models."
        model_steps("resnet50_b64_bf16", resnet50, {
            "off": None,
            "teacher_resnet152": dict(teacher=mod + "lasagne_model_zoo.resnet152_outdated:ResNet152", checkpoint=r152),
            "teacher_resnet50": dict(teacher=mod + "lasagne_model_zoo.resnet50:ResNet50", checkpoint=r50)}, args)
        model_steps("alexnet_b128_bf16", alexnet, {"off": None, "teacher_alexnet": dict(teacher=mod + "alex_net:AlexNet", checkpoint=alex)},
                    args)
    if args.parent:
        bench_py(args.parent, args.rounds)
    print(json.dumps({"card_after": card()}))


if __name__ == "__main__":
    main()
