"""ms per ``train_iter`` of the native GANs and their torch twins at batch 64, on one GPU.

    python scripts/bench_gan.py [--dtype bf16|tf32] [--iters 50] [--repeats 5]

One ``train_iter`` = ``critic_runs`` critic steps (each with its real batch copied to the device) + one generator step; WGAN runs
with ``critic_runs=2`` (its schedule after the first generator updates), LSGAN with 1.  Host clock around ``--iters`` calls that
end in a device synchronise, after 10 warm-up calls (graph capture included); prints one JSON line per model with the median and
range over ``--repeats`` and the card's name, power limit and SM clock sampled after the timed region.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ZOO = "theanompi_b200.models.lasagne_model_zoo."
MODELS = (("wgan", "wgan", "NativeWGAN", dict(critic_runs=2, data_kwargs=dict(n_synthetic=2048))),
          ("wgan_torch", "wgan", "WGAN", dict(critic_runs=2, data_kwargs=dict(n_synthetic=2048))),
          ("lsgan_cifar", "lsgan_cifar10", "NativeLSGAN", dict(data_kwargs=dict(n_synthetic=2048, synthetic=True))),
          ("lsgan_cifar_torch", "lsgan_cifar10", "LSGAN", dict(data_kwargs=dict(n_synthetic=2048, synthetic=True))))


def _smi(q):
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", default="bf16", choices=["bf16", "tf32"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    from theanompi_b200.utils.recorder import Recorder
    assert torch.cuda.is_available(), "bench_gan.py measures on a GPU"
    for name, mod, cls, cfg in MODELS:
        m = getattr(importlib.import_module(ZOO + mod), cls)(dict(verbose=False, rank=0, size=1, device="cuda:0", dtype=args.dtype, **cfg))
        m.compile_iter_fns("avg")
        rec = Recorder(None, 10 ** 6, name, False, device="cuda:0")
        c = 0
        for _ in range(10):
            c = m.train_iter(c, rec)
        torch.cuda.synchronize()
        res = []
        for _ in range(args.repeats):
            t = time.perf_counter()
            for _ in range(args.iters):
                c = m.train_iter(c, rec)
            torch.cuda.synchronize()
            res.append((time.perf_counter() - t) * 1000.0 / args.iters)
        res.sort()
        print(json.dumps({"model": name, "class": cls, "dtype": args.dtype, "batch": m.batch_size,
                          "critic_runs": cfg.get("critic_runs", 1), "ms_per_train_iter": res[len(res) // 2], "min": res[0],
                          "max": res[-1], "gpu": _smi("name,power.limit"), "sm_clock": _smi("clocks.sm")}), flush=True)


if __name__ == "__main__":
    main()
