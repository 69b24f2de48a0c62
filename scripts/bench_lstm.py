"""ms per ``train_iter`` of the native LSTM (bucketed CUDA graphs and eager) and of ``LSTMTorch`` (cuDNN), on one GPU.

    python scripts/bench_lstm.py [--dtype bf16 tf32] [--iters 50] [--repeats 5]

Batch 16, H 128, vocabulary 10000, synthetic sequence lengths 20-80 and 100-500.  Every arm trains on the same ``--iters`` batches
per repeat.  Warm-up first runs the first batch of every length bucket those batches use three times (two eager warm-ups, then the
capture of that bucket's graph) and then one pass over all of them, so the timed window replays captured graphs only (and the
eager arms see every shape once).  Time: host clock around ``--iters`` calls that end in a device synchronise; the median and range
over ``--repeats``.  One JSON line per (dtype, length range, arm), with the card's name and power limit, the SM clock sampled after
the timed region and the arm's peak ``torch.cuda.max_memory_allocated()`` above what was allocated before its model was built
(for the graph arm: with every bucket captured).
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

ARMS = (("graphs", "LSTM", dict(cuda_graph=True)), ("eager", "LSTM", dict(cuda_graph=False)), ("cudnn", "LSTMTorch", {}))
LENGTHS = ((20, 80), (100, 500))


def _smi(q):
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dtype", nargs="+", default=["bf16", "tf32"], choices=["bf16", "tf32"])
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    import torch
    from theanompi_b200.models import lstm
    from theanompi_b200.utils.recorder import Recorder
    assert torch.cuda.is_available(), "bench_lstm.py measures on a GPU"
    for dtype in args.dtype:
        for lo, hi in LENGTHS:
            for arm, cls, extra in ARMS:
                gc.collect()
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                base = torch.cuda.memory_allocated()
                cfg = dict(verbose=False, rank=0, size=1, device="cuda:0", dtype=dtype, dim_proj=128,
                           data_kwargs=dict(n_synthetic=2048, n_words=10000, seq_len=(lo, hi)), **extra)
                m = getattr(lstm, cls)(cfg)
                m.compile_iter_fns("avg")
                rec = Recorder(None, 10 ** 6, cls, False, device="cuda:0")
                it = m.data.batches("train", m.batch_size, True, seed=0)
                batches = [next(it) for _ in range(args.iters)]
                first = {}
                for b in batches:
                    first.setdefault(lstm.bucket_len(b[0].shape[1], m.data.maxlen), b)
                warm = [b for b in first.values() for _ in range(3)] + batches
                m._train_it = iter(warm)
                for i in range(len(warm)):
                    m.train_iter(i, rec)
                torch.cuda.synchronize()
                res = []
                for _ in range(args.repeats):
                    m._train_it = iter(batches)
                    t = time.perf_counter()
                    for i in range(args.iters):
                        m.train_iter(i, rec)
                    torch.cuda.synchronize()
                    res.append((time.perf_counter() - t) * 1000.0 / args.iters)
                res.sort()
                captured = sorted(m.captured_steps())
                print(json.dumps({"arm": arm, "class": cls, "dtype": dtype, "seq_len": [lo, hi], "batch": m.batch_size, "H": 128,
                                  "mean_T": sum(b[0].shape[1] for b in batches) / len(batches), "buckets": sorted(first),
                                  "graphs_captured": captured, "ms_per_train_iter": res[len(res) // 2], "min": res[0],
                                  "max": res[-1], "peak_memory_MiB": (torch.cuda.max_memory_allocated() - base) / 2 ** 20,
                                  "gpu": _smi("name,power.limit"), "sm_clock": _smi("clocks.sm")}), flush=True)
                del m
                torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
