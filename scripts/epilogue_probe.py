"""Epilogue probe: the same GEMMs with the classic epilogue (coalesced 16-byte st.global / red.global.add.v4) and through the
bulk copy engine (cp.async.bulk / cp.reduce.async.bulk, one row segment per lane), bf16 and tf32 operands.  Prints µs (CUDA
events, L2 flushed between repeats), effective output bandwidth and the max |difference| between the two epilogues.

    python scripts/epilogue_probe.py
"""
import sys
import torch

sys.path.insert(0, ".")
from theanompi_b200.ops import native  # noqa: E402

L = native.require()
dev = torch.device("cuda:0")
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=8):
    st = torch.cuda.current_stream()
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record(st); fn(); e1.record(st); e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def S():
    return torch.cuda.current_stream().cuda_stream


def case(name, M, N, K, a_mn, b_mn, out_bf16, tf32, splitk):
    dt = torch.float32 if tf32 else torch.bfloat16
    A = torch.randn((K, M) if a_mn else (M, K), device=dev).to(dt)
    B = torch.randn((K, N) if b_mn else (N, K), device=dev).to(dt)
    outs = []
    times = []
    for mask in (0, 7):
        L.gemm_set_bulk(mask)
        C = torch.zeros(M, N, device=dev, dtype=torch.bfloat16 if out_bf16 else torch.float32)

        def f():
            L.gemm(A.data_ptr(), B.data_ptr(), C.data_ptr(), 0, M, N, K, A.shape[1], B.shape[1], N, int(a_mn), int(b_mn), int(out_bf16),
                   0, 0, 1.0, 0, splitk, int(tf32), S())
        times.append(timeit(f))
        f(); torch.cuda.synchronize()
        outs.append(C.float().clone())
    L.gemm_set_bulk(-1)
    diff = float((outs[0] - outs[1]).abs().max())
    ob = M * N * (2 if out_bf16 else 4)
    print("%-44s classic %8.1f us  bulk %8.1f us  (%5.2fx)  out %6.1f MB  %6.0f -> %6.0f GB/s   max|diff| %.3g"
          % (name, times[0], times[1], times[0] / times[1], ob / 1e6, ob / times[0] / 1e3, ob / times[1] / 1e3, diff), flush=True)


def main():
    case("fc6 wgrad 4096x9216x128 fp32 out (mn,mn)", 4096, 9216, 128, 1, 1, 0, 0, 1)
    case("fc7 wgrad 4096x4096x128 fp32 out (mn,mn)", 4096, 4096, 128, 1, 1, 0, 0, 1)
    case("fc6 wgrad, tf32 operands", 4096, 9216, 128, 1, 1, 0, 1, 1)
    case("conv-wgrad-like 256x2304x21632 split-K", 256, 2304, 21632, 1, 1, 0, 0, 0)
    case("conv-wgrad-like 256x2304x21632 split-K tf32", 256, 2304, 21632, 1, 1, 0, 1, 0)
    case("square 4096^3 bf16 out", 4096, 4096, 4096, 0, 0, 1, 0, 1)
    case("square 4096^3 tf32", 4096, 4096, 4096, 0, 0, 0, 1, 1)
    case("tall 21632x384x2304 bf16 out", 21632, 384, 2304, 0, 0, 1, 0, 1)


if __name__ == "__main__":
    main()
