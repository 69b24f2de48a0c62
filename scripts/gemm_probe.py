"""Bottleneck probe for the wgmma GEMM / implicit-conv kernel on the AlexNet-128b shapes.

For each shape: time the kernel (CUDA events, L2 flushed by a 256 MiB write between repeats) normally and with the
probe knobs of ``gemm_set_debug`` (1 = no A loads, 2 = no B loads, 4 = no MMAs) and print achieved TFLOP/s and the
L2→SM operand traffic rate, so "L2-bandwidth bound" vs "issue bound" vs "latency bound" can be read off one table.

    python scripts/gemm_probe.py [--quick]
"""
import sys
import torch

sys.path.insert(0, ".")
from theanompi_b200.ops import native  # noqa: E402

L = native.require()
dev = torch.device("cuda:0")
BF = torch.bfloat16
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)


def timeit(fn, reps=8):
    st = torch.cuda.current_stream()
    for _ in range(2):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record(st)
        fn()
        e1.record(st)
        e1.synchronize()
        ts.append(e0.elapsed_time(e1) * 1e3)
    ts.sort()
    return ts[len(ts) // 2]


def S():
    return torch.cuda.current_stream().cuda_stream


def conv_case(name, N, H, W, C, O, K, s, p):
    Ho = (H + 2 * p - K) // s + 1
    x = torch.randn(N, H, W, C, device=dev).to(BF)
    w = torch.randn(O, K, K, C, device=dev).to(BF) * 0.05
    y = torch.empty(N, Ho, Ho, O, device=dev, dtype=BF)
    dy = torch.randn(N, Ho, Ho, O, device=dev).to(BF)
    dw = torch.empty(O, K, K, C, device=dev, dtype=torch.float32)
    b = torch.zeros(O, device=dev)
    flops = 2.0 * N * Ho * Ho * O * K * K * C

    def f():
        L.conv_fprop(x.data_ptr(), w.data_ptr(), y.data_ptr(), b.data_ptr(), N, H, W, C, 0, C, K, K, Ho, Ho, s, p, O, O, 1, 0, 0, S())

    def g():
        L.conv_wgrad(dy.data_ptr(), x.data_ptr(), dw.data_ptr(), N, H, W, C, 0, C, K, K, Ho, Ho, s, p, O, O, 0, S())

    return [(name + " fprop", f, flops), (name + " wgrad", g, flops)]


def gemm_case(name, M, Nn, K, a_mn, b_mn, out_bf16):
    A = torch.randn((K, M) if a_mn else (M, K), device=dev).to(BF)
    B = torch.randn((K, Nn) if b_mn else (Nn, K), device=dev).to(BF)
    Cc = torch.empty(M, Nn, device=dev, dtype=BF if out_bf16 else torch.float32)

    def f():
        L.gemm(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), 0, M, Nn, K, A.shape[1], B.shape[1], Nn, int(a_mn), int(b_mn),
               int(out_bf16), 0, 0, 1.0, 0, 0, 0, S())

    return [(name, f, 2.0 * M * Nn * K)]


def main():
    quick = "--quick" in sys.argv
    cases = []
    cases += conv_case("conv2g 27x27 48->128 k5", 128, 27, 27, 48, 128, 5, 1, 2)
    cases += conv_case("conv3 13x13 256->384 k3", 128, 13, 13, 256, 384, 3, 1, 1)
    cases += conv_case("conv4g 13x13 192->192 k3", 128, 13, 13, 192, 192, 3, 1, 1)
    cases += conv_case("conv5g 13x13 192->128 k3", 128, 13, 13, 192, 128, 3, 1, 1)
    cases += conv_case("conv1s2d 57x57 48->96 k3", 128, 57, 57, 48, 96, 3, 1, 0)
    cases += gemm_case("fc6 fwd 128x4096x9216", 128, 4096, 9216, 0, 0, 1)
    cases += gemm_case("fc6 wgrad 4096x9216x128 (mn,mn)", 4096, 9216, 128, 1, 1, 0)
    cases += gemm_case("gemm 8192^3 (k,k) bf16 out", 8192, 8192, 8192, 0, 0, 1)
    if not quick:
        cases += gemm_case("gemm 8192^3 (mn,mn) bf16 out", 8192, 8192, 8192, 1, 1, 1)
        cases += gemm_case("gemm 4096x4096x4096 (k,k)", 4096, 4096, 4096, 0, 0, 1)
    print("%-40s %9s %9s | %9s %9s %9s  (us; TF = TFLOP/s of the normal run)" % ("case", "normal", "TF", "noA", "noB", "noMMA"))
    for name, fn, flops in cases:
        L.gemm_set_debug(0)
        t = timeit(fn)
        row = [t, flops / t / 1e6]
        for d in (1, 2, 4):
            L.gemm_set_debug(d)
            row.append(timeit(fn, reps=4))
        L.gemm_set_debug(0)
        print("%-40s %9.1f %9.1f | %9.1f %9.1f %9.1f" % ((name,) + tuple(row)), flush=True)
    # cuBLAS yardstick for the square case
    a = torch.randn(8192, 8192, device=dev).to(BF)
    b = torch.randn(8192, 8192, device=dev).to(BF)
    t = timeit(lambda: torch.matmul(a, b))
    print("%-40s %9.1f %9.1f" % ("cuBLAS 8192^3 (torch.matmul)", t, 2.0 * 8192 ** 3 / t / 1e6))


if __name__ == "__main__":
    main()
