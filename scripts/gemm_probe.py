"""Bottleneck probe for the wgmma GEMM / implicit-conv kernel on the AlexNet-128b shapes.

For each shape: time the kernel (CUDA events, L2 flushed by a 256 MiB write between repeats) normally and with the
probe knobs of ``gemm_set_debug`` (1 = no A loads, 2 = no B loads, 4 = no MMAs) and print achieved TFLOP/s and the
L2→SM operand traffic rate, so "L2-bandwidth bound" vs "issue bound" vs "latency bound" can be read off one table.

    python scripts/gemm_probe.py [--quick] [--convs]

``--convs``: only the AlexNet-128b convolution GEMMs (fprop, dgrad, wgrad; grouped layers as one two-group launch), without
the probe knobs.  The "issued" column is the MACs the wgmma instructions issue under the launcher's tile plan (zero-filled
rows, columns and channels included) over the useful MACs.
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


def issued_macs(kind, M, N, Cg, taps, groups, f32=False):
    """MACs the wgmma instructions of one conv launch issue (zero-filled rows / columns / channels included) under the
    launcher's tile plan, or None when the extension has no planner export."""
    if not hasattr(L, "gemm_plan_conv"):
        return None
    BK, MMA_K = (32, 8) if f32 else (64, 16)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    if kind == 2:                                            # wgrad: M = out-channels, N = (tap, chunk) boxes, K = pixels
        boxes = taps * -(-Cg // BK)
        bn, _, _ = L.gemm_plan_conv(2, M, boxes * BK, groups, -(-N // BK), 0, sms)
        return groups * (-(-M // 64) * 64) * (-(-boxes * BK // bn) * bn) * (-(-N // BK) * BK)
    chunks = -(-Cg // BK)
    tail = -(-(Cg - (chunks - 1) * BK) // MMA_K) * MMA_K     # the last chunk's k-steps
    bn, _, _ = L.gemm_plan_conv(kind, M, N, groups, taps * chunks, 0 if (f32 and kind == 1) else 1, sms)
    return groups * (-(-M // 64) * 64) * (-(-N // bn) * bn) * taps * ((chunks - 1) * BK + tail)


def conv_case(name, N, H, W, C, O, K, s, p, groups=1, dgrad=True):
    """fprop, dgrad (stride 1) and wgrad of a convolution with C input / O output channels PER GROUP; two groups run in one
    launch, as the model does."""
    Ho = (H + 2 * p - K) // s + 1
    G = groups
    x = torch.randn(N, H, W, C * G, device=dev).to(BF)
    ws = [torch.randn(O, K, K, C, device=dev).to(BF) * 0.05 for _ in range(G)]
    y = torch.empty(N, Ho, Ho, O * G, device=dev, dtype=BF)
    dy = torch.randn(N, Ho, Ho, O * G, device=dev).to(BF)
    dx = torch.empty(N, H, W, C * G, device=dev, dtype=BF)
    dws = [torch.empty(O, K, K, C, device=dev, dtype=torch.float32) for _ in range(G)]
    b = torch.zeros(O * G, device=dev)
    M = N * Ho * Ho
    useful = float(G) * M * O * K * K * C
    es = 2

    def f():
        if G == 1:
            L.conv_fprop(x.data_ptr(), ws[0].data_ptr(), y.data_ptr(), b.data_ptr(), N, H, W, C, 0, C, K, K, Ho, Ho, s, p, O, O, 1, 0, 0, S())
        else:
            L.conv_fprop2(x.data_ptr(), ws[0].data_ptr(), ws[1].data_ptr(), y.data_ptr(), y.data_ptr() + O * es, b.data_ptr(),
                          b.data_ptr() + O * 4, N, H, W, C * G, 0, C, C, K, K, Ho, Ho, s, p, O, O * G, 1, 0, 0, S())

    def d():                                                 # dx = conv(dy, mirrored transposed w), padding K - 1 - p
        if G == 1:
            L.conv_fprop(dy.data_ptr(), ws[0].data_ptr(), dx.data_ptr(), 0, N, Ho, Ho, O, 0, O, K, K, H, W, 1, K - 1 - p, C, C, 0, 1, 0, S())
        else:
            L.conv_fprop2(dy.data_ptr(), ws[0].data_ptr(), ws[1].data_ptr(), dx.data_ptr(), dx.data_ptr() + C * es, 0, 0, N, Ho, Ho,
                          O * G, 0, O, O, K, K, H, W, 1, K - 1 - p, C, C * G, 0, 1, 0, S())

    def g():
        if G == 1:
            L.conv_wgrad(dy.data_ptr(), x.data_ptr(), dws[0].data_ptr(), N, H, W, C, 0, C, K, K, Ho, Ho, s, p, O, O, 0, 0, S())
        else:
            L.conv_wgrad2(dy.data_ptr(), dy.data_ptr() + O * es, x.data_ptr(), dws[0].data_ptr(), dws[1].data_ptr(), N, H, W, C * G,
                          0, C, C, K, K, Ho, Ho, s, p, O, O * G, 0, 0, S())

    cases = [(name + " fprop", f, useful, issued_macs(0, M, O, C, K * K, G))]
    if dgrad:
        cases.append((name + " dgrad", d, useful, issued_macs(1, M, C, O, K * K, G)))
    cases.append((name + " wgrad", g, useful, issued_macs(2, O, M, C, K * K, G)))
    return cases


def gemm_case(name, M, Nn, K, a_mn, b_mn, out_bf16):
    A = torch.randn((K, M) if a_mn else (M, K), device=dev).to(BF)
    B = torch.randn((K, Nn) if b_mn else (Nn, K), device=dev).to(BF)
    Cc = torch.empty(M, Nn, device=dev, dtype=BF if out_bf16 else torch.float32)

    def f():
        L.gemm(A.data_ptr(), B.data_ptr(), Cc.data_ptr(), 0, M, Nn, K, A.shape[1], B.shape[1], Nn, int(a_mn), int(b_mn),
               int(out_bf16), 0, 0, 1.0, 0, 0, 0, S())

    return [(name, f, float(M) * Nn * K, None)]


def main():
    quick = "--quick" in sys.argv
    convs_only = "--convs" in sys.argv
    cases = []
    cases += conv_case("conv1 s2d 57x57 48->96 k3", 128, 57, 57, 48, 96, 3, 1, 0, dgrad=False)
    cases += conv_case("conv2 27x27 2x(48->128) k5", 128, 27, 27, 48, 128, 5, 1, 2, groups=2)
    cases += conv_case("conv3 13x13 256->384 k3", 128, 13, 13, 256, 384, 3, 1, 1)
    cases += conv_case("conv4 13x13 2x(192->192) k3", 128, 13, 13, 192, 192, 3, 1, 1, groups=2)
    cases += conv_case("conv5 13x13 2x(192->128) k3", 128, 13, 13, 192, 128, 3, 1, 1, groups=2)
    if not convs_only:
        cases += gemm_case("fc6 fwd 128x4096x9216", 128, 4096, 9216, 0, 0, 1)
        cases += gemm_case("fc6 wgrad 4096x9216x128 (mn,mn)", 4096, 9216, 128, 1, 1, 0)
        cases += gemm_case("gemm 8192^3 (k,k) bf16 out", 8192, 8192, 8192, 0, 0, 1)
    if not (quick or convs_only):
        cases += gemm_case("gemm 8192^3 (mn,mn) bf16 out", 8192, 8192, 8192, 1, 1, 1)
        cases += gemm_case("gemm 4096x4096x4096 (k,k)", 4096, 4096, 4096, 0, 0, 1)
    print("%-40s %9s %9s %8s | %9s %9s %9s  (us; TF = TFLOP/s of useful work in the normal run; issued / useful MACs)"
          % ("case", "normal", "TF", "issued", "noA", "noB", "noMMA"))
    tot = 0.0
    for name, fn, macs, issued in cases:
        L.gemm_set_debug(0)
        t = timeit(fn)
        tot += t
        row = [t, 2.0 * macs / t / 1e6, "%8.3f" % (issued / macs) if issued else "%8s" % "-"]
        if not convs_only:
            for dbg in (1, 2, 4):
                L.gemm_set_debug(dbg)
                row.append(timeit(fn, reps=4))
            L.gemm_set_debug(0)
        print(("%-40s %9.1f %9.1f %s" % ((name,) + tuple(row[:3]))) + ("".join(" | %9.1f %9.1f %9.1f" % tuple(row[3:]) if len(row) > 3 else "")),
              flush=True)
    print("%-40s %9.1f" % ("sum of the rows above", tot))
    if convs_only:
        return
    # cuBLAS yardstick for the square case
    a = torch.randn(8192, 8192, device=dev).to(BF)
    b = torch.randn(8192, 8192, device=dev).to(BF)
    t = timeit(lambda: torch.matmul(a, b))
    print("%-40s %9.1f %9.1f" % ("cuBLAS 8192^3 (torch.matmul)", t, 2.0 * 8192 ** 3 / t / 1e6))


if __name__ == "__main__":
    main()
