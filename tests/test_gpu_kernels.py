"""Numerics of every hand-written sm_90a kernel against a plain-PyTorch fp32 reference
of the same op (run with ``pytest -m gpu`` on an H100)."""
import numpy as np
import pytest
import torch

from theanompi_b200 import ops
from theanompi_b200.ops import reference as ref

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _impl():
    from theanompi_b200.ops import cuda_impl
    return cuda_impl


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


# ------------------------------------------------------------------ GEMM (wgmma / TMA)
@pytest.mark.parametrize("a_mn,b_mn", [(False, False), (False, True), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,K", [(128, 128, 64), (256, 384, 512), (200, 136, 328), (128, 4096, 1024), (1000, 72, 136),
                                   (2304, 2200, 192)])   # the last one exercises the banded (L2-friendly) tile raster
def test_gemm_majors(M, N, K, a_mn, b_mn):
    ci = _impl()
    torch.manual_seed(0)
    A = torch.randn(M, K, device=DEV).to(torch.bfloat16)
    B = torch.randn(N, K, device=DEV).to(torch.bfloat16)
    want = A.float() @ B.float().t()
    a = A.t().contiguous() if a_mn else A
    b = B.t().contiguous() if b_mn else B
    lda = M if a_mn else K
    ldb = N if b_mn else K
    out = ci.gemm(a, b, M, N, K, a_mn=a_mn, b_mn=b_mn, out_dtype=torch.float32, lda=lda, ldb=ldb)
    torch.cuda.synchronize()
    assert rel_err(out, want) < 2e-3, (rel_err(out, want))


@pytest.mark.parametrize("bn", [32, 64, 128])
def test_gemm_epilogue_bias_relu_bf16(bn):
    ci = _impl()
    torch.manual_seed(1)
    M, N, K = 384, 256, 192
    A = torch.randn(M, K, device=DEV).to(torch.bfloat16)
    B = torch.randn(N, K, device=DEV).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV)
    want = torch.relu(A.float() @ B.float().t() + bias)
    out = ci.gemm(A, B, M, N, K, bias=bias, bias_mode=1, relu=True, lda=K, ldb=K, bn=bn)
    torch.cuda.synchronize()
    assert out.dtype == torch.bfloat16
    assert rel_err(out, want) < 1e-2


@pytest.mark.parametrize("M,N,K,a_mn,b_mn", [(4096, 1024, 256, False, False), (4000, 520, 200, False, True),
                                             (4232, 1024, 128, True, False), (4196, 640, 192, False, False)])
def test_gemm_tall_tiles(M, N, K, a_mn, b_mn):
    """bf16-output GEMMs with many rows run 256-row CTA tiles (two MMAs per k-step sharing the B tile); the last tile's
    second half may be partial (4232, 4000) or entirely out of range (4196)."""
    ci = _impl()
    torch.manual_seed(21)
    A = torch.randn((K, M) if a_mn else (M, K), device=DEV).to(torch.bfloat16)
    B = torch.randn((K, N) if b_mn else (N, K), device=DEV).to(torch.bfloat16)
    bias = torch.randn(N, device=DEV)
    Af = A.float().t() if a_mn else A.float()
    Bf = B.float() if b_mn else B.float().t()
    want = torch.relu(Af @ Bf + bias)
    out = ci.gemm(A, B, M, N, K, a_mn=a_mn, b_mn=b_mn, bias=bias, bias_mode=1, relu=True, lda=A.shape[1], ldb=B.shape[1])
    torch.cuda.synchronize()
    assert rel_err(out, want) < 1e-2


def test_gemm_splitk_and_strided_out():
    ci = _impl()
    torch.manual_seed(2)
    M, N, K = 96, 363, 8192          # conv1-wgrad-like: tiny output, long K
    A = torch.randn(K, M, device=DEV).to(torch.bfloat16)      # MN-major storage [K, M]
    B = torch.randn(K, 368, device=DEV).to(torch.bfloat16)    # MN-major storage [K, N] with pitch 368
    want = A.float().t() @ B.float()[:, :N]
    out = torch.full((M, N), 7.0, device=DEV)
    ci.gemm(A, B, M, N, K, a_mn=True, b_mn=True, out=out, lda=M, ldb=368, ldc=N)
    torch.cuda.synchronize()
    assert rel_err(out, want) < 2e-3


# ------------------------------------------------------------------ layer kernels
def test_linear_fwd_bwd():
    torch.manual_seed(3)
    x = torch.randn(128, 512, device=DEV).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(256, 512, device=DEV) * 0.05).to(torch.bfloat16).requires_grad_(True)
    b = torch.randn(256, device=DEV).requires_grad_(True)
    y = ops.linear_bias_act(x, w, b, True)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr, wr, br = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True), b.detach().clone().requires_grad_(True)
    yr = ref.linear_bias_act(xr, wr, br, True)
    yr.backward((dy.float() * 1.0))
    assert rel_err(y, yr) < 1e-2
    assert rel_err(x.grad, xr.grad) < 2e-2
    assert rel_err(w.grad, wr.grad) < 2e-2
    assert rel_err(b.grad, br.grad) < 2e-2


@pytest.mark.parametrize("B,I,O,relu", [(128, 2048, 1000, False), (64, 4096, 512, True)])
def test_linear_small_batch_splitk_forward(B, I, O, relu):
    """Small-batch FC forward: n-tiles x split-K into an fp32 scratch tile + the bias / ReLU / bf16 finishing kernel."""
    torch.manual_seed(31)
    x = torch.randn(B, I, device=DEV).to(torch.bfloat16).requires_grad_(True)
    w = (torch.randn(O, I, device=DEV) * 0.03).to(torch.bfloat16).requires_grad_(True)
    b = torch.randn(O, device=DEV).requires_grad_(True)
    y = ops.linear_bias_act(x, w, b, relu)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr, wr, br = x.detach().float().requires_grad_(True), w.detach().float().requires_grad_(True), b.detach().clone().requires_grad_(True)
    yr = ref.linear_bias_act(xr, wr, br, relu)
    yr.backward(dy.float())
    assert y.dtype == torch.bfloat16 and rel_err(y, yr) < 1e-2
    assert rel_err(x.grad, xr.grad) < 2e-2 and rel_err(w.grad, wr.grad) < 2e-2 and rel_err(b.grad, br.grad) < 2e-2


@pytest.mark.parametrize("cfg", [
    dict(N=4, H=31, W=31, C=3, O=32, k=11, s=4, p=0),      # conv1-like (C=3, K % 8 != 0)
    dict(N=3, H=64, W=64, C=3, O=64, k=7, s=2, p=3),       # ResNet / GoogLeNet stem: padding folded into the space-to-depth image
    dict(N=2, H=33, W=37, C=3, O=16, k=5, s=2, p=2),       # odd sizes, padded, strided few-channel conv
    dict(N=3, H=13, W=13, C=64, O=96, k=3, s=1, p=1),
    dict(N=2, H=14, W=14, C=32, O=48, k=5, s=1, p=2),
    dict(N=2, H=12, W=12, C=64, O=32, k=1, s=1, p=0),      # 1x1
    dict(N=2, H=16, W=16, C=64, O=128, k=3, s=2, p=1),     # strided: implicit fprop/wgrad, explicit dgrad
    dict(N=2, H=9, W=9, C=16, O=24, k=1, s=1, p=0),        # C < 64: TMA zero-fills the channel tail
    dict(N=2, H=12, W=12, C=192, O=64, k=3, s=1, p=1),     # 3 channel chunks per tap
    dict(N=3, H=27, W=27, C=48, O=128, k=5, s=1, p=2),     # AlexNet conv2 group shape (C = 48)
    dict(N=40, H=13, W=13, C=256, O=384, k=3, s=1, p=1),   # many tiles + split-K wgrad
    dict(N=32, H=27, W=27, C=48, O=128, k=5, s=1, p=2),    # enough pixels for 256-row tiles in fprop and dgrad (BN = 64)
    dict(N=80, H=13, W=13, C=192, O=192, k=3, s=1, p=1),   # 256-row tiles with a ragged last tile
])
def test_conv_fwd_bwd(cfg):
    torch.manual_seed(4)
    N, H, W, C, O, k, s, p = (cfg[q] for q in "N H W C O k s p".split())
    first = C == 3
    x = torch.randn(N, H, W, C, device=DEV).to(torch.bfloat16)
    if not first:
        x.requires_grad_(True)
    w = (torch.randn(O, k, k, C, device=DEV) * 0.1).to(torch.bfloat16).requires_grad_(True)
    b = torch.randn(O, device=DEV).requires_grad_(True)
    y = ops.conv2d_bias_act(x, w, b, s, p, 1, True)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(not first)
    wr, br = w.detach().float().requires_grad_(True), b.detach().clone().requires_grad_(True)
    yr = ref.conv2d_bias_act(xr, wr, br, s, p, 1, True)
    # reference backward with the SAME mask (bf16 rounding can flip y>0 at exactly 0)
    dxr, dwr, dbr = ref.conv2d_bias_act_bwd(xr.detach(), wr.detach(), y.detach().float(), dy.float(), s, p, 1, True, not first)
    assert rel_err(y, yr) < 1e-2
    assert rel_err(w.grad, dwr) < 2e-2
    assert rel_err(b.grad, dbr) < 2e-2
    if not first:
        assert rel_err(x.grad, dxr) < 2e-2


@pytest.mark.parametrize("N,C,O", [(2, 32, 64), (2, 96, 256), (64, 96, 256)])    # the last: both groups in one launch of 256-row tiles
def test_conv_group2(N, C, O):
    torch.manual_seed(5)
    H, W = 13, 13
    x = torch.randn(N, H, W, C, device=DEV).to(torch.bfloat16).requires_grad_(True)
    ws = [(torch.randn(O // 2, 3, 3, C // 2, device=DEV) * 0.1).to(torch.bfloat16).requires_grad_(True) for _ in range(2)]
    bs = [torch.randn(O // 2, device=DEV).requires_grad_(True) for _ in range(2)]
    y = ops.conv2d_group2_bias_act(x, ws[0], bs[0], ws[1], bs[1], 1, 1, True)
    dy = torch.randn_like(y)
    y.backward(dy)
    wfull = torch.cat([w.detach().float() for w in ws], 0)
    bfull = torch.cat([b.detach() for b in bs], 0)
    yr = ref.conv2d_bias_act(x.detach().float(), wfull, bfull, 1, 1, 2, True)
    dxr, dwr, dbr = ref.conv2d_bias_act_bwd(x.detach().float(), wfull, y.detach().float(), dy.float(), 1, 1, 2, True, True)
    assert rel_err(y, yr) < 1e-2
    assert rel_err(x.grad, dxr) < 2e-2
    assert rel_err(torch.cat([w.grad for w in ws], 0), dwr) < 2e-2
    assert rel_err(torch.cat([b.grad for b in bs], 0), dbr) < 2e-2


@pytest.mark.parametrize("groups,C,O,H,k,st,pd", [(1, 16, 64, 13, 3, 1, 1), (2, 32, 256, 15, 5, 1, 2), (1, 3, 96, 35, 11, 4, 0)])
def test_conv_pool_fused_backward(groups, C, O, H, k, st, pd):
    """conv(+ReLU)→max-pool block: the fused pool-scatter + ReLU-mask + bias-grad backward kernel vs the unfused
    conv → pool2d composition and vs the fp32 reference."""
    torch.manual_seed(11)
    N = 2
    pool = (3, 2, 0, "max")

    def make():
        torch.manual_seed(12)
        x = torch.randn(N, H, H, C, device=DEV).to(torch.bfloat16).requires_grad_(C >= 8)
        ws = [(torch.randn(O // groups, k, k, C // groups, device=DEV) * 0.1).to(torch.bfloat16).requires_grad_(True) for _ in range(groups)]
        bs = [(torch.randn(O // groups, device=DEV) * 0.1).requires_grad_(True) for _ in range(groups)]
        return x, ws, bs

    def run(fused):
        x, ws, bs = make()
        pl = pool if fused else None
        if groups == 1:
            y = ops.conv2d_bias_act(x, ws[0], bs[0], st, pd, 1, True, pl)
        else:
            y = ops.conv2d_group2_bias_act(x, ws[0], bs[0], ws[1], bs[1], st, pd, True, pl)
        if not fused:
            y = ops.pool2d(y, *pool)
        torch.manual_seed(13)
        dy = torch.randn_like(y)
        y.backward(dy)
        return y, x.grad, torch.cat([w.grad for w in ws], 0), torch.cat([b.grad for b in bs], 0), dy

    yf, dxf, dwf, dbf, dy = run(True)
    yu, dxu, dwu, dbu, _ = run(False)
    assert torch.equal(yf, yu)
    assert rel_err(dwf, dwu) < 1e-3 and rel_err(dbf, dbu) < 1e-3
    if dxf is not None:
        assert rel_err(dxf, dxu) < 1e-3
    # fp32 reference of the block's backward, pooling the kernel's own (bf16) conv output so the argmax cannot differ by a
    # rounding tie
    x, ws, bs = make()
    with torch.no_grad():
        if groups == 1:
            yc = ops.conv2d_bias_act(x.detach(), ws[0].detach(), bs[0].detach(), st, pd, 1, True)
        else:
            yc = ops.conv2d_group2_bias_act(x.detach(), ws[0].detach(), bs[0].detach(), ws[1].detach(), bs[1].detach(), st, pd, True)
    wr = torch.cat([w.detach().float() for w in ws], 0)
    br = torch.cat([b.detach() for b in bs], 0)
    ycr = ref.conv2d_bias_act(x.detach().float(), wr, br, st, pd, groups, True)
    assert rel_err(yc, ycr) < 1e-2
    ypr = ref.pool2d(yc.float(), *pool)
    assert rel_err(yf, ypr) < 1e-2
    dyc = ref.pool2d_bwd(yc.float(), ypr, dy.float(), *pool)
    dxr, dwr, dbr = ref.conv2d_bias_act_bwd(x.detach().float(), wr, yc.float(), dyc, st, pd, groups, True, dxf is not None)
    assert rel_err(dwf, dwr) < 3e-2 and rel_err(dbf, dbr) < 3e-2
    if dxf is not None:
        assert rel_err(dxf, dxr) < 3e-2


@pytest.mark.parametrize("mode,k,s,p", [("max", 3, 2, 0), ("max", 2, 2, 0), ("max", 3, 1, 1), ("avg", 5, 3, 0), ("avg", 7, 1, 0)])
def test_pool(mode, k, s, p):
    torch.manual_seed(6)
    x = torch.randn(2, 15, 15, 16, device=DEV).to(torch.bfloat16).requires_grad_(True)
    y = ops.pool2d(x, k, s, p, mode)
    dy = torch.randn_like(y)
    y.backward(dy)
    xr = x.detach().float().requires_grad_(True)
    yr = ref.pool2d(xr, k, s, p, mode)
    yr.backward(dy.float())
    assert rel_err(y, yr) < 1e-2
    assert rel_err(x.grad, xr.grad) < 2e-2


def test_lrn():
    torch.manual_seed(7)
    x = (torch.randn(2, 9, 9, 96, device=DEV) * 20).to(torch.bfloat16).requires_grad_(True)
    y = ops.lrn(x)
    dy = torch.randn_like(y)
    y.backward(dy)
    yr, _ = ref.lrn(x.detach().float())
    dxr = ref.lrn_bwd(x.detach().float(), dy.float())
    assert rel_err(y, yr) < 1e-2
    assert rel_err(x.grad, dxr) < 2e-2


def test_dropout_mask_statistics_and_bwd():
    x = torch.ones(128, 4096, device=DEV, dtype=torch.bfloat16, requires_grad=True)
    y = ops.dropout(x, 0.5, True, layer_id=3)
    keep = float(y.float().mean())
    assert abs(keep - 0.5) < 0.01
    y.backward(torch.ones_like(y))
    assert torch.equal(x.grad, y.detach())
    from theanompi_b200.ops import cuda_impl
    cuda_impl.advance_step(x.device)
    y2 = ops.dropout(x, 0.5, True, layer_id=3)
    assert not torch.equal(y2, y)                      # new step → new mask
    assert float((ops.dropout(x, 0.5, False) .float().mean())) == pytest.approx(0.5, abs=1e-3)


def test_softmax_xent():
    torch.manual_seed(8)
    lg = (torch.randn(128, 1000, device=DEV) * 3).to(torch.bfloat16).requires_grad_(True)
    lab = torch.randint(0, 1000, (128,), device=DEV)
    loss, e1, e5 = ops.softmax_xent(lg, lab)
    loss.backward()
    lr, e1r, e5r, dlr = ref.softmax_xent(lg.detach().float(), lab)
    assert abs(float(loss) - float(lr)) < 1e-3
    assert abs(float(e1) - float(e1r)) < 1e-6
    assert abs(float(e5) - float(e5r)) < 1e-6
    assert rel_err(lg.grad, dlr) < 2e-2


def test_crop_mirror_normalize():
    torch.manual_seed(9)
    x = torch.randint(0, 256, (4, 32, 32, 3), device=DEV, dtype=torch.uint8)
    mean = torch.rand(32, 32, 3, device=DEV) * 255
    offs = torch.tensor([[0, 0], [3, 4], [5, 1], [2, 2]], dtype=torch.int32, device=DEV)
    flips = torch.tensor([0, 1, 1, 0], dtype=torch.uint8, device=DEV)
    out = ops.crop_mirror_normalize(x, mean, 1 / 255.0, (27, 27), offs, flips)
    want = ref.crop_mirror_normalize(x.cpu(), mean.cpu(), 1 / 255.0, (27, 27), offs.cpu(), flips.cpu())
    # per-channel scale (1 / 255 / img_std, ref proc_load_mpi.py:99)
    cs = torch.tensor([1 / 255.0 / 0.229, 1 / 255.0 / 0.224, 1 / 255.0 / 0.225])
    out_c = ops.crop_mirror_normalize(x, mean, cs.to(DEV), (27, 27), offs, flips)
    want_c = ref.crop_mirror_normalize(x.cpu(), mean.cpu(), cs, (27, 27), offs.cpu(), flips.cpu())
    assert torch.allclose(out_c.float().cpu(), want_c.float(), atol=3e-2, rtol=2e-2)
    assert rel_err(out.cpu(), want) < 1e-2


def test_sgd_flat_matches_reference():
    from theanompi_b200.parallel.arena import FlatArena
    torch.manual_seed(10)
    ps = [torch.randn(300, 70), torch.randn(300), torch.randn(5000, 3), torch.randn(17)]
    wt = ["W", "b", "W", "b"]
    arena = FlatArena([p.clone() for p in ps], wt, DEV, weight_decay=5e-4)
    cpu = FlatArena([p.clone() for p in ps], wt, "cpu", weight_decay=5e-4)
    g = torch.randn(arena.numel)
    arena.G.copy_(g); cpu.G.copy_(g)
    from theanompi_b200.utils.opt import FlatSGD
    for a in (arena, cpu):
        a.hyper[0] = 0.01
        s = FlatSGD(a, 0.9, False, True)
        s.step(0.01, 1)
        s.step(0.01, 1)
    torch.cuda.synchronize()
    assert rel_err(arena.W.cpu(), cpu.W) < 1e-5
    assert rel_err(arena.U.cpu(), cpu.U) < 1e-5
    assert rel_err(arena.H.float().cpu(), cpu.W) < 1e-2


def test_legacy_kernels_k1_k5():
    L = ops.native.require()
    st = torch.cuda.current_stream().cuda_stream
    x = torch.randn(10000, device=DEV)
    h = torch.empty(10000, device=DEV, dtype=torch.float16)
    L.cast_flat(x.data_ptr(), h.data_ptr(), x.numel(), 0, st)
    back = torch.empty_like(x)
    L.cast_flat(h.data_ptr(), back.data_ptr(), x.numel(), 1, st)
    assert rel_err(back, x.half().float()) == 0
    src = torch.randn(4 * 2500, device=DEV)
    dst = torch.empty(2500, device=DEV)
    L.sum_chunks(src.data_ptr(), dst.data_ptr(), 2500, 4, 0, st)
    assert rel_err(dst, src.view(4, 2500).sum(0)) < 1e-6
    a, b = torch.randn(999, device=DEV), torch.randn(999, device=DEV)
    want = a + b
    L.vecadd(a.data_ptr(), b.data_ptr(), 999, 0, st)
    assert rel_err(a, want) < 1e-6


# ------------------------------------------------------------------ batch norm (+ residual)(+ ReLU), residual add
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("relu,with_res", [(False, False), (True, False), (True, True), (False, True)])
def test_batch_norm_fwd_bwd(dtype, relu, with_res):
    from theanompi_b200.ops import precision
    old = precision.precision()
    precision.set_precision("tf32" if dtype == torch.float32 else "bf16")
    try:
        torch.manual_seed(11)
        N, H, W, C = 8, 14, 14, 72 if dtype == torch.float32 else 96
        x = (torch.randn(N, H, W, C, device=DEV) * 2 + 0.5).to(dtype).requires_grad_(True)
        res = torch.randn(N, H, W, C, device=DEV).to(dtype).requires_grad_(True) if with_res else None
        g = (torch.rand(C, device=DEV) + 0.5).requires_grad_(True)
        b = torch.randn(C, device=DEV).requires_grad_(True)
        rm, rv = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
        y = ops.batch_norm(x, g, b, rm, rv, True, 0.1, 1e-5, relu, res)
        dy = torch.randn_like(y)
        y.backward(dy)
        # fp32 torch reference on the same (rounded) inputs
        xr = x.detach().float().requires_grad_(True)
        rr = res.detach().float().requires_grad_(True) if with_res else None
        gr, br = g.detach().clone().requires_grad_(True), b.detach().clone().requires_grad_(True)
        rm2, rv2 = torch.zeros(C, device=DEV), torch.ones(C, device=DEV)
        yr = torch.nn.functional.batch_norm(xr.permute(0, 3, 1, 2), rm2, rv2, gr, br, True, 0.1, 1e-5).permute(0, 2, 3, 1)
        if with_res:
            yr = yr + rr
        if relu:
            yr = torch.relu(yr)
        # the kernel masks with ITS OWN (rounded) output; use the same mask for the reference gradient
        dyr = dy.float()
        yr.backward(dyr)
        tol = 2e-2 if dtype == torch.bfloat16 else 1e-4
        assert rel_err(y, yr) < tol
        assert rel_err(x.grad, xr.grad) < 3 * tol
        assert rel_err(g.grad, gr.grad) < 3 * tol and rel_err(b.grad, br.grad) < 3 * tol
        if with_res:
            assert rel_err(res.grad, rr.grad) < tol
        assert rel_err(rm, rm2) < 1e-3 and rel_err(rv, rv2) < 1e-3
        # eval mode uses the running statistics
        ye = ops.batch_norm(x.detach(), g.detach(), b.detach(), rm, rv, False, 0.1, 1e-5, relu, res.detach() if with_res else None)
        yer = torch.nn.functional.batch_norm(xr.detach().permute(0, 3, 1, 2), rm2, rv2, gr.detach(), br.detach(), False, 0.1, 1e-5).permute(0, 2, 3, 1)
        if with_res:
            yer = yer + rr.detach()
        if relu:
            yer = torch.relu(yer)
        assert rel_err(ye, yer) < tol
        # residual add kernel
        a1 = torch.randn(4, 7, 7, 40, device=DEV).to(dtype).requires_grad_(True)
        a2 = torch.randn(4, 7, 7, 40, device=DEV).to(dtype).requires_grad_(True)
        s = ops.add(a1, a2)
        s.backward(torch.ones_like(s))
        assert rel_err(s, a1.detach().float() + a2.detach().float()) < tol
        assert torch.equal(a1.grad, torch.ones_like(a1)) and torch.equal(a2.grad, torch.ones_like(a2))
    finally:
        precision.set_precision(old)


def test_adam_flat_matches_torch():
    from theanompi_b200.parallel.arena import FlatArena
    from theanompi_b200.utils.opt import FlatAdam
    torch.manual_seed(4)
    shapes = [(300, 70), (300,), (64, 3, 3, 16)]
    params = [torch.randn(s) * 0.1 for s in shapes]
    arena = FlatArena(params, ["W", "b", "W"], torch.device(DEV), weight_decay=0.0, bias_lr_mult=1.0)
    ref_p = [p.detach().clone().float().to(DEV).requires_grad_(True) for p in arena.params]
    opt = torch.optim.Adam(ref_p, lr=1e-3)
    adam = FlatAdam(arena)
    arena.hyper[0] = 1e-3
    for it in range(5):
        arena.G.normal_()
        for p, q in zip(ref_p, arena.views("G")):
            p.grad = q.detach().clone().view_as(p)
        opt.step()
        adam.step()
    torch.cuda.synchronize()
    for p, q in zip(ref_p, arena.params):
        assert rel_err(q, p) < 1e-5


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_inception_node_matches_composition(dtype):
    """The fused inception node (slice-writing epilogues, 4 streams, native gradient merge) against the fp32 torch composition
    conv / pool / cat of the same weights."""
    from theanompi_b200.ops import precision
    from theanompi_b200.ops.inception import inception
    old = precision.precision()
    precision.set_precision("tf32" if dtype == torch.float32 else "bf16")
    try:
        torch.manual_seed(17)
        N, H, W, C = 8, 14, 14, 192
        n1, nr3, n3, nr5, n5, npj = 64, 96, 128, 16, 32, 32
        x = torch.randn(N, H, W, C, device=DEV).to(dtype).requires_grad_(True)
        shapes = [(n1, 1, 1, C), (nr3, 1, 1, C), (n3, 3, 3, nr3), (nr5, 1, 1, C), (n5, 5, 5, nr5), (npj, 1, 1, C)]
        ws = [(torch.randn(s, device=DEV) * 0.05).to(dtype).requires_grad_(True) for s in shapes]
        bs = [torch.randn(s[0], device=DEV).requires_grad_(True) for s in shapes]
        ps = []
        for w, b in zip(ws, bs):
            ps += [w, b]
        y = inception(x, tuple(ps))
        dy = torch.randn_like(y)
        y.backward(dy)
        torch.cuda.synchronize()
        # fp32 reference, ReLU masks taken from our own outputs where they are visible (final convs)
        F = torch.nn.functional
        xr = x.detach().float().permute(0, 3, 1, 2).requires_grad_(True)
        wr = [w.detach().float().permute(0, 3, 1, 2).requires_grad_(True) for w in ws]
        br = [b.detach().clone().requires_grad_(True) for b in bs]
        a = torch.relu(F.conv2d(xr, wr[0], br[0]))
        b_ = torch.relu(F.conv2d(torch.relu(F.conv2d(xr, wr[1], br[1])), wr[2], br[2], padding=1))
        c = torch.relu(F.conv2d(torch.relu(F.conv2d(xr, wr[3], br[3])), wr[4], br[4], padding=2))
        d = torch.relu(F.conv2d(F.max_pool2d(xr, 3, 1, 1), wr[5], br[5]))
        yr = torch.cat([a, b_, c, d], 1)
        yr.backward(dy.float().permute(0, 3, 1, 2))
        tol = 3e-2 if dtype == torch.bfloat16 else 5e-3
        assert rel_err(y, yr.permute(0, 2, 3, 1)) < tol
        assert rel_err(x.grad, xr.grad.permute(0, 2, 3, 1)) < 2 * tol
        for i in range(6):
            assert rel_err(ws[i].grad, wr[i].grad.permute(0, 2, 3, 1)) < 2 * tol, i
            assert rel_err(bs[i].grad, br[i].grad) < 2 * tol, i
    finally:
        precision.set_precision(old)
