"""Numerics of the GAN kernels on an H100, in both precision modes, against the fp64 / fp32 plain-PyTorch reference: the
transposed convolution (wgmma GEMM + col2im_bias_act), leaky-ReLU / sigmoid in bias_act, relu_bias_bwd and the batch-norm
passes, the flat RMSProp (eager and graph-replayed), the GAN losses and the Philox noise."""
import pytest
import torch

from theanompi_b200.ops import functional as fn
from theanompi_b200.ops import native, precision
from theanompi_b200.ops import reference as ref
from theanompi_b200.parallel.arena import FlatArena
from theanompi_b200.utils.opt import FlatRMSProp

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {"bf16": 2e-2, "tf32": 5e-3}


def _ci():
    from theanompi_b200.ops import cuda_impl
    return cuda_impl


def rel_err(a, b):
    a, b = a.double(), b.double()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.fixture(params=["bf16", "tf32"])
def mode(request):
    old = precision.precision()
    precision.set_precision(request.param)
    yield request.param
    precision.set_precision(old)


# (N, Cin, Cout, c_real, Hi): the MNIST DCGAN generator layers 128->64 at 7->14 and 64->8 (1 real channel) at 14->28, and the
# CIFAR-10 ones 128->64 at 8->16 and 64->8 (3 real channels) at 16->32; all 5x5, stride 2, pad 2, output_padding 1
SHAPES = [(64, 128, 64, 64, 7), (64, 64, 8, 1, 14), (64, 128, 64, 64, 8), (64, 64, 8, 3, 16)]


@pytest.mark.parametrize("N,Cin,Cout,c_real,Hi", SHAPES)
@pytest.mark.parametrize("act", ["none", "relu", "sigmoid"])
def test_conv_transpose_matches_fp64_reference(mode, N, Cin, Cout, c_real, Hi, act):
    if act == "none" and c_real < Cout:
        c_real = Cout                                    # padding is zeroed through the bias / activation pass only
    ci = _ci()
    dt = precision.act_dtype()
    if mode == "tf32" and Cout == 8:
        Cout = 4 if c_real < 4 else 8                    # fp32 activations pad to 4 channels
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(N, Hi, Hi, Cin, device=DEV, generator=g).to(dt)
    w = torch.randn(Cin, 5, 5, Cout, device=DEV, generator=g) * (1.0 / (Cin * 25) ** 0.5)
    w[..., c_real:] = 0
    b = torch.randn(Cout, device=DEV, generator=g) * 0.1
    b[c_real:] = 0
    wd = w.to(dt)
    y = ci.conv_transpose2d_bias_act(x, wd, b, 2, 2, 1, act, c_real)
    y64 = ref.conv_transpose2d_bias_act(x.double(), wd.double(), b.double(), 2, 2, 1, act, c_real)
    assert y.shape == (N, 2 * Hi, 2 * Hi, Cout) and y.dtype == dt
    assert rel_err(y, y64) < TOL[mode], rel_err(y, y64)
    assert torch.all(y[..., c_real:] == 0)
    dy = torch.randn(y.shape, device=DEV, generator=g).to(dt)  # nonzero on padded channels too: the mask must zero them
    dx, dw, db = ci.conv_transpose2d_bias_act_bwd(x, wd, y, dy, 2, 2, act, True)
    dx64, dw64, db64 = ref.conv_transpose2d_bias_act_bwd(x.double(), wd.double(), y.double(), dy.double(), 2, 2, act)
    torch.cuda.synchronize()
    for got, want, name in ((dx, dx64, "dx"), (dw, dw64, "dW"), (db, db64, "db")):
        assert rel_err(got, want) < TOL[mode], (name, rel_err(got, want))
    assert torch.all(dw64[..., c_real:] == 0) and torch.all(dw[..., c_real:] == 0) and torch.all(db[c_real:] == 0)


@pytest.mark.parametrize("act", ["leaky", "sigmoid"])
def test_bias_act_and_mask_bias_grad(mode, act):
    """bias_act (split-K FC finish and the plain FC path), then relu_bias_bwd's activation mask and bias gradient."""
    ci = _ci()
    dt = precision.act_dtype()
    g = torch.Generator(device=DEV).manual_seed(1)
    for B, I, O in ((64, 6272, 1024), (64, 1024, 1024), (200, 64, 96)):
        x = torch.randn(B, I, device=DEV, generator=g).to(dt)
        w = (torch.randn(O, I, device=DEV, generator=g) / I ** 0.5).to(dt)
        b = torch.randn(O, device=DEV, generator=g)
        y = ci.linear_bias_act(x, w, b, act)
        y64 = ref.linear_bias_act(x.double(), w.double(), b.double(), act)
        assert y.dtype == dt and rel_err(y, y64) < TOL[mode], rel_err(y, y64)
        dy = torch.randn(B, O, device=DEV, generator=g).to(dt)
        dx, dw, db = ci.linear_bias_act_bwd(x, w, y, dy, act, True)
        dx64, dw64, db64 = ref.linear_bias_act_bwd(x.double(), w.double(), y.double(), dy.double(), act)
        for got, want in ((dx, dx64), (dw, dw64), (db, db64)):
            assert rel_err(got, want) < TOL[mode], rel_err(got, want)


def test_leaky_conv_forward_backward(mode):
    """The critic's first layer: 5x5/2 conv + bias + leaky ReLU on the channel-padded image, with an input gradient."""
    ci = _ci()
    dt = precision.act_dtype()
    C = 8 if mode == "bf16" else 4
    g = torch.Generator(device=DEV).manual_seed(2)
    x = torch.rand(64, 28, 28, C, device=DEV, generator=g).to(dt)
    x[..., 1:] = 0
    w = (torch.randn(64, 5, 5, C, device=DEV, generator=g) * 0.1).to(dt)
    b = torch.randn(64, device=DEV, generator=g) * 0.1
    y, cols = ci.conv2d_bias_act(x, w, b, 2, 2, 1, "leaky", return_cols=True)
    y64 = ref.conv2d_bias_act(x.double(), w.double(), b.double(), 2, 2, 1, "leaky")
    assert rel_err(y, y64) < TOL[mode]
    dy = torch.randn(y.shape, device=DEV, generator=g).to(dt)
    dx, dw, db = ci.conv2d_bias_act_bwd(x, w, y, dy, 2, 2, 1, "leaky", True, cols=cols)
    dx64, dw64, db64 = ref.conv2d_bias_act_bwd(x.double(), w.double(), y.double(), dy.double(), 2, 2, 1, "leaky", True)
    for got, want in ((dx, dx64), (dw, dw64), (db, db64)):
        assert rel_err(got, want) < TOL[mode], rel_err(got, want)


@pytest.mark.parametrize("act", ["leaky", "sigmoid"])
@pytest.mark.parametrize("shape", [(64, 14, 14, 128), (64, 1024)])
def test_batch_norm_activations(mode, act, shape):
    ci = _ci()
    dt = precision.act_dtype()
    C = shape[-1]
    g = torch.Generator(device=DEV).manual_seed(3)
    x = (torch.randn(shape, device=DEV, generator=g) * 2 + 0.5).to(dt)
    gamma = torch.rand(C, device=DEV, generator=g) + 0.5
    beta = torch.randn(C, device=DEV, generator=g) * 0.1
    y, mean, rstd = ci.batch_norm_fwd(x, gamma, beta, None, None, True, 0.1, 1e-5, act)
    y_r, mean_r, rstd_r = ref.batch_norm_fwd(x.float(), gamma, beta, None, None, True, 0.1, 1e-5, act)
    assert rel_err(y, y_r) < TOL[mode]
    dy = torch.randn(shape, device=DEV, generator=g).to(dt)
    dx, _, dg, dbeta = ci.batch_norm_bwd(x, dy, y, gamma, mean, rstd, act, False)
    dx_r, _, dg_r, db_r = ref.batch_norm_bwd(x.float(), dy.float(), y.float(), gamma, mean_r, rstd_r, act, False)
    for got, want in ((dx, dx_r), (dg, dg_r), (dbeta, db_r)):
        assert rel_err(got, want) < TOL[mode], rel_err(got, want)


def _arena():
    g = torch.Generator(device=DEV).manual_seed(4)
    ps = [torch.randn(64, 5, 5, 8, device=DEV, generator=g) * 0.02, torch.randn(64, device=DEV, generator=g) * 0.02,
          torch.randn(1024, 6272, device=DEV, generator=g) * 0.02, torch.randn(1, 1024, device=DEV, generator=g) * 0.02]
    return FlatArena(ps, device=DEV, bias_lr_mult=1.0, shadow=True)


@pytest.mark.parametrize("clip", [0.0, 0.01])
def test_rmsprop_flat_matches_reference_and_graph_replay(clip):
    a, b = _arena(), _arena()
    for ar in (a, b):
        ar.hyper[0] = 1e-3
    w0, v0 = a.W.clone(), torch.zeros_like(a.W)
    opt_e, opt_g = FlatRMSProp(a, clip=clip), FlatRMSProp(b, clip=clip)
    g = torch.Generator(device=DEV).manual_seed(5)
    grads = [torch.randn(a.W.shape, device=DEV, generator=g) for _ in range(10)]
    # eager native vs the reference
    w_ref, v_ref = w0.clone(), v0.clone()
    for gr in grads:
        a.G.copy_(gr)
        opt_e.step()
        ref.rmsprop_flat(w_ref, gr, v_ref, a.lr_mult_vector(), a.wd_vector(), 1e-3, clip=clip)
    torch.cuda.synchronize()
    torch.testing.assert_close(a.W, w_ref, rtol=1e-5, atol=1e-7)
    torch.testing.assert_close(opt_e.V, v_ref, rtol=1e-5, atol=1e-12)
    torch.testing.assert_close(a.H.float(), a.W, rtol=2 ** -8, atol=0)      # the bf16 shadow written in the same pass
    if clip:
        assert float(a.W.abs().max()) <= clip
    # the same 10 steps as replays of one captured step
    gbuf = torch.empty_like(b.G)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph, stream=s):
            b.G.copy_(gbuf)
            opt_g.step()
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    b.W.copy_(w0); opt_g.V.zero_()
    for gr in grads:
        gbuf.copy_(gr)
        graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(b.W, a.W) and torch.equal(opt_g.V, opt_e.V)


@pytest.mark.parametrize("kind,a", [("wgan", 1.0), ("wgan", -1.0), ("lsgan", 1.0), ("lsgan", 0.0)])
def test_gan_loss_matches_reference(mode, kind, a):
    ci = _ci()
    dt = precision.act_dtype()
    scores = torch.randn(64, 1, device=DEV).to(dt)
    loss, d = ci.gan_loss(scores, kind, a)
    loss_r, d_r = ref.gan_loss(scores.double(), kind, a)
    assert abs(float(loss) - float(loss_r)) < 1e-5 * max(1.0, abs(float(loss_r)))
    assert d.shape == scores.shape and rel_err(d, d_r) < TOL[mode]
    # through autograd: the device scalar's gradient is the kernel's d
    s = scores.detach().requires_grad_(True)
    fn.gan_loss(s, kind, a).backward()
    assert rel_err(s.grad, d_r) < TOL[mode]


def test_uniform_noise_matches_reference_and_advances(mode):
    ci = _ci()
    step = torch.full((1,), 5, dtype=torch.int64, device=DEV)
    u = ci.uniform_noise((64, 100), 1234, 3, step, dtype=torch.float32)
    want = ref.uniform_noise((64, 100), 1234, 3, 5, DEV)
    assert torch.equal(u, want)
    ub = ci.uniform_noise((64, 100), 1234, 3, step)
    assert ub.dtype == precision.act_dtype() and torch.equal(ub, want.to(ub.dtype))
    native.reset_launch_count()
    ci.L().advance_step(step.data_ptr(), ci._st(step))
    u2 = ci.uniform_noise((64, 100), 1234, 3, step, dtype=torch.float32)
    assert native.launch_count() == 2
    assert torch.equal(u2, ref.uniform_noise((64, 100), 1234, 3, 6, DEV)) and not torch.equal(u, u2)
