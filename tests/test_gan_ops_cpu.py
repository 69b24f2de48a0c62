"""CPU checks of the GAN building blocks: the reference transposed convolution with leaky-ReLU / sigmoid activations, the flat
RMSProp, the GAN losses and the Philox noise (no GPU needed)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from theanompi_b200 import ops
from theanompi_b200.ops import reference as ref
from theanompi_b200.parallel.arena import FlatArena
from theanompi_b200.utils.opt import FlatRMSProp

TORCH_ACT = {"none": lambda t: t, "relu": torch.relu, "sigmoid": torch.sigmoid,
             "leaky": lambda t: F.leaky_relu(t, ref.LEAKY_SLOPE)}


# (Cin, Cout, Hi, K, stride, pad, output_padding): the DCGAN 5x5/2 p2 op1 layer, a 4x4/2 p1 and a 3x3/1 layer
@pytest.mark.parametrize("Cin,Cout,Hi,K,s,p,op", [(16, 8, 7, 5, 2, 2, 1), (8, 12, 5, 4, 2, 1, 0), (6, 10, 6, 3, 1, 1, 0)])
@pytest.mark.parametrize("act", ["none", "relu", "sigmoid", "leaky"])
def test_reference_conv_transpose_matches_torch_autograd(Cin, Cout, Hi, K, s, p, op, act):
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, Hi, Hi + 1, Cin, generator=g, dtype=torch.float64)
    w = torch.randn(Cin, K, K, Cout, generator=g, dtype=torch.float64) * 0.3     # [Cin, KH, KW, Cout]
    b = torch.randn(Cout, generator=g, dtype=torch.float64)
    xt, wt, bt = (t.clone().requires_grad_(True) for t in (x, w, b))
    want = TORCH_ACT[act](F.conv_transpose2d(xt.permute(0, 3, 1, 2), wt.permute(0, 3, 1, 2), bt, stride=s, padding=p,
                                             output_padding=op)).permute(0, 2, 3, 1)
    y = ref.conv_transpose2d_bias_act(x, w, b, s, p, op, act)
    assert y.shape == want.shape
    torch.testing.assert_close(y, want.detach(), rtol=1e-10, atol=1e-10)
    dy = torch.randn(want.shape, generator=g, dtype=torch.float64)
    want.backward(dy)
    dx, dw, db = ref.conv_transpose2d_bias_act_bwd(x, w, y, dy, s, p, act)
    torch.testing.assert_close(dx, xt.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(dw, wt.grad, rtol=1e-10, atol=1e-10)
    torch.testing.assert_close(db, bt.grad, rtol=1e-10, atol=1e-10)


def test_functional_conv_transpose_autograd_and_padded_channels():
    """The autograd op on the CPU path: padded output channels (c_real) are zero and their weight columns get zero gradient
    when the next layer ignores them."""
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 7, 7, 16, generator=g, requires_grad=True)
    w = torch.zeros(16, 5, 5, 8)
    w[..., :1] = torch.randn(16, 5, 5, 1, generator=g) * 0.1
    w.requires_grad_(True)
    b = torch.zeros(8, requires_grad=True)
    y = ops.functional.conv_transpose2d_bias_act(x, w, b, 2, 2, 1, "sigmoid", c_real=1)
    assert y.shape == (2, 14, 14, 8)
    assert torch.all(y[..., 1:] == 0)
    (y[..., :1] ** 2).sum().backward()
    assert torch.all(w.grad[..., 1:] == 0) and torch.all(b.grad[1:] == 0)
    assert w.grad[..., :1].abs().sum() > 0 and x.grad.abs().sum() > 0


@pytest.mark.parametrize("act", ["leaky", "sigmoid"])
def test_reference_activations_in_linear_and_batch_norm(act):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(16, 24, generator=g, dtype=torch.float64, requires_grad=True)
    w = torch.randn(8, 24, generator=g, dtype=torch.float64, requires_grad=True)
    b = torch.randn(8, generator=g, dtype=torch.float64, requires_grad=True)
    want = TORCH_ACT[act](F.linear(x, w, b))
    y = ref.linear_bias_act(x.detach(), w.detach(), b.detach(), act)
    torch.testing.assert_close(y, want.detach())
    dy = torch.randn(16, 8, generator=g, dtype=torch.float64)
    want.backward(dy)
    dx, dw, db = ref.linear_bias_act_bwd(x.detach(), w.detach(), y, dy, act)
    torch.testing.assert_close(dx, x.grad); torch.testing.assert_close(dw, w.grad); torch.testing.assert_close(db, b.grad)

    z = torch.randn(4, 5, 5, 8, generator=g, dtype=torch.float64, requires_grad=True)
    gamma = torch.rand(8, generator=g, dtype=torch.float64) + 0.5
    beta = torch.randn(8, generator=g, dtype=torch.float64)
    gt, bt = gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    want = TORCH_ACT[act](F.batch_norm(z.permute(0, 3, 1, 2), None, None, gt, bt, True, 0.1, 1e-5)).permute(0, 2, 3, 1)
    yb, mean, rstd = ref.batch_norm_fwd(z.detach(), gamma, beta, None, None, True, 0.1, 1e-5, act)
    tol = dict(rtol=1e-5, atol=1e-5)                       # the reference batch norm computes in fp32
    torch.testing.assert_close(yb.double(), want.detach(), **tol)
    dy = torch.randn(want.shape, generator=g, dtype=torch.float64)
    want.backward(dy)
    dz, _, dg, dbeta = ref.batch_norm_bwd(z.detach(), dy, yb, gamma, mean, rstd, act, False)
    for got, exp in ((dz, z.grad), (dg, gt.grad), (dbeta, bt.grad)):
        torch.testing.assert_close(got.double(), exp, **tol)


def _arena(seed):
    g = torch.Generator().manual_seed(seed)
    ps = [torch.randn(64, 3, 5, 5, generator=g) * 0.05, torch.randn(64, generator=g) * 0.05, torch.randn(10, 1500, generator=g) * 0.05,
          torch.randn(10, generator=g) * 0.05]
    return ps, FlatArena([p.clone() for p in ps], device="cpu", bias_lr_mult=1.0)


@pytest.mark.parametrize("clip", [0.0, 0.01])
def test_reference_rmsprop_matches_torch_rmsprop(clip):
    """FlatRMSProp (CPU path = ops.reference.rmsprop_flat) over a multi-tensor arena vs torch.optim.RMSprop(alpha=0.99,
    eps=1e-8), clamping after each step when clip > 0 (WGAN.critic_clip_fn)."""
    ps, arena = _arena(3)
    tp = [torch.nn.Parameter(p.clone()) for p in ps]
    topt = torch.optim.RMSprop(tp, lr=5e-3, alpha=0.99, eps=1e-8)
    arena.hyper[0] = 5e-3
    opt = FlatRMSProp(arena, clip=clip)
    g = torch.Generator().manual_seed(4)
    for _ in range(5):
        grads = [torch.randn(p.shape, generator=g) for p in ps]
        for p, gr in zip(tp, grads):
            p.grad = gr.clone()
        topt.step()
        if clip:
            with torch.no_grad():
                for p in tp:
                    p.clamp_(-clip, clip)
        for v, gr in zip(arena.views("G"), grads):
            v.copy_(gr)
        opt.step()
    for v, p in zip(arena.views("W"), tp):
        torch.testing.assert_close(v, p.detach(), rtol=1e-5, atol=1e-7)
    sd = opt.state_dict()
    opt2 = FlatRMSProp(_arena(3)[1])
    opt2.load_state_dict(sd)
    assert torch.equal(opt2.V, opt.V)


@pytest.mark.parametrize("kind,a", [("wgan", 1.0), ("wgan", -1.0), ("lsgan", 1.0), ("lsgan", 0.0)])
def test_reference_gan_loss(kind, a):
    o = torch.randn(64, 1, dtype=torch.float64, requires_grad=True)
    want = a * o.mean() if kind == "wgan" else 0.5 * ((o - a) ** 2).mean()
    want.backward()
    loss, d = ref.gan_loss(o.detach(), kind, a)
    torch.testing.assert_close(loss.double(), want.detach())
    torch.testing.assert_close(d.double(), o.grad)


def test_reference_noise_is_philox():
    # Philox4x32-10 known-answer vector (Salmon et al., Random123): counter 0, key 0
    r = ref._philox4x32((np.zeros(1, np.uint64),) * 4, 0, 0)
    assert [int(v[0]) for v in r] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    u = ref.uniform_noise((64, 100), seed=7, stream=1, step=0)
    assert u.shape == (64, 100) and u.dtype == torch.float32
    assert float(u.min()) >= 0.0 and float(u.max()) < 1.0 and abs(float(u.mean()) - 0.5) < 0.02
    assert not torch.equal(u, ref.uniform_noise((64, 100), seed=7, stream=1, step=1))
    assert not torch.equal(u, ref.uniform_noise((64, 100), seed=7, stream=2, step=0))
    assert torch.equal(u, ref.uniform_noise((64, 100), seed=7, stream=1, step=0))
