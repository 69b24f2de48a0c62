"""Implicit-GEMM convolutions at the tile widths sized to the channel counts (96- and 192-wide n-tiles, 256-row 96-wide
tiles, k-steps trimmed to a partial channel chunk, warpgroups with no rows below M), bf16 and tf32, against an fp64 PyTorch
reference.  test_conv_tile_plan_cpu.py checks that these shapes reach each of those tiles."""
import pytest
import torch

from theanompi_b200 import ops
from theanompi_b200.ops import precision

pytestmark = pytest.mark.gpu
DEV = "cuda"
TOL = {"bf16": (1e-2, 2e-2), "tf32": (1e-3, 1e-3)}           # (output, gradients)


def rel_err(a, b):
    a, b = a.float(), b.float()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


@pytest.mark.parametrize("prec", ["bf16", "tf32"])
@pytest.mark.parametrize("cfg", [
    dict(N=8, H=227, C=3, O=96, k=11, s=4, p=0, g=1),       # AlexNet conv1 (space-to-depth, Cp = 48): 256-row x 96 fprop
    dict(N=24, H=227, C=3, O=96, k=11, s=4, p=0, g=1),      # the same at batch 24: 128-row x 96 fprop, 192-wide wgrad
    dict(N=48, H=13, C=384, O=384, k=3, s=1, p=1, g=2),     # AlexNet conv4: 192-wide fprop / dgrad, wgrad M = 192
    dict(N=48, H=13, C=384, O=256, k=3, s=1, p=1, g=2),     # AlexNet conv5: 192-wide dgrad
])
def test_conv_channel_sized_tiles(cfg, prec):
    old = precision.precision()
    precision.set_precision(prec)
    try:
        _check(cfg, prec)
    finally:
        precision.set_precision(old)


def _check(cfg, prec):
    torch.manual_seed(6)
    N, H, C, O, k, s, p, g = (cfg[n] for n in ("N", "H", "C", "O", "k", "s", "p", "g"))
    dt = torch.bfloat16 if prec == "bf16" else torch.float32
    first = C < 4
    x = torch.randn(N, H, H, C, device=DEV).to(dt).requires_grad_(not first)
    if g == 1:
        w = (torch.randn(O, k, k, C, device=DEV) * 0.1).to(dt).requires_grad_(True)
        b = torch.randn(O, device=DEV).requires_grad_(True)
        y = ops.conv2d_bias_act(x, w, b, s, p, 1, True)
        ws, bs = [w], [b]
    else:
        ws = [(torch.randn(O // 2, k, k, C // 2, device=DEV) * 0.1).to(dt).requires_grad_(True) for _ in range(2)]
        bs = [torch.randn(O // 2, device=DEV).requires_grad_(True) for _ in range(2)]
        y = ops.conv2d_group2_bias_act(x, ws[0], bs[0], ws[1], bs[1], s, p, True)
    dy = torch.randn_like(y)
    y.backward(dy)
    # fp64 reference (NCHW) on the same rounded inputs, ReLU through our own output's mask (an activation next to zero may
    # flip between the two, which would change a whole gradient row)
    xr = x.detach().double().permute(0, 3, 1, 2).clone().requires_grad_(not first)
    wr = torch.cat([t.detach().double().permute(0, 3, 1, 2) for t in ws], 0).clone().requires_grad_(True)
    br = torch.cat([t.detach().double() for t in bs], 0).clone().requires_grad_(True)
    lin = torch.nn.functional.conv2d(xr, wr, br, s, p, groups=g)
    tol_y, tol_g = TOL[prec]
    assert y.dtype == dt
    assert rel_err(y, torch.relu(lin).permute(0, 2, 3, 1)) < tol_y
    (lin * (y.detach().permute(0, 3, 1, 2) > 0)).backward(dy.double().permute(0, 3, 1, 2))
    if not first:
        assert rel_err(x.grad, xr.grad.permute(0, 2, 3, 1)) < tol_g
    assert rel_err(torch.cat([t.grad for t in ws], 0), wr.grad.permute(0, 2, 3, 1)) < tol_g
    assert rel_err(torch.cat([t.grad for t in bs]), br.grad) < tol_g
