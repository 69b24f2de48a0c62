"""Tile choice of the implicit-GEMM convolution launcher (host code of the native extension, no GPU needed): the (BN, MT)
each AlexNet-128b convolution GEMM gets on an H100 SXM (132 SMs), and the plans of the shapes ``test_gpu_conv_tiles.py``
runs, so that the GPU suite is known to reach every tile width in bf16 and in tf32."""
import pytest

SMS = 132                                                    # H100 SXM
FPROP, DGRAD, WGRAD = 0, 1, 2


def _lib():
    from theanompi_b200.ops import native
    L = native.lib()
    if L is None:
        pytest.skip("native extension not built")
    return L


def _plan(kind, M, N, groups, num_kb, tall_ok):
    bn, mt, splits = _lib().gemm_plan_conv(kind, M, N, groups, num_kb, tall_ok, SMS)
    return bn, mt, splits


def _fd(kind, batch, hw, cin, cout, taps, groups, f32=False):
    """fprop / dgrad of a convolution with `cin` input channels per group (the GEMM's K) and `cout` outputs per group."""
    bk = 32 if f32 else 64
    return _plan(kind, batch * hw * hw, cout, groups, taps * -(-cin // bk), 0 if (f32 and kind == DGRAD) else 1)[:2]


def _wg(batch, hw, cin, cout, taps, groups, f32=False):
    bk = 32 if f32 else 64
    bn, mt, _ = _plan(WGRAD, cout, taps * -(-cin // bk) * bk, groups, -(-batch * hw * hw // bk), 0)
    return bn, mt


def test_alexnet_conv_tiles():
    B = 128
    # conv1 (space-to-depth: 55x55 outputs, 3x3 taps, 48 channels): 96 columns instead of 128, 256-row tiles
    assert _fd(FPROP, B, 55, 48, 96, 9, 1) == (96, 2)
    # conv4 fprop / dgrad and conv5 dgrad (192 output channels per group): one 192-wide n-tile instead of 128 + half-empty 128
    assert _fd(FPROP, B, 13, 192, 192, 9, 2) == (192, 1)
    assert _fd(DGRAD, B, 13, 192, 192, 9, 2) == (192, 1)
    assert _fd(DGRAD, B, 13, 128, 192, 9, 2) == (192, 1)
    # unchanged: conv2 / conv3 fprop (256-row, 128 wide), conv3 dgrad (128-row, 128 wide), conv2 dgrad (48 outputs), conv5 fprop
    assert _fd(FPROP, B, 27, 48, 128, 25, 2) == (128, 2)
    assert _fd(FPROP, B, 13, 256, 384, 9, 1) == (128, 2)
    assert _fd(DGRAD, B, 13, 384, 256, 9, 1) == (128, 1)
    assert _fd(DGRAD, B, 27, 128, 48, 25, 2) == (64, 2)
    assert _fd(FPROP, B, 13, 192, 128, 9, 2) == (128, 1)
    # wgrad: 3-box tiles for the deep reductions of conv1 (9 boxes: 3 tiles instead of 5 with an empty box) and conv2 (25
    # boxes); the shallower conv3-5 wgrads (338 pixel blocks) keep 2-box tiles
    assert _wg(B, 55, 48, 96, 9, 1) == (192, 1)
    assert _wg(B, 27, 48, 128, 25, 2) == (192, 1)
    assert _wg(B, 13, 192, 192, 9, 2) == (128, 1)
    assert _wg(B, 13, 192, 128, 9, 2) == (128, 1)


def test_tile_legality():
    for M in (512, 12100, 20000, 400000):
        # dgrad reads MN-major weights in 64-wide atoms: never 96 columns
        assert _plan(DGRAD, M, 96, 1, 9, 1)[0] in (64, 128, 192)
        for kind in (FPROP, DGRAD):
            bn, mt, splits = _plan(kind, M, 192, 1, 27, 1)
            assert not (bn == 192 and mt == 2) and splits == 1       # 192-wide tiles are 128 rows only; no split-K
    # wgrad: 128-row tiles, 128 or 192 wide
    for N in (576, 1728, 2304):
        bn, mt, _ = _plan(WGRAD, 192, N, 2, 338, 0)
        assert bn in (128, 192) and mt == 1
    # narrow outputs keep 64-wide tiles
    assert _fd(FPROP, 32, 27, 48, 48, 25, 1)[0] == 64
    # no 256-row tiles for fp32-output dgrad (the tf32 transpose path is 128-row only)
    assert _plan(DGRAD, 400000, 128, 1, 36, 0)[1] == 1


@pytest.mark.parametrize("f32", [False, True])
def test_gpu_suite_shapes_reach_every_tile(f32):
    """The shapes of test_gpu_conv_tiles.py cover BN 96 (128- and 256-row) and BN 192 fprop, dgrad and wgrad."""
    # conv1 through space-to-depth: 227x227 RGB, 11x11 / 4 → 55x55 outputs over a 57x57x48 image, 3x3 taps
    assert _fd(FPROP, 8, 55, 48, 96, 9, 1, f32) == (96, 2)
    assert _fd(FPROP, 24, 55, 48, 96, 9, 1, f32) == (96, 1)
    assert _wg(24, 55, 48, 96, 9, 1, f32) == (192, 1)      # 1135 (bf16) / 2269 (tf32) pixel blocks: 3-box / 6-box tiles
    # conv4 / conv5 (two groups, 192 input channels each) at batch 48
    assert _fd(FPROP, 48, 13, 192, 192, 9, 2, f32) == (192, 1)
    assert _fd(DGRAD, 48, 13, 192, 192, 9, 2, f32) == (192, 1)
    assert _fd(DGRAD, 48, 13, 128, 192, 9, 2, f32) == (192, 1)
    assert _wg(48, 13, 192, 192, 9, 2, f32) == (128, 1)     # M = 192: the second m-tile's upper warpgroup has no rows
