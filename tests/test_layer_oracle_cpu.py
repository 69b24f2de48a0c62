"""Keeps tests/layer_oracle.py honest without a GPU: every float64 reference against ``torch.nn.functional`` in float64, the top-k
tie rule on hand-built rows, the host twin of the dropout kernel's mask, and the two comparison helpers on synthetic errors."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import layer_oracle as lo
from theanompi_b200.ops import reference as ref

D = torch.float64


def _close(a, b, tol=1e-11):
    assert a.shape == b.shape, (a.shape, b.shape)
    assert float((a - b).abs().max()) <= tol * (1.0 + float(b.abs().max())), float((a - b).abs().max())


# --------------------------------------------------------------------------- batch norm
@pytest.mark.parametrize("act", [None, "relu", "leaky", "sigmoid"])
@pytest.mark.parametrize("with_res,with_drop", [(False, False), (True, False), (True, True)])
def test_bn_matches_torch_autograd(act, with_res, with_drop):
    if with_drop and act not in (None, "relu"):
        pytest.skip("drop-path takes ReLU or no activation")
    g = torch.Generator().manual_seed(1)
    N, H, W, C = 3, 5, 4, 8
    x = (torch.randn(N, H, W, C, generator=g, dtype=D) * 2 + 0.5).requires_grad_(True)
    res = torch.randn(N, H, W, C, generator=g, dtype=D).requires_grad_(True) if with_res else None
    gamma = (torch.rand(C, generator=g, dtype=D) + 0.5).requires_grad_(True)
    beta = torch.randn(C, generator=g, dtype=D).requires_grad_(True)
    drop = torch.tensor([0.0, 1.25, 1.25], dtype=D) if with_drop else None
    rm, rv = torch.randn(C, generator=g, dtype=D), torch.rand(C, generator=g, dtype=D) + 0.5
    rm_t, rv_t = rm.clone(), rv.clone()
    z = F.batch_norm(x.permute(0, 3, 1, 2), rm_t, rv_t, gamma, beta, True, 0.1, 1e-5).permute(0, 2, 3, 1)
    if with_drop:
        z = z * drop[:, None, None, None]
    if with_res:
        z = z + res
    y = {None: lambda t: t, "relu": torch.relu, "leaky": lambda t: F.leaky_relu(t, 0.2), "sigmoid": torch.sigmoid}[act](z)
    dy = torch.randn(N, H, W, C, generator=g, dtype=D)
    y.backward(dy)
    f = lo.bn_fwd64(x.detach(), gamma.detach(), beta.detach(), 1e-5, act, res.detach() if with_res else None, drop, run_mean=rm,
                    run_var=rv, momentum=0.1)
    _close(f["y"], y.detach())
    _close(f["run_mean"], rm_t)
    _close(f["run_var"], rv_t)
    X = x.detach().reshape(-1, C)
    _close(f["sum_x"], X.sum(0)); _close(f["sum_x2"], (X * X).sum(0)); _close(f["abs_x"], X.abs().sum(0))
    assert bool((f["s"] >= f["y"].abs() * (1 - 1e-12)).all()) or act == "sigmoid"
    b = lo.bn_bwd64(x.detach(), dy, y.detach(), gamma.detach(), f["mean"], f["rstd"], act, drop)
    _close(b["dx"], x.grad, 1e-9)
    _close(b["dgamma"], gamma.grad, 1e-9)
    _close(b["dbeta"], beta.grad, 1e-9)
    if with_res:
        _close(b["dres"], res.grad, 1e-9)
    assert bool((b["abs_dgamma"] >= b["dgamma"].abs() * (1 - 1e-12)).all()) and bool((b["s_dx"] >= b["dx"].abs() * (1 - 1e-9)).all())
    # eval mode: the running statistics
    e = lo.bn_fwd64(x.detach(), gamma.detach(), beta.detach(), 1e-5, None, training=False, run_mean=rm, run_var=rv)
    want = F.batch_norm(x.detach().permute(0, 3, 1, 2), rm.clone(), rv.clone(), gamma.detach(), beta.detach(), False, 0.1, 1e-5)
    _close(e["y"], want.permute(0, 2, 3, 1))


def test_bn_single_row_has_zero_variance_and_unit_unbias():
    x = torch.tensor([[1.0, -2.0, 3.0, 0.5]], dtype=D)
    f = lo.bn_fwd64(x, torch.ones(4, dtype=D), torch.zeros(4, dtype=D), run_mean=torch.zeros(4, dtype=D), run_var=torch.ones(4, dtype=D))
    assert torch.equal(f["var"], torch.zeros(4, dtype=D)) and torch.equal(f["y"], torch.zeros(1, 4, dtype=D))
    _close(f["run_var"], torch.full((4,), 0.9, dtype=D))


# --------------------------------------------------------------------------- pooling
POOLS = [("max", 3, 2, 1, 12, 10), ("max", 3, 2, 0, 13, 13), ("max", 2, 2, 0, 8, 6), ("max", 3, 1, 1, 7, 7), ("max", 5, 1, 0, 9, 8),
         ("max", 4, 1, 0, 7, 9), ("avg", 5, 3, 0, 14, 14), ("avg", 7, 1, 0, 7, 7), ("avg", 3, 2, 1, 8, 9), ("avg", 3, 1, 1, 6, 5)]


@pytest.mark.parametrize("mode,k,s,p,H,W", POOLS)
def test_pool_matches_torch(mode, k, s, p, H, W):
    g = torch.Generator().manual_seed(2)
    x = torch.randn(2, H, W, 4, generator=g, dtype=D).requires_grad_(True)        # tie-free
    xc = x.permute(0, 3, 1, 2)
    if mode == "max":
        yt, it = F.max_pool2d(xc, k, s, p, return_indices=True)
    else:
        yt = F.avg_pool2d(xc, k, s, p, count_include_pad=False)
    dy = torch.randn(yt.shape, generator=g, dtype=D)
    yt.backward(dy)
    y, arg, sc = lo.pool64(x.detach(), k, s, p, mode)
    assert tuple(y.shape[1:3]) == lo.pool_out_hw(H, W, k, s, p)
    _close(y, yt.detach().permute(0, 2, 3, 1))
    if mode == "max":
        # the window index decodes to torch's flat input index
        Ho, Wo = y.shape[1], y.shape[2]
        ho = torch.arange(Ho)[None, :, None, None]; wo = torch.arange(Wo)[None, None, :, None]
        flat = (ho * s - p + arg // k) * W + (wo * s - p + arg % k)
        assert torch.equal(flat, it.permute(0, 2, 3, 1))
    dx, sd = lo.pool_bwd64(dy.permute(0, 2, 3, 1), arg, tuple(x.shape), k, s, p, mode)
    _close(dx, x.grad)
    assert bool((sd >= dx.abs() * (1 - 1e-12)).all())


def test_max_pool_first_maximum_wins_and_padding_never_does():
    x = torch.zeros(1, 4, 4, 1, dtype=D)                       # every tap ties
    y, arg, _ = lo.pool64(x, 3, 2, 1, "max")
    # window (0, 0) starts at (-1, -1): its first in-image tap is (kh, kw) = (1, 1) → t = 4; window (1, 1) starts inside: t = 0
    assert arg[0, 0, 0, 0] == 4 and arg[0, 0, 1, 0] == 3 and arg[0, 1, 0, 0] == 1 and arg[0, 1, 1, 0] == 0
    dx, _ = lo.pool_bwd64(torch.ones(1, 2, 2, 1, dtype=D), arg, (1, 4, 4, 1), 3, 2, 1, "max")
    want = torch.zeros(4, 4, dtype=D)
    want[0, 0] = want[0, 1] = want[1, 0] = want[1, 1] = 1.0
    assert torch.equal(dx[0, :, :, 0], want)
    x = -torch.ones(1, 2, 2, 1, dtype=D) * 5                   # negative inputs: the padding (−inf) must not win
    assert torch.equal(lo.pool64(x, 3, 1, 1, "max")[0], x)


# --------------------------------------------------------------------------- LRN
@pytest.mark.parametrize("n", [3, 5, 7, 9])
@pytest.mark.parametrize("C", [8, 20])
def test_lrn_matches_torch(n, C):
    """torch divides α by the window size; the kernels (and the oracle) multiply the window SUM by α."""
    g = torch.Generator().manual_seed(3)
    x = (torch.randn(6, C, generator=g, dtype=D) * 20).requires_grad_(True)
    k, alpha, beta = 2.0, 1e-4, 0.75
    yt = F.local_response_norm(x[:, :, None], n, alpha * n, beta, k)[:, :, 0]
    dy = torch.randn(6, C, generator=g, dtype=D)
    yt.backward(dy)
    _close(lo.lrn64(x.detach(), n, k, alpha, beta), yt.detach())
    dx, s = lo.lrn_bwd64(x.detach(), dy, n, k, alpha, beta)
    _close(dx, x.grad)
    assert bool((s >= dx.abs() * (1 - 1e-12)).all())


# --------------------------------------------------------------------------- softmax
@pytest.mark.parametrize("B,C", [(1, 2), (16, 10), (8, 1003)])
@pytest.mark.parametrize("eps", [0.0, 0.1, 1.0])
def test_softmax_xent_matches_torch(B, C, eps):
    g = torch.Generator().manual_seed(4)
    z = (torch.randn(B, C, generator=g, dtype=D) * 3).requires_grad_(True)        # tie-free
    lab = torch.randint(0, C, (B,), generator=g)
    loss = F.cross_entropy(z, lab, label_smoothing=eps)
    loss.backward()
    o = lo.softmax_xent64(z.detach(), lab, eps, grad_scale=0.25)
    _close(o["loss"], loss.detach())
    _close(o["dlogits"], z.grad * 0.25)
    top = z.detach().topk(min(5, C), 1).indices
    assert float(o["err1"]) == float((top[:, 0] != lab).double().mean())
    assert float(o["err5"]) == float(1.0 - (top == lab[:, None]).any(1).double().mean())
    assert float(o["abs_loss"]) >= abs(float(o["loss"]))


def test_top_k_tie_rule():
    """Among equal logits the lower class index ranks first, so a label tied with m lower-indexed classes has rank ≥ m."""
    z = torch.tensor([[1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0],      # label 0: rank 0
                      [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0],      # label 4: rank 4 (in the top 5)
                      [1.0, 1.0, 1.0, 1.0, 1.0, 1.0, 0.0],      # label 5: rank 5 (out of it)
                      [2.0, 1.0, 1.0, 3.0, 1.0, 1.0, 0.0],      # label 2: two greater + one equal before it = 3
                      [0.0, 0.0, 0.0, 0.0, 0.0, 0.0, 0.0]], dtype=D)
    lab = torch.tensor([0, 4, 5, 2, 6])
    assert lo.label_rank(z, lab).tolist() == [0, 4, 5, 3, 6]
    o = lo.softmax_xent64(z, lab)
    assert float(o["err1"]) == 4 / 5 and float(o["err5"]) == 2 / 5


# --------------------------------------------------------------------------- dropout mask
@pytest.mark.parametrize("p", [0.0, 1 / 65536, 0.1, 0.5, 0.9, 1 - 1 / 65536])
def test_dropout_mask_philox_keep_rate(p):
    n = 1 << 20
    m = ref.dropout_mask_philox(n, p, 0x5EED, 3, 7)
    assert m.dtype == torch.bool and m.shape == (n,)
    keep = 1.0 - math.floor(float(np.float32(p)) * 65536) / 65536
    got = float(m.double().mean())
    assert abs(got - keep) <= 4.5 * math.sqrt(max(keep * (1 - keep), 1e-12) / n) + 1e-12, (got, keep)
    if p == 0.0:
        assert bool(m.all())


def test_dropout_mask_philox_streams_are_independent():
    n = 1 << 16
    base = ref.dropout_mask_philox(n, 0.5, 0x5EED, 3, 7)
    assert torch.equal(base, ref.dropout_mask_philox(n, 0.5, 0x5EED, 3, 7))
    assert torch.equal(base[:4096], ref.dropout_mask_philox(4096, 0.5, 0x5EED, 3, 7))          # a prefix: the counter is the group index
    for other in (ref.dropout_mask_philox(n, 0.5, 0x5EED, 4, 7), ref.dropout_mask_philox(n, 0.5, 0x5EED, 3, 8),
                  ref.dropout_mask_philox(n, 0.5, 0x5EEE, 3, 7), ref.dropout_mask_philox(n, 0.5, 0x5EED + (1 << 32), 3, 7)):
        agree = float((other == base).double().mean())
        assert abs(agree - 0.5) < 4.5 * 0.5 / math.sqrt(n), agree
    # a lower threshold keeps a superset: the same 16-bit draws are compared
    assert bool((ref.dropout_mask_philox(n, 0.1, 0x5EED, 3, 7) | ~base).all())
    with pytest.raises(ValueError):
        ref.dropout_mask_philox(12, 0.5, 1, 0, 0)


def test_philox_known_answer():
    """Philox4x32-10 test vectors of the Random123 distribution (counter and key all zero / all ones)."""
    r = ref._philox4x32(([0], [0], [0], [0]), 0, 0)
    assert [int(v[0]) for v in r] == [0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8]
    f = 0xFFFFFFFF
    r = ref._philox4x32(([f], [f], [f], [f]), f, f)
    assert [int(v[0]) for v in r] == [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD]


# --------------------------------------------------------------------------- the comparison helpers
def test_elementwise_bound_sees_one_wrong_element_the_old_metric_does_not():
    g = torch.Generator().manual_seed(5)
    want = torch.randn(1000, 1000, generator=g, dtype=D)
    got = want.to(torch.bfloat16)
    lo.assert_elementwise(got, want, torch.bfloat16)             # one bf16 rounding passes
    bad = got.clone().float()
    i = int(want.abs().reshape(-1).argmin())                     # a small-magnitude element
    bad.view(-1)[i] += 0.009 * float(want.abs().max())           # wrong by just under 1 % of the largest element
    assert lo.old_rel_err(bad, want) < 1e-2                      # the metric of test_gpu_kernels.py passes it
    with pytest.raises(AssertionError, match="1 of 1000000 elements"):
        lo.assert_elementwise(bad, want, torch.bfloat16)
    nan = got.clone(); nan[3, 4] = float("nan")
    with pytest.raises(AssertionError):
        lo.assert_elementwise(nan, want, torch.bfloat16)


def test_elementwise_bound_allows_cancellation_only_with_its_scale():
    a = torch.tensor([[1000.0, 3.0]], dtype=D)
    b = torch.tensor([[-999.0, 4.0]], dtype=D)
    got = (a + b).float() + torch.tensor([[2.0, 0.0]])           # 1000 − 999 computed from bf16-rounded terms can be off by ~2
    with pytest.raises(AssertionError, match=r"r=0, c=0"):
        lo.assert_elementwise(got, a + b, torch.bfloat16)
    lo.assert_elementwise(got, a + b, torch.bfloat16, s=a.abs() + b.abs())
    with pytest.raises(AssertionError):                          # the scale of one element does not excuse another
        lo.assert_elementwise((a + b).float() + torch.tensor([[0.0, 2.0]]), a + b, torch.bfloat16, s=a.abs() + b.abs())


def test_failure_message_names_row_and_channel_vector():
    want = torch.zeros(2, 3, 4, 16, dtype=D)
    got = want.clone().float()
    got[1, 2, 3, 9] = 1.0
    with pytest.raises(AssertionError, match=r"n=1, h=2, w=3, c=9\): row 23 of 24, channel vector 1 of 2"):
        lo.assert_elementwise(got, want, torch.bfloat16)
    with pytest.raises(AssertionError, match=r"channel vector 2 of 4"):
        lo.assert_elementwise(got, want, torch.float32)


def test_reduction_bound():
    g = torch.Generator().manual_seed(6)
    n = 100000
    t = torch.randn(n, 8, generator=g, dtype=D)
    want, abs_sum = t.sum(0), t.abs().sum(0)
    lo.assert_reduction(t.float().sum(0), want, abs_sum, n)
    seq = torch.zeros(8)
    for chunk in t.float().split(1, 0)[:2000]:                   # a plain sequential fp32 sum of a prefix stays inside too
        seq = seq + chunk[0]
    lo.assert_reduction(seq, t[:2000].sum(0), t[:2000].abs().sum(0), 2000)
    off = t.float().sum(0)
    off[5] -= 10.0                                               # 10 in a sum of 100,000 terms with Σ|t| ≈ 80,000 (the bound is ≈ 6)
    with pytest.raises(AssertionError, match="worst at index 5"):
        lo.assert_reduction(off, want, abs_sum, n)
