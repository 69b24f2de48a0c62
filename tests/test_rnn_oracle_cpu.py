"""The float64 references of tests/rnn_oracle.py checked without a GPU: the masked recurrence against ``torch.nn.LSTM``, the
hand-written backward against autograd, the fp32 CPU branch of ``ops/rnn.py`` against the references within fp32 bounds, the
embedding and masked-mean references against direct sums, and every allowance against a result moved by twice it."""
import numpy as np
import pytest
import torch
from torch.nn.utils.rnn import pack_padded_sequence, pad_packed_sequence

import gemm_oracle as go
import layer_oracle as lo
import rnn_oracle as ro
from theanompi_b200.ops import rnn

F64 = torch.float64


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _torch_lstm(gx, U):
    """``torch.nn.LSTM`` (gate order i, f, g, o) set up to run this project's recurrence: identity input weight so its input is
    gx with the gates permuted from i | f | o | c̃, U's rows permuted the same way, zero biases."""
    T, B, H4 = gx.shape
    H = H4 // 4
    perm = torch.cat([torch.arange(0, 2 * H), torch.arange(3 * H, 4 * H), torch.arange(2 * H, 3 * H)])
    m = torch.nn.LSTM(H4, H).double()
    with torch.no_grad():
        m.weight_ih_l0.copy_(torch.eye(H4, dtype=F64)[perm])
        m.weight_hh_l0.copy_(U.double()[perm])
        m.bias_ih_l0.zero_()
        m.bias_hh_l0.zero_()
    return m


@pytest.mark.parametrize("T,B,H", [(7, 3, 5), (20, 4, 16)])
def test_oracle_matches_torch_lstm_all_valid(T, B, H):
    g = _gen(T)
    gx = torch.randn(T, B, 4 * H, generator=g, dtype=F64) * 2
    U = torch.randn(4 * H, H, generator=g, dtype=F64) / H ** 0.5
    r = ro.lstm_seq64(gx, U, torch.ones(T, B, dtype=F64))
    with torch.no_grad():
        h, (hn, cn) = _torch_lstm(gx, U)(gx)
    torch.testing.assert_close(r["hs"][1:], h, rtol=1e-12, atol=1e-13)
    torch.testing.assert_close(r["cs"][-1], cn[0], rtol=1e-12, atol=1e-13)


def test_oracle_matches_torch_lstm_packed_prefixes():
    T, B, H = 9, 5, 6
    g = _gen(3)
    gx = torch.randn(T, B, 4 * H, generator=g, dtype=F64) * 2
    U = torch.randn(4 * H, H, generator=g, dtype=F64) / H ** 0.5
    lengths = torch.tensor([9, 1, 4, 7, 2])
    mask = (torch.arange(T)[:, None] < lengths[None, :]).double()
    r = ro.lstm_seq64(gx, U, mask)
    with torch.no_grad():
        out, _ = _torch_lstm(gx, U)(pack_padded_sequence(gx, lengths, enforce_sorted=False))
    h, _ = pad_packed_sequence(out, total_length=T)
    for b, n in enumerate(lengths.tolist()):
        torch.testing.assert_close(r["hs"][1:n + 1, b], h[:n, b], rtol=1e-12, atol=1e-13)
        # padded steps carry the last valid state, exactly
        assert torch.equal(r["hs"][n + 1:, b], r["hs"][n, b].expand(T - n, H))
        assert torch.equal(r["cs"][n + 1:, b], r["cs"][n, b].expand(T - n, H))


def test_backward_matches_autograd():
    T, B, H = 5, 3, 4
    g = _gen(11)
    gx = (torch.randn(T, B, 4 * H, generator=g, dtype=F64) * 2).requires_grad_(True)
    U = (torch.randn(4 * H, H, generator=g, dtype=F64) / H ** 0.5).requires_grad_(True)
    mask = (torch.rand(T, B, generator=g) < 0.7).double()
    mask[:, 0] = 1
    mask[1:, 1] = 0                                   # a length-1 row
    mask[2, 2] = 0                                    # a hole
    dh_all = torch.randn(T, B, H, generator=g, dtype=F64)
    r = ro.lstm_seq64(gx, U, mask)
    dgx, dU = torch.autograd.grad((r["hs"][1:] * dh_all).sum(), (gx, U))
    b = ro.lstm_seq64(gx.detach(), U.detach(), mask, dh_all)
    torch.testing.assert_close(b["dG"], dgx, rtol=1e-10, atol=1e-12)
    torch.testing.assert_close(b["dU"], dU, rtol=1e-10, atol=1e-12)
    # and the forward itself against torch.autograd.gradcheck of the same function
    assert torch.autograd.gradcheck(lambda a, u: ro.lstm_seq64(a, u, mask)["hs"], (gx.detach().requires_grad_(True),
                                                                                   U.detach().requires_grad_(True)))


def _cpu_branch(T, B, H, seed):
    g = _gen(seed)
    gx = (torch.randn(T, B, 4 * H, generator=g) * 2).requires_grad_(True)
    U = (torch.randn(4 * H, H, generator=g) / H ** 0.5).requires_grad_(True)
    lengths = torch.randint(1, T + 1, (B,), generator=g)
    lengths[0], lengths[-1] = 1, T
    mask = (torch.arange(T)[:, None] < lengths[None, :]).float()
    h = rnn.lstm_sequence(gx, U, mask)
    hs, cs, act, _ = [t.clone() for t in h.grad_fn.saved_tensors]
    dh_all = torch.randn(T, B, H, generator=g)
    h.backward(dh_all)
    return dict(gx=gx.detach(), U=U.detach(), mask=mask, hs=hs, cs=cs, act=act, dh_all=dh_all, dgx=gx.grad, dU=U.grad)


def test_oracle_matches_fp32_cpu_branch():
    """Forward step by step from the branch's own state (fp32 matmul bound + cell bound), then the backward against the float64
    backward from the same forward states, within n·2⁻²⁴ of its magnitude twin (n: the fp32 roundings of T steps)."""
    T, B, H = 12, 6, 16
    r = _cpu_branch(T, B, H, 5)
    for t in range(T):
        hp = r["hs"][t].double()
        gh, s = hp @ r["U"].double().t(), hp.abs() @ r["U"].double().abs().t()
        c = ro.lstm_cell_fwd64(r["gx"][t], gh, r["cs"][t], r["hs"][t], r["mask"][t], dgh=go.gemm_gamma(H) * s)
        lo.assert_elementwise(r["act"][t], c["act"], torch.float32, extra_abs=c["tol_act"], what="act[%d]" % t)
        lo.assert_elementwise(r["cs"][t + 1], c["c"], torch.float32, extra_abs=c["tol_c"], what="c[%d]" % t)
        lo.assert_elementwise(r["hs"][t + 1], c["h"], torch.float32, extra_abs=c["tol_h"], what="h[%d]" % t)
    b = ro.lstm_seq_bwd64(r["act"], r["cs"], r["hs"], r["U"], r["mask"], r["dh_all"])
    a = r["act"].double().clone()
    a[..., 3 * H:] = a[..., 3 * H:].abs()
    s = ro.lstm_seq_bwd64(a, r["cs"].abs(), r["hs"].abs(), r["U"].abs(), r["mask"], r["dh_all"].abs())
    n = T * (4 * H + 12)
    lo.assert_elementwise(r["dgx"], b["dG"], torch.float32, extra_abs=n * ro.U24 * s["dG"], what="gx.grad")
    lo.assert_elementwise(r["dU"], b["dU"], torch.float32, extra_abs=(n + T * B) * ro.U24 * s["dU"], what="dU")


def test_embedding_oracles():
    g = _gen(7)
    V, D = 50, 12
    ids = torch.randint(0, V, (9, 4), generator=g)
    ids[0, 0], ids[0, 1] = 0, V - 1
    W = torch.randn(V, D, generator=g)
    e = ro.embedding64(ids, W)
    assert e.shape == (9, 4, D) and torch.equal(e, W.double()[ids])
    dout = torch.randn(9, 4, D, generator=g, dtype=F64)
    dW, s, cnt = ro.embedding_bwd64(ids, dout, V)
    want = np.zeros((V, D))
    np.add.at(want, ids.reshape(-1).numpy(), dout.reshape(-1, D).numpy())
    np.testing.assert_allclose(dW.numpy(), want, rtol=1e-13, atol=1e-13)
    assert torch.equal(cnt, torch.bincount(ids.reshape(-1), minlength=V))
    assert bool((s >= dW.abs()).all()) and int(cnt.sum()) == ids.numel()


def test_masked_mean_oracles():
    g = _gen(9)
    T, B, H = 6, 4, 5
    h = torch.randn(T, B, H, generator=g, dtype=F64)
    mask = torch.tensor([[1, 1, 0, 1], [1, 0, 0, 1], [1, 0, 0, 0], [0, 0, 0, 1], [1, 0, 0, 1], [1, 0, 0, 1]], dtype=F64)
    out, s, cnt = ro.masked_mean64(h, mask)
    for b in range(B):
        n = int(mask[:, b].sum())
        want = sum(h[t, b] for t in range(T) if mask[t, b]) / max(n, 1) if n else torch.zeros(H, dtype=F64)
        torch.testing.assert_close(out[b], want, rtol=1e-14, atol=1e-15)
    assert torch.equal(out[2], torch.zeros(H, dtype=F64)) and float(cnt[2]) == 0
    dout = torch.randn(B, H, generator=g, dtype=F64)
    dh, tol = ro.masked_mean_bwd64(dout, mask)
    hh = h.clone().requires_grad_(True)
    (ro.masked_mean64(hh, mask)[0] * dout).sum().backward()
    torch.testing.assert_close(dh, hh.grad, rtol=1e-14, atol=1e-15)
    assert torch.equal(dh[:, 2], torch.zeros(T, H, dtype=F64))


def test_fast_math_terms():
    x = torch.tensor([0.0, 1.0, -10.0, 40.0], dtype=F64)
    assert torch.equal(ro.expf_rel(x), torch.tensor([2.0, 3.0, 13.0, 48.0], dtype=F64) * 2.0 ** -23)
    assert ro.RCP_REL == 2.0 ** -23 and ro.DIV_REL == 2.0 ** -22 and 2.0 ** -11 < ro.TANH_REL < 2.0 ** -10.9
    # σ's allowance: the exponential's share vanishes as σ → 1
    assert float(ro.sigm_rel(torch.tensor([40.0], dtype=F64))) < 2.0 ** -21
    assert float(ro.sigm_rel(torch.tensor([-40.0], dtype=F64))) > 48 * 2.0 ** -23


def _moved_fails(got, want, dtype, tol, what):
    """``got`` shifted by twice its bound (u_store·|want| + tol) in the direction away from ``want`` must be rejected."""
    bound = lo.U_STORE[dtype] * want.abs() + tol
    moved = want + 2 * bound * torch.where(got.double() >= want, 1.0, -1.0)
    with pytest.raises(AssertionError):
        lo.assert_elementwise(moved, want, dtype, extra_abs=tol, what=what)


def test_every_bound_rejects_twice_its_size():
    g = _gen(13)
    B, H = 4, 8
    gx = torch.randn(B, 4 * H, generator=g, dtype=F64) * 3
    gh = torch.randn(B, 4 * H, generator=g, dtype=F64)
    cp, hp = torch.randn(B, H, generator=g, dtype=F64), torch.randn(B, H, generator=g, dtype=F64)
    m = torch.tensor([1.0, 1.0, 0.0, 1.0], dtype=F64)
    f = ro.lstm_cell_fwd64(gx, gh, cp, hp, m, dgh=1e-3 * gh.abs())
    for dt in (torch.bfloat16, torch.float32):
        _moved_fails(f["act"], f["act"], dt, f["tol_act"], "act")
        _moved_fails(f["c"], f["c"], torch.float32, f["tol_c"], "c")
        _moved_fails(f["h"], f["h"], dt, f["tol_h"], "h")
    b = ro.lstm_cell_bwd64(torch.randn(B, H, generator=g, dtype=F64), torch.randn(B, H, generator=g, dtype=F64),
                           torch.randn(B, H, generator=g, dtype=F64), torch.randn(B, H, generator=g, dtype=F64), f["act"], f["c"],
                           cp, m)
    for dt in (torch.bfloat16, torch.float32):
        _moved_fails(b["dG"], b["dG"], dt, b["tol_dG"], "dG")
    _moved_fails(b["dc_prev"], b["dc_prev"], torch.float32, b["tol_dc_prev"], "dc_prev")
    h = torch.randn(6, 3, H, generator=g, dtype=F64)
    mm = torch.ones(6, 3, dtype=F64)
    out, s, _ = ro.masked_mean64(h, mm)
    moved = out + 2 * (lo.red_rel(6) * s + ro.DIV_REL * out.abs())
    with pytest.raises(AssertionError):
        lo.assert_reduction(moved, out, s, 6, extra_abs=ro.DIV_REL * out.abs(), what="masked mean")
    dh, tol = ro.masked_mean_bwd64(torch.randn(3, H, generator=g, dtype=F64), mm)
    _moved_fails(dh, dh, torch.float32, tol, "masked mean dh")
    want, s = go.gemm64(torch.randn(5, 8, generator=g), torch.randn(6, 8, generator=g), 5, 6, 8)
    bnd = go.bound(want, s, 8, torch.float32, torch.float32)
    with pytest.raises(AssertionError):
        go.check(want + 2 * bnd, want, bnd, "h·Uᵀ")
