"""The recurrent kernels (``csrc/rnn_kernels.cu``) and the launch sequence of ``ops/rnn.py::_LSTMSeqFn`` at the LSTM's shapes and
at the edges of their launch geometry, against the float64 references of tests/rnn_oracle.py with per-element bounds (run with
``pytest -m gpu`` on an H100).  Both precision modes.

* cell kernels, called directly: every output within its bound, the masked rows exact;
* σ and tanh of the fp32-storage mode over [−40, 40] against the documented fast-math errors;
* the sequence node forward and a driver of its backward launches, each step checked from the kernel's own state (so error does
  not compound), the node tied to the driver bit for bit in deterministic mode, dU against float64, the padded steps exact;
* the drift of the whole sequence against float64, recorded and not asserted (the recurrence is not provably contractive);
* the embedding gather (exact), its scatter (exact on integers, a per-id reduction bound on random data, the fixed ascending-row
  order in deterministic mode) and the masked mean.

``TMPI_TEST_OUT`` names the directory that ``rnn_ratios.json`` (the largest |diff| / bound per family and the drift table) is
written to; by default it is pytest's temporary directory."""
import gc
import json
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import gemm_oracle as go
import layer_oracle as lo
import rnn_oracle as ro
from theanompi_b200.models.lstm import bucket_len, pad_batch
from theanompi_b200.ops import precision, rnn

pytestmark = pytest.mark.gpu
DEV = "cuda"
HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
DT = {"bf16": torch.bfloat16, "tf32": torch.float32}
F32 = torch.float32
MAXLEN = 500                   # the LSTM's maxlen: buckets up to 512 steps
RATIOS = {}
DRIFT = []


def _ci():
    from theanompi_b200.ops import cuda_impl
    return cuda_impl


@pytest.fixture(params=["bf16", "tf32"])
def dtype(request):
    old = precision.precision()
    precision.set_precision(request.param)
    try:
        yield DT[request.param]
    finally:
        precision.set_precision(old)


@pytest.fixture(autouse=True)
def _release_memory():
    yield
    gc.collect()
    torch.cuda.empty_cache()


@pytest.fixture(scope="module", autouse=True)
def _ratios(tmp_path_factory):
    yield
    out = os.environ.get("TMPI_TEST_OUT") or str(tmp_path_factory.mktemp("rnn"))
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "rnn_ratios.json"), "w") as f:
        json.dump(dict(card=torch.cuda.get_device_name(0), ratios=dict(sorted(RATIOS.items())), drift=DRIFT), f, indent=1)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _fam(family, dtype):
    return family + ("-bf16" if dtype == torch.bfloat16 else "-tf32")


def _chk(got, want, store, tol, what, family, dtype):
    """assert_elementwise with u_store·|want| + ``tol``, and the largest |diff| / bound recorded under ``family``."""
    _, diff, bound = lo.elementwise_violations(got, want, store, extra_abs=tol)
    if diff.numel():
        r = float(torch.where(bound > 0, diff / bound.clamp_min(1e-300), torch.where(diff > 0, math.inf, 0.0)).max())
        RATIOS[_fam(family, dtype)] = max(RATIOS.get(_fam(family, dtype), 0.0), r)
    lo.assert_elementwise(got, want, store, extra_abs=tol, what=what)


def _f32(dtype):
    return int(dtype == F32)


def _st():
    return torch.cuda.current_stream().cuda_stream


def _ptr(t):
    return 0 if t is None else t.data_ptr()


# =========================================================================== a. cell kernels
CELL_SHAPES = [(16, 128), (1, 8), (2, 128), (37, 72), (16, 264)]      # the model; tiny; one 256-thread CTA; ragged last CTA; wide
PRE = ["normal3", "wide40"]
MASKS = ["ones", "zeros", "mixed"]


def _mask_rows(B, kind, g):
    if kind == "ones":
        return torch.ones(B, device=DEV)
    if kind == "zeros":
        return torch.zeros(B, device=DEV)
    m = (torch.rand(B, device=DEV, generator=g) < 0.5).float()
    m[0] = 1
    m[-1] = 0 if B > 1 else 1
    return m


def _cell_inputs(B, H, pre, mkind, dtype, seed):
    g = _gen(seed)
    if pre == "normal3":
        gx = torch.randn(B, 4 * H, device=DEV, generator=g) * 3
        gh = torch.randn(B, 4 * H, device=DEV, generator=g)
    else:                                      # out to |z| ≈ 40: σ and tanh saturate, __expf's ulp count is largest
        gx = (torch.rand(B, 4 * H, device=DEV, generator=g) * 2 - 1) * 38
        gh = torch.randn(B, 4 * H, device=DEV, generator=g)
    cp = torch.randn(B, H, device=DEV, generator=g) * 2
    hp = torch.tanh(torch.randn(B, H, device=DEV, generator=g)).to(dtype)
    return gx.to(dtype), gh.to(dtype), cp, hp, _mask_rows(B, mkind, g)


def _cell_fwd(gx, gh, cp, hp, m, dtype):
    B, H = cp.shape
    act = torch.empty(B, 4 * H, dtype=dtype, device=DEV)
    c = torch.empty(B, H, dtype=F32, device=DEV)
    h = torch.empty(B, H, dtype=dtype, device=DEV)
    _ci().L().lstm_cell_fwd(gx.data_ptr(), gh.data_ptr(), cp.data_ptr(), hp.data_ptr(), m.data_ptr(), act.data_ptr(), c.data_ptr(),
                            h.data_ptr(), B, H, _f32(dtype), _st())
    return act, c, h


def _cell_bwd(dh_out, dh_rec, dpass_in, dc_next, act, c, cp, m, dtype):
    B, H = cp.shape
    dG = torch.empty(B, 4 * H, dtype=dtype, device=DEV)
    dc_prev = torch.empty(B, H, dtype=F32, device=DEV)
    dh_pass = torch.empty(B, H, dtype=F32, device=DEV)
    _ci().L().lstm_cell_bwd(dh_out.data_ptr(), _ptr(dh_rec), _ptr(dpass_in), _ptr(dc_next), act.data_ptr(), c.data_ptr(), cp.data_ptr(),
                            m.data_ptr(), dG.data_ptr(), dc_prev.data_ptr(), dh_pass.data_ptr(), B, H, _f32(dtype), _st())
    return dG, dc_prev, dh_pass


@pytest.mark.parametrize("mkind", MASKS)
@pytest.mark.parametrize("pre", PRE)
@pytest.mark.parametrize("shape", CELL_SHAPES, ids=lambda s: "B%dH%d" % s)
def test_cell_forward(shape, pre, mkind, dtype):
    B, H = shape
    gx, gh, cp, hp, m = _cell_inputs(B, H, pre, mkind, dtype, seed=B * 1000 + H)
    act, c, h = _cell_fwd(gx, gh, cp, hp, m, dtype)
    torch.cuda.synchronize()
    f = ro.lstm_cell_fwd64(gx, gh, cp, hp, m)
    _chk(act, f["act"], dtype, f["tol_act"], "act", "cell-act", dtype)
    _chk(c, f["c"], F32, f["tol_c"], "c", "cell-c", dtype)
    _chk(h, f["h"], dtype, f["tol_h"], "h", "cell-h", dtype)
    off = m == 0
    assert torch.equal(c[off], cp[off]), "a masked row carries c_prev, bit for bit"
    assert torch.equal(h[off], hp[off]), "a masked row carries h_prev, bit for bit"


@pytest.mark.parametrize("optional", [True, False], ids=["all-inputs", "last-step"])
@pytest.mark.parametrize("mkind", MASKS)
@pytest.mark.parametrize("pre", PRE)
@pytest.mark.parametrize("shape", CELL_SHAPES, ids=lambda s: "B%dH%d" % s)
def test_cell_backward(shape, pre, mkind, optional, dtype):
    B, H = shape
    gx, gh, cp, hp, m = _cell_inputs(B, H, pre, mkind, dtype, seed=B * 1000 + H + 1)
    act, c, _ = _cell_fwd(gx, gh, cp, hp, m, dtype)
    g = _gen(B + H)
    dh_out = torch.randn(B, H, device=DEV, generator=g).to(dtype)
    dh_rec = torch.randn(B, H, device=DEV, generator=g).to(dtype) if optional else None
    dpass_in = torch.randn(B, H, device=DEV, generator=g) if optional else None
    dc_next = torch.randn(B, H, device=DEV, generator=g) * 2 if optional else None
    dG, dc_prev, dh_pass = _cell_bwd(dh_out, dh_rec, dpass_in, dc_next, act, c, cp, m, dtype)
    torch.cuda.synchronize()
    b = ro.lstm_cell_bwd64(dh_out, dh_rec, dpass_in, dc_next, act, c, cp, m)
    _chk(dG, b["dG"], dtype, b["tol_dG"], "dG", "cell-dG", dtype)
    _chk(dc_prev, b["dc_prev"], F32, b["tol_dc_prev"], "dc_prev", "cell-dc", dtype)
    _chk(dh_pass, b["dh_pass"], F32, b["tol_dh_pass"], "dh_pass", "cell-dhpass", dtype)
    off, on = m == 0, m != 0
    assert torch.equal(dG[off], torch.zeros_like(dG[off])), "a masked row has no gate gradient"
    assert torch.equal(dc_prev[off], dc_next[off] if optional else torch.zeros_like(dc_prev[off])), "dc passes a masked row unchanged"
    dh = dh_out.float()
    if optional:
        dh = (dh + dh_rec.float()) + dpass_in
    assert torch.equal(dh_pass[off], dh[off]), "dh passes a masked row as (dh_out + dh_rec) + dh_pass_in"
    assert torch.equal(dh_pass[on], torch.zeros_like(dh_pass[on])), "a valid row passes nothing"


# =========================================================================== b. transcendental sweep (fp32 storage)
def test_fast_math_sweep():
    """σ and tanh as the fp32-storage cell computes them (gh = 0, so the pre-activation is exact), 2²⁰ arguments over [−40, 40]
    and 0, against float64 with the documented fast-math errors (rnn_oracle)."""
    old = precision.precision()
    precision.set_precision("tf32")
    try:
        B, H = 4096, 256
        z = torch.linspace(-40.0, 40.0, B * H - 1, device=DEV)
        z = torch.cat([z, torch.zeros(1, device=DEV)]).view(B, H)
        gx = torch.cat([z, z, z, z], 1).contiguous()
        gh = torch.zeros_like(gx)
        zero = torch.zeros(B, H, device=DEV)
        act, _, _ = _cell_fwd(gx, gh, zero, zero, torch.ones(B, device=DEV), F32)
        torch.cuda.synchronize()
        z64 = z.double()
        sig, th = torch.sigmoid(z64), torch.tanh(z64)
        for k, name in ((0, "i"), (1, "f"), (2, "o")):
            got = act[:, k * H:(k + 1) * H]
            _, diff, _ = lo.elementwise_violations(got, sig, F32)
            bound = ro.sigm_rel(z64) * sig
            RATIOS["sweep-sigmoid"] = max(RATIOS.get("sweep-sigmoid", 0.0), float((diff / bound).max()))
            go.check(got, sig, bound, "σ (%s gate)" % name)
        got = act[:, 3 * H:]
        bound = ro.FM_SLACK * ro.TANH_REL * th.abs()
        diff = (got.double() - th).abs()
        RATIOS["sweep-tanh"] = float(torch.where(bound > 0, diff / bound.clamp_min(1e-300), diff * math.inf).nan_to_num(0.0).max())
        go.check(got, th, bound, "tanh (g)")
    finally:
        precision.set_precision(old)


# =========================================================================== c–f. the sequence node
SEQ_SHAPES = [(16, 128, 1), (16, 128, 2), (16, 128, 16), (16, 128, 80), (16, 128, 512), (1, 8, 3), (37, 72, 17)]
SEQ_MASKS = ["ones", "prefix", "bucket", "holes"]


def _lengths(B, T, g):
    n = torch.randint(1, T + 1, (B,), generator=g)
    n[0] = 1
    n[-1] = T
    return n.numpy()


def _seq_inputs(B, H, T, mkind, dtype, seed):
    """(gx [Tb, B, 4H] in the activation dtype, U fp32 [4H, H], mask [Tb, B], lengths or None).  ``bucket``: lengths up to T,
    the batch padded to its graph bucket with the model's own bucket_len / pad_batch (token id 0, mask 0)."""
    g = torch.Generator().manual_seed(seed)
    lens = None
    if mkind == "ones":
        mask = np.ones((B, T), dtype=np.float32)
    elif mkind == "holes":                       # masked steps anywhere, also between valid ones
        mask = (torch.rand(B, T, generator=g) < 0.7).float().numpy()
        mask[:, 0] = 1
    else:
        lens = _lengths(B, T, g)
        mask = (np.arange(T)[None, :] < lens[:, None]).astype(np.float32)
        if mkind == "bucket":
            x = np.ones((B, T), dtype=np.int64)
            _, mask = pad_batch(x, mask, bucket_len(T, MAXLEN))
    Tb = mask.shape[1]
    gx = (torch.randn(Tb, B, 4 * H, generator=g) * 1.5).to(DEV).to(dtype)
    U = (torch.randn(4 * H, H, generator=g) / H ** 0.5).to(DEV)
    return gx, U, torch.from_numpy(mask).t().contiguous().to(DEV), lens


def _node(gx, U, mask, dh_all=None):
    """The sequence through ``rnn.lstm_sequence``; returns h, the saved hs / cs / act and, with ``dh_all``, gx.grad and dU."""
    gx = gx.detach().clone().requires_grad_(True)
    U = U.detach().clone().requires_grad_(True)
    h = rnn.lstm_sequence(gx, U, mask)
    hs, cs, act, m = [t.clone() for t in h.grad_fn.saved_tensors]
    out = dict(h=h.detach(), hs=hs, cs=cs, act=act, mask=m)
    if dh_all is not None:
        h.backward(dh_all)
        out.update(dgx=gx.grad, dU=U.grad)
    torch.cuda.synchronize()
    return out


def _drive_bwd(hs, cs, act, mask, uc, dh_all):
    """The launch sequence of ``_LSTMSeqFn.backward``, with the ring buffers it does not save recorded at every step: returns dG,
    dU and per step the inputs the cell kernel read (dh_rec, dh_pass_in, dc_next; zero at the last step) and the drec it made."""
    ci = _ci()
    L = ci.L()
    Tn, B, H4 = act.shape
    H = H4 // 4
    dt = act.dtype
    dG = torch.empty((Tn, B, H4), dtype=dt, device=DEV)
    dc = [torch.zeros((B, H), device=DEV) for _ in range(2)]
    dpass = [torch.zeros((B, H), device=DEV) for _ in range(2)]
    drec = torch.empty((B, H), dtype=dt, device=DEV)
    rec = dict(dh_rec=torch.zeros((Tn, B, H), dtype=dt, device=DEV), dpass_in=torch.zeros((Tn, B, H), device=DEV),
               dc_next=torch.zeros((Tn, B, H), device=DEV), dc_prev=torch.empty((Tn, B, H), device=DEV),
               dh_pass=torch.empty((Tn, B, H), device=DEV))
    for t in range(Tn - 1, -1, -1):
        last = t == Tn - 1
        k = t & 1
        if not last:
            rec["dh_rec"][t].copy_(drec); rec["dpass_in"][t].copy_(dpass[1 - k]); rec["dc_next"][t].copy_(dc[1 - k])
        L.lstm_cell_bwd(dh_all[t].data_ptr(), 0 if last else drec.data_ptr(), 0 if last else dpass[1 - k].data_ptr(),
                        0 if last else dc[1 - k].data_ptr(), act[t].data_ptr(), cs[t + 1].data_ptr(), cs[t].data_ptr(),
                        mask[t].data_ptr(), dG[t].data_ptr(), dc[k].data_ptr(), dpass[k].data_ptr(), B, H, _f32(dt), _st())
        rec["dc_prev"][t].copy_(dc[k]); rec["dh_pass"][t].copy_(dpass[k])
        if t > 0:
            ci.gemm(dG[t], uc, B, H, H4, b_mn=True, out=drec, lda=H4, ldb=H, ldc=H)
    dU = torch.empty((H4, H), device=DEV)
    ci.gemm(dG.view(Tn * B, H4), hs[:Tn].reshape(Tn * B, H), H4, H, Tn * B, a_mn=True, b_mn=True, out=dU, lda=H4, ldb=H, ldc=H)
    torch.cuda.synchronize()
    rec.update(dG=dG, dU=dU)
    return rec


def _rows(t):
    return t.reshape(-1, t.shape[-1])


def _check_forward_steps(r, uc, gx, dtype, tag):
    """Every step from the kernel's own h_{t−1}, c_{t−1}: h·Uᵀ in float64 with the GEMM's bound, then the cell with its bound."""
    hs, cs, act, mask = r["hs"], r["cs"], r["act"], r["mask"]
    Tn, B, H4 = act.shape
    H = H4 // 4
    hp = hs[:Tn].double()
    gh = hp @ uc.double().t()
    s = hp.abs() @ uc.double().abs().t()
    dgh = go.bound(gh, s, H, dtype, dtype)
    f = ro.lstm_cell_fwd64(_rows(gx), _rows(gh), _rows(cs[:Tn]), _rows(hs[:Tn]), mask.reshape(-1), dgh=_rows(dgh))
    _chk(_rows(act), f["act"], dtype, f["tol_act"], tag + "act", "seq-act", dtype)
    _chk(_rows(cs[1:]), f["c"], F32, f["tol_c"], tag + "c", "seq-c", dtype)
    _chk(_rows(hs[1:]), f["h"], dtype, f["tol_h"], tag + "h", "seq-h", dtype)


def _check_backward_steps(d, r, uc, mask, dh_all, dtype, tag):
    """Every cell step from the inputs it read, every drec = dG_t·U and dU = Σ dG_tᵀ·h_{t−1} against float64."""
    act, cs, hs = r["act"], r["cs"], r["hs"]
    Tn, B, H4 = act.shape
    H = H4 // 4
    b = ro.lstm_cell_bwd64(_rows(dh_all), _rows(d["dh_rec"]), _rows(d["dpass_in"]), _rows(d["dc_next"]), _rows(act), _rows(cs[1:]),
                           _rows(cs[:Tn]), mask.reshape(-1))
    _chk(_rows(d["dG"]), b["dG"], dtype, b["tol_dG"], tag + "dG", "seq-dG", dtype)
    _chk(_rows(d["dc_prev"]), b["dc_prev"], F32, b["tol_dc_prev"], tag + "dc", "seq-dc", dtype)
    _chk(_rows(d["dh_pass"]), b["dh_pass"], F32, b["tol_dh_pass"], tag + "dpass", "seq-dhpass", dtype)
    if Tn > 1:                                       # drec made at step t is the dh_rec step t − 1 read
        dG = d["dG"][1:].double()
        want, s = dG @ uc.double(), dG.abs() @ uc.double().abs()
        go.check(d["dh_rec"][:-1], want, go.bound(want, s, H4, dtype, dtype), tag + "drec = dG·U", RATIOS, _fam("seq-drec", dtype))
    dGn = r["dgx"].double().reshape(Tn * B, H4)
    hh = hs[:Tn].double().reshape(Tn * B, H)
    want, s = dGn.t() @ hh, dGn.abs().t() @ hh.abs()
    splits = go.gemm_plan(_ci().L(), H4, H, Tn * B, dtype == F32, True, True, out_bf16=False)[2]
    go.check(r["dU"], want, go.bound(want, s, Tn * B, dtype, F32, splits=splits), tag + "dU", RATIOS, _fam("seq-dU", dtype))


def _seq_case(B, H, T, mkind, dtype, seed):
    gx, U, mask, lens = _seq_inputs(B, H, T, mkind, dtype, seed)
    uc = U.to(dtype)
    dh_all = (torch.randn(gx.shape[:2] + (H,), device=DEV, generator=_gen(seed)) * 0.5).to(dtype)
    r = _node(gx, U, mask, dh_all)
    return gx, U, uc, mask, lens, dh_all, r


@pytest.mark.parametrize("mkind", SEQ_MASKS)
@pytest.mark.parametrize("shape", SEQ_SHAPES, ids=lambda s: "B%dH%dT%d" % s)
def test_sequence_steps(shape, mkind, dtype):
    B, H, T = shape
    gx, U, uc, mask, lens, dh_all, r = _seq_case(B, H, T, mkind, dtype, seed=B + H + T)
    tag = "B%d H%d T%d %s: " % (B, H, mask.shape[0], mkind)
    _check_forward_steps(r, uc, gx, dtype, tag)
    d = _drive_bwd(r["hs"], r["cs"], r["act"], r["mask"], uc, dh_all)
    _check_backward_steps(d, r, uc, r["mask"], dh_all, dtype, tag)
    if lens is not None:                             # e. padded steps: exact
        hs = r["hs"]
        for b, n in enumerate(lens.tolist()):
            Tb = mask.shape[0]
            assert torch.equal(hs[n + 1:, b], hs[n, b].expand(Tb - n, H)), "padded steps carry the last valid h, bit for bit"
            assert torch.equal(r["dgx"][n:, b], torch.zeros_like(r["dgx"][n:, b])), "padded steps have no input gradient"


@pytest.mark.parametrize("T", [1, 16, 80, 512])
def test_sequence_drift(T, dtype):
    """The node against the float64 recurrence from the same gx, U (its compute copy) and mask: recorded, finite."""
    B, H = 16, 128
    gx, U, uc, mask, _, dh_all, r = _seq_case(B, H, T, "bucket", dtype, seed=T + 7)
    w = ro.lstm_seq64(gx, uc, mask, dh_all)
    dh = float((r["h"].double() - w["hs"][1:]).abs().max())
    dg = float((r["dgx"].double() - w["dG"]).abs().max())
    du = float((r["dU"].double() - w["dU"]).abs().max())
    DRIFT.append(dict(T=mask.shape[0], dtype="bf16" if dtype == torch.bfloat16 else "tf32", max_abs_dh=dh, max_abs_dgx=dg, max_abs_dU=du,
                      max_abs_h=float(w["hs"].abs().max()), max_abs_dU_ref=float(w["dU"].abs().max())))
    assert all(math.isfinite(v) for v in (dh, dg, du))


def check_node_matches_driver():
    """Run with TMPI_DETERMINISTIC=1 (no split-K: every GEMM has one summation order): the node's gx.grad and dU are the driver's,
    bit for bit."""
    for name in ("bf16", "tf32"):
        precision.set_precision(name)
        dtype = DT[name]
        for (B, H, T), mkind in (((16, 128, 80), "bucket"), ((37, 72, 17), "prefix"), ((16, 128, 512), "ones")):
            _, _, uc, mask, _, dh_all, r = _seq_case(B, H, T, mkind, dtype, seed=3)
            d = _drive_bwd(r["hs"], r["cs"], r["act"], r["mask"], uc, dh_all)
            assert torch.equal(r["dgx"], d["dG"]), (name, B, H, T, "gx.grad")
            assert torch.equal(r["dU"], d["dU"]), (name, B, H, T, "dU")
    return True


def _subprocess(code, timeout=900):
    env = dict(os.environ, TMPI_DETERMINISTIC="1", PYTHONPATH=ROOT)
    r = subprocess.run([sys.executable, "-c", "import sys; sys.path.insert(0, %r)\n" % HERE + code], env=env, cwd=ROOT,
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=timeout)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:]


def test_node_matches_driver_deterministic():
    _subprocess("import test_gpu_rnn_shapes as t\nt.check_node_matches_driver()\nprint('OK')\n")


# =========================================================================== g. embedding
V = 10000                       # the LSTM's vocabulary


def _model_ids(seed, T=512, B=16):
    """Token ids of the model's padded batch: lengths 100–500 padded to the 512-step bucket with id 0, time-major [T, B] (the layout
    ``forward_logits`` passes); ids 0 and V − 1 both occur."""
    rs = np.random.RandomState(seed)
    lens = rs.randint(100, 501, B)
    lens[-1] = 500
    x = np.zeros((B, int(lens.max())), dtype=np.int64)
    for b, n in enumerate(lens):
        x[b, :n] = rs.randint(2, V, n)
    x[0, 0], x[1, 0] = 0, V - 1
    xp, _ = pad_batch(x, np.ones_like(x, dtype=np.float32), bucket_len(x.shape[1], MAXLEN))
    assert xp.shape[1] == T
    return torch.from_numpy(xp).t().contiguous().to(DEV)


@pytest.mark.parametrize("D", [8, 128, 136, 264])
def test_embedding_forward_exact(D, dtype):
    ids = _model_ids(D)
    W = torch.randn(V, D, device=DEV, generator=_gen(D))
    e = rnn.embedding(ids, W)
    torch.cuda.synchronize()
    assert e.dtype == dtype and torch.equal(e, W.to(dtype)[ids]), "the gather copies rows, bit for bit"


def _emb_bwd(ids, dout):
    W = torch.zeros(V, dout.shape[-1], device=DEV, requires_grad=True)
    rnn.embedding(ids, W).backward(dout)
    torch.cuda.synchronize()
    return W.grad


@pytest.mark.parametrize("D", [8, 128, 136, 264])
def test_embedding_backward_integers_exact(D, dtype):
    """Integer dout: every fp32 partial sum is exact, so any order gives the exact sum; the padded batch puts thousands of rows on
    id 0."""
    ids = _model_ids(D + 1)
    dout = torch.randint(-4, 5, tuple(ids.shape) + (D,), device=DEV, generator=_gen(D)).float().to(dtype)
    want, s, cnt = ro.embedding_bwd64(ids, dout, V)
    assert int(cnt[0]) > 1000 and int(cnt[V - 1]) >= 1
    go.assert_exact_range(s)
    go.assert_exact(_emb_bwd(ids, dout), want, "dW (integers)")


@pytest.mark.parametrize("D", [8, 128, 264])
def test_embedding_backward_random(D, dtype):
    ids = _model_ids(D + 2)
    dout = torch.randn(tuple(ids.shape) + (D,), device=DEV, generator=_gen(D)).to(dtype)
    want, s, cnt = ro.embedding_bwd64(ids, dout, V)
    got = _emb_bwd(ids, dout)
    assert torch.equal(got[cnt == 0], torch.zeros_like(got[cnt == 0]))
    for n in torch.unique(cnt[cnt > 0]).tolist():      # a reduction bound over each id's own number of rows
        sel = cnt == n
        lo.assert_reduction(got[sel], want[sel], s[sel], int(n), what="dW of the ids with %d rows" % n)


def check_embedding_deterministic():
    """Run with TMPI_DETERMINISTIC=1: dW is np.add.at on float32 (rows added in ascending index order), twice the same bits, eagerly
    and replayed from a captured CUDA graph."""
    L = _ci().L()
    for name in ("bf16", "tf32"):
        precision.set_precision(name)
        dtype = DT[name]
        for D in (128, 264):
            ids = _model_ids(D + 3)
            n = ids.numel()
            dout = torch.randn(n, D, device=DEV, generator=_gen(D)).to(dtype)
            want = np.zeros((V, D), dtype=np.float32)
            np.add.at(want, ids.reshape(-1).cpu().numpy(), dout.float().cpu().numpy())
            want = torch.from_numpy(want).to(DEV)
            flat = ids.reshape(-1).contiguous()
            runs = []
            for _ in range(2):
                dW = torch.full((V, D), float("nan"), device=DEV)
                L.embedding_bwd(flat.data_ptr(), dout.data_ptr(), dW.data_ptr(), n, D, V, _f32(dtype), _st())
                torch.cuda.synchronize()
                runs.append(dW)
            assert torch.equal(runs[0], runs[1]), (name, D, "two runs differ")
            assert torch.equal(runs[0], want), (name, D, "dW is not the ascending-order fp32 sum", int((runs[0] != want).sum()))
            dW = torch.full((V, D), float("nan"), device=DEV)
            s = torch.cuda.Stream()
            s.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(s):
                L.embedding_bwd(flat.data_ptr(), dout.data_ptr(), dW.data_ptr(), n, D, V, _f32(dtype), _st())
            torch.cuda.current_stream().wait_stream(s)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                L.embedding_bwd(flat.data_ptr(), dout.data_ptr(), dW.data_ptr(), n, D, V, _f32(dtype), _st())
            dW.fill_(float("nan"))
            graph.replay()
            torch.cuda.synchronize()
            assert torch.equal(dW, want), (name, D, "graph replay")
    return True


def test_embedding_backward_deterministic():
    _subprocess("import test_gpu_rnn_shapes as t\nt.check_embedding_deterministic()\nprint('OK')\n")


# =========================================================================== h. masked mean
def _mean_mask(T, B, kind, g):
    if kind == "prefix":
        lens = torch.randint(1, T + 1, (B,), generator=g)
        lens[0] = T
        m = (torch.arange(T)[:, None] < lens[None, :]).float()
    else:                                              # holes anywhere
        m = (torch.rand(T, B, generator=g) < 0.6).float()
        m[:, 0] = 1
    m[:, B // 2] = 0                                   # a sequence with no valid step
    return m.to(DEV)


@pytest.mark.parametrize("kind", ["prefix", "holes"])
@pytest.mark.parametrize("T,B,H", [(1, 16, 128), (16, 16, 128), (512, 16, 128), (17, 37, 72)])
def test_masked_mean(T, B, H, kind, dtype):
    g = torch.Generator().manual_seed(T + B)
    mask = _mean_mask(T, B, kind, g)
    h = (torch.randn(T, B, H, generator=g) * 2).to(DEV).to(dtype).requires_grad_(True)
    dout = torch.randn(B, H, generator=g).to(DEV).to(dtype)
    out = rnn.masked_mean(h, mask)
    out.backward(dout)
    torch.cuda.synchronize()
    want, s, cnt = ro.masked_mean64(h.detach(), mask)
    extra = (ro.FM_SLACK * ro.DIV_REL + go.U_STORE_REL[dtype]) * want.abs()
    lo.assert_reduction(out, want, s, T, extra_abs=extra, what="masked mean")
    dh, tol = ro.masked_mean_bwd64(dout, mask)
    _chk(h.grad, dh, dtype, tol, "masked mean dh", "mean-dh", dtype)
    e = B // 2
    assert torch.equal(out[e], torch.zeros_like(out[e])) and torch.equal(h.grad[:, e], torch.zeros_like(h.grad[:, e]))
