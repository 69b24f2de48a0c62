"""float64 references of the recurrent kernels (``csrc/rnn_kernels.cu``: the LSTM cell forward / backward, the embedding gather /
scatter and the masked mean over time) and of the whole masked sequence that ``ops/rnn.py::_LSTMSeqFn`` builds from them, written
from each operation's definition.  No GPU is needed: the functions run on the device of their inputs in float64 (a bf16 or fp32
value is exact there).

Conventions (those of the kernels):

* pre-activations ``[B, 4H]`` are sliced i | f | o | c̃ (input, forget, output gate, candidate); the state starts at zero;
* masked carry: ``c = m·c_t + (1 − m)·c_prev`` and ``h = m·h_t + (1 − m)·h_prev`` with m ∈ {0, 1} per row and step;
* backward: ``dh = dh_out + dh_rec + dh_pass_in`` (added in that order), ``dc_prev = dct·f + (1 − m)·dc_next``,
  ``dh_pass = (1 − m)·dh``; dG is the gradient of the pre-activations;
* masked mean over time divides by max(1, Σ_t mask).

Bounds.  Every comparison goes through ``layer_oracle.assert_elementwise`` / ``assert_reduction`` and, for the recurrent GEMMs,
``gemm_oracle.bound``.  Each reference returns, next to a value, ``tol_*``: an absolute allowance per element for everything but
the final store, which ``assert_elementwise`` adds as u_store·|want|.  It is the sum of

* fp32 arithmetic: ``n·2⁻²⁴·s`` with s the magnitude twin of the expression (the same expression on |operands|) and n the
  number of fp32 roundings on its longest chain;
* the fast-math intrinsics.  The kernels are built with ``--use_fast_math``; their SASS holds ``MUFU.EX2``, ``MUFU.RCP`` and
  ``MUFU.TANH`` and no libdevice exp / tanh / divide:

  - ``__expf(x)`` (σ's exponential): at most 2 + ⌊1.173·|x|⌋ ulp (CUDA C++ Programming Guide, single-precision intrinsic
    functions); an ulp of an fp32 result is at most 2⁻²³ of it (:func:`expf_rel`);
  - ``1.f / x`` (σ's reciprocal) is ``rcp.approx.f32``: at most 1 ulp (PTX ISA, ``rcp``), :data:`RCP_REL`;
  - ``x / y`` (the masked mean) is ``div.approx.f32``, computed as x·(1/y): at most 2 ulp for |y| in [2⁻¹²⁶, 2¹²⁶] (PTX ISA,
    ``div``), :data:`DIV_REL`;
  - ``tanhf`` is ``tanh.approx.f32`` (``MUFU.TANH``): maximum relative error 2⁻¹⁰·⁹⁸⁷ (PTX ISA, ``tanh``), :data:`TANH_REL`.
    In the fp32-storage (tf32) mode this, not the storage type, sets the accuracy of g and of tanh(c).

  So σ(z) = 1 / (1 + e^−z) is within (1 − σ)·expf_rel(z) + 2⁻²⁴ + RCP_REL of itself (:func:`sigm_rel`), to first order;
  ``FM_SLACK`` covers the second-order terms;
* the propagation of an error already in an input (the bf16 rounding of the recurrent GEMM's output in a sequence step): the
  allowance of a monotone function (σ, tanh) at z ± Δz, and |a|·Δb + |b|·Δa + Δa·Δb through a product.
"""
import math

import torch

U24 = 2.0 ** -24                 # one fp32 round-to-nearest
ULP = 2.0 ** -23                 # one fp32 ulp, relative to the value it belongs to (upper end)
RCP_REL = 1 * ULP                # rcp.approx.f32: 1 ulp
DIV_REL = 2 * ULP                # div.approx.f32: 2 ulp
TANH_REL = 2.0 ** -10.987        # tanh.approx.f32
FM_SLACK = 1.01


def expf_rel(x):
    """Relative error of ``__expf(x)``: (2 + ⌊1.173·|x|⌋) ulp."""
    return (2.0 + torch.floor(1.173 * x.double().abs())) * ULP


def sigm_rel(z):
    """Relative error of the kernels' σ(z) = rcp(1 + __expf(−z)) at an exact argument z."""
    z = z.double()
    return FM_SLACK * ((1.0 - torch.sigmoid(z)) * expf_rel(z) + U24 + RCP_REL)


def _mono(fn, z, dz):
    """Largest |fn(z ± dz) − fn(z)| of a monotone ``fn``: the effect of an input error dz."""
    y = fn(z)
    return torch.maximum((fn(z + dz) - y).abs(), (fn(z - dz) - y).abs())


def _split(t, H):
    return t[..., :H], t[..., H:2 * H], t[..., 2 * H:3 * H], t[..., 3 * H:]


# --------------------------------------------------------------------------- cell
def lstm_cell_fwd64(gx, gh, c_prev, h_prev, mask, dgh=None):
    """One step: pre = gx + gh, (i, f, o) = σ, g = tanh, c_t = f·c_prev + i·g, h_t = o·tanh(c_t), masked carry.  ``dgh``: an
    absolute error allowance of ``gh`` per element (the recurrent GEMM's, when ``gh`` is recomputed here in float64).  Returns a
    dict: act ([B, 4H], i | f | o | g), c, h, ct, ht and the allowances tol_act, tol_c, tol_h."""
    gx, gh, cp, hp = gx.double(), gh.double(), c_prev.double(), h_prev.double()
    H = cp.shape[-1]
    m = mask.double().reshape(-1, 1)
    pre = gx + gh
    zi, zf, zo, zg = _split(pre, H)
    i, f, o, g = torch.sigmoid(zi), torch.sigmoid(zf), torch.sigmoid(zo), torch.tanh(zg)
    ct = f * cp + i * g
    tc = torch.tanh(ct)
    ht = o * tc
    # pre-activation error: the fp32 add gx + gh, plus what the caller says gh carries
    dpre = U24 * (gx.abs() + gh.abs())
    if dgh is not None:
        dpre = dpre + dgh.double()
    di_, df_, do_, dg_ = _split(dpre, H)
    di = _mono(torch.sigmoid, zi, di_) + sigm_rel(zi) * i
    df = _mono(torch.sigmoid, zf, df_) + sigm_rel(zf) * f
    do = _mono(torch.sigmoid, zo, do_) + sigm_rel(zo) * o
    dg = _mono(torch.tanh, zg, dg_) + FM_SLACK * TANH_REL * g.abs()
    # c_t = fma(f, c_prev, i·g): two fp32 roundings
    dct = (cp.abs() * df + g.abs() * di + i * dg + di * dg) + 2 * U24 * (f * cp.abs() + (i * g).abs())
    dtc = _mono(torch.tanh, ct, dct) + FM_SLACK * TANH_REL * tc.abs()
    dht = tc.abs() * do + o * dtc + do * dtc + U24 * ht.abs()
    act = torch.cat([i, f, o, g], -1)
    return dict(act=act, ct=ct, ht=ht, c=m * ct + (1 - m) * cp, h=m * ht + (1 - m) * hp, pre=pre,
                tol_act=torch.cat([di, df, do, dg], -1), tol_c=m * dct, tol_h=m * dht)


def lstm_cell_bwd64(dh_out, dh_rec, dh_pass_in, dc_next, act, c, c_prev, mask):
    """One backward step from the kernel's own saved ``act`` (i | f | o | g as stored), c = c_t and c_prev; the optional inputs
    may be None (the last step).  Returns a dict: dG, dc_prev, dh_pass, dh, dct and the allowances tol_dG, tol_dc_prev."""
    z = torch.zeros_like(c, dtype=torch.float64)
    dho = dh_out.double()
    dhr = dh_rec.double() if dh_rec is not None else z
    dhp = dh_pass_in.double() if dh_pass_in is not None else z
    dcn = dc_next.double() if dc_next is not None else z
    H = c.shape[-1]
    i, f, o, g = _split(act.double(), H)
    c, cp = c.double(), c_prev.double()
    m = mask.double().reshape(-1, 1)
    dh = dho + dhr + dhp
    s_dh = dho.abs() + dhr.abs() + dhp.abs()
    tc = torch.tanh(c)
    dtanh = 1 - tc * tc
    dht = m * dh
    dct = m * dcn + dht * o * dtanh
    dc_prev = dct * f + (1 - m) * dcn
    dG = torch.cat([dct * g * i * (1 - i), dct * cp * f * (1 - f), dht * tc * o * (1 - o), dct * i * (1 - g * g)], -1)
    # tanh(c) is tanh.approx: |Δtc| ≤ TANH_REL·|tc|, so |Δ(1 − tc²)| ≤ 2·|tc|·|Δtc| (+ its square)
    e_tc = FM_SLACK * TANH_REL * tc.abs()
    e_dtanh = 2 * tc.abs() * e_tc + e_tc * e_tc
    # dh: two adds; dct: tc·tc, 1 − ·, dht·o, ·(1 − tc²), + m·dc_next
    s_dct = m * dcn.abs() + m * s_dh * o * (1 + tc * tc)
    e_dct = (m * s_dh * o) * e_dtanh + 8 * U24 * s_dct
    e_dG = torch.cat([e_dct * (g * i * (1 - i)).abs() + 8 * U24 * (dct * g * i).abs(),
                      e_dct * (cp * f * (1 - f)).abs() + 8 * U24 * (dct * cp * f).abs(),
                      m * s_dh * (e_tc + 8 * U24 * tc.abs()) * o * (1 - o),
                      e_dct * (i * (1 - g * g)).abs() + 8 * U24 * (dct * i).abs() * (1 + g * g)], -1)
    e_dc = e_dct * f + 4 * U24 * (s_dct * f + (1 - m) * dcn.abs())
    return dict(dG=dG, dc_prev=dc_prev, dh_pass=(1 - m) * dh, dh=dh, dct=dct, tol_dG=e_dG, tol_dc_prev=e_dc,
                tol_dh_pass=(1 - m) * 2 * U24 * s_dh)


# --------------------------------------------------------------------------- whole sequence
def lstm_seq64(gx, U, mask, dh_all=None):
    """The masked recurrence over ``gx`` [T, B, 4H] with ``U`` [4H, H] from a zero state: h_t from pre_t = gx_t + h_{t−1}·Uᵀ.
    Returns a dict: hs, cs ([T + 1, B, H]; index 0 is the zero state), act [T, B, 4H] and, with ``dh_all`` [T, B, H] (the
    gradient reaching every h_t from above), dG [T, B, 4H] (= the gradient of gx), dU = Σ_t dG_tᵀ·h_{t−1}."""
    gx, U, mask = gx.double(), U.double(), mask.double()
    T, B, H4 = gx.shape
    H = H4 // 4
    hs, cs, act = [gx.new_zeros((B, H))], [gx.new_zeros((B, H))], []
    for t in range(T):
        r = lstm_cell_fwd64(gx[t], hs[t] @ U.t(), cs[t], hs[t], mask[t])
        hs.append(r["h"]); cs.append(r["c"]); act.append(r["act"])
    out = dict(hs=torch.stack(hs), cs=torch.stack(cs), act=torch.stack(act))
    if dh_all is not None:
        out.update(lstm_seq_bwd64(out["act"], out["cs"], out["hs"], U, mask, dh_all))
    return out


def lstm_seq_bwd64(act, cs, hs, U, mask, dh_all):
    """The backward of :func:`lstm_seq64` from given forward states (act [T, B, 4H], cs / hs [T + 1, B, H]).  Returns a dict: dG,
    dU.  Called with |dh_all|, |U|, |cs|, |hs| and act with |g|, every term of every sum is non-negative: the result is then
    the magnitude twin of the backward (the scale of its rounding errors)."""
    act, cs, hs, U, mask, dh_all = act.double(), cs.double(), hs.double(), U.double(), mask.double(), dh_all.double()
    T, B, H4 = act.shape
    dG = [None] * T
    dc = dpass = drec = None
    for t in range(T - 1, -1, -1):
        r = lstm_cell_bwd64(dh_all[t], drec, dpass, dc, act[t], cs[t + 1], cs[t], mask[t])
        dG[t], dc, dpass = r["dG"], r["dc_prev"], r["dh_pass"]
        drec = dG[t] @ U
    dG = torch.stack(dG)
    return dict(dG=dG, dU=dG.reshape(T * B, H4).t() @ hs[:T].reshape(T * B, H4 // 4))


# --------------------------------------------------------------------------- embedding
def embedding64(ids, W):
    return W.double()[ids.reshape(-1)].reshape(tuple(ids.shape) + (W.shape[1],))


def embedding_bwd64(ids, dout, V):
    """dW[v] = Σ_{n: ids[n] = v} dout[n]; returns (dW, Σ|term| per element, occurrences of each id)."""
    flat = ids.reshape(-1)
    D = dout.shape[-1]
    d = dout.double().reshape(-1, D)
    dW = d.new_zeros((V, D)).index_add_(0, flat, d)
    s = d.new_zeros((V, D)).index_add_(0, flat, d.abs())
    cnt = torch.bincount(flat, minlength=V)
    return dW, s, cnt


# --------------------------------------------------------------------------- masked mean
def masked_mean64(h, mask):
    """out[b] = Σ_t m[t, b]·h[t, b] / max(1, Σ_t m[t, b]) for h [T, B, H]; returns (out, Σ_t |m·h| / max(1, count), count)."""
    h, m = h.double(), mask.double()
    cnt = m.sum(0)
    den = cnt.clamp_min(1)[:, None]
    return (h * m[..., None]).sum(0) / den, (h * m[..., None]).abs().sum(0) / den, cnt


def masked_mean_bwd64(dout, mask):
    """dh[t, b] = dout[b]·m[t, b] / max(1, Σ_s m[s, b]) and its allowance: one fp32 product and the approximate divide."""
    m = mask.double()
    dh = dout.double()[None] * (m / m.sum(0).clamp_min(1))[..., None]
    return dh, (U24 + FM_SLACK * DIV_REL) * dh.abs()
