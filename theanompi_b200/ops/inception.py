"""GoogLeNet inception module as ONE autograd node (ref ``theanompi/models/googlenet.py:46-181``: four branches + concat).

What the composition of separate layers costs at batch 32 — the reference's batch size — is not FLOPs but launches
and idle SMs: 6 convolutions + a pool + a ``torch.cat`` forward, the mirror image plus three gradient adds backward, each conv
with 13–196 output tiles for 132 SMs.  This node

* writes every branch's output straight into its channel slice of the concatenated tensor (the implicit-GEMM epilogue takes a
  channel offset and a row pitch) and reads the gradient slices in place — no concat, no split copies;
* runs the four branches on four CUDA streams (fork / join with events, captured as parallel branches of the step's CUDA
  graph), forward and backward, so the small persistent GEMM launches share the machine instead of queueing;
* merges the four input gradients with one native kernel.
"""
from __future__ import annotations

import torch

from . import reference as ref
from .functional import _gout, _sink, compute_weight

_STREAMS = {}


def _side_streams(device, n=3):
    key = (device.index, n)
    if key not in _STREAMS:
        _STREAMS[key] = [torch.cuda.Stream(device=device) for _ in range(n)]
    return _STREAMS[key]


def _cuda_ok(x, ws):
    from . import cuda_impl as ci
    C = x.shape[3]
    al = ci._al(x)
    return x.is_cuda and C % al == 0 and all(w.shape[0] % al == 0 and w.shape[3] % al == 0 for w in ws)


class _InceptFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w1, b1, wr3, br3, w3, b3, wr5, br5, w5, b5, wpj, bpj):
        from . import cuda_impl as ci
        L = ci.L()
        x = ci._bf(x).contiguous()
        N, H, W, C = x.shape
        n1, nr3, n3, nr5, n5, npj = w1.shape[0], wr3.shape[0], w3.shape[0], wr5.shape[0], w5.shape[0], wpj.shape[0]
        Ot = n1 + n3 + n5 + npj
        dev, dt = x.device, x.dtype
        # every tensor is allocated on the main stream; the side streams only launch kernels between the fork and the join
        y = torch.empty((N, H, W, Ot), dtype=dt, device=dev)
        r3 = torch.empty((N, H, W, nr3), dtype=dt, device=dev)
        r5 = torch.empty((N, H, W, nr5), dtype=dt, device=dev)
        pl = torch.empty((N, H, W, C), dtype=dt, device=dev)
        arg = torch.empty((N, H, W, C), dtype=torch.uint8, device=dev)
        cw = compute_weight
        main = torch.cuda.current_stream(dev)
        s1, s2, s3 = _side_streams(dev)
        fork = torch.cuda.Event(); fork.record(main)
        ci._conv_fwd_group(x, cw(w1), b1, y, 0, 0, C, 1, 0, True)
        joins = []
        with torch.cuda.stream(s1):
            s1.wait_event(fork)
            ci._conv_fwd_group(x, cw(wr3), br3, r3, 0, 0, C, 1, 0, True)
            ci._conv_fwd_group(r3, cw(w3), b3, y, n1, 0, nr3, 1, 1, True)
            e = torch.cuda.Event(); e.record(s1); joins.append(e)
        with torch.cuda.stream(s2):
            s2.wait_event(fork)
            ci._conv_fwd_group(x, cw(wr5), br5, r5, 0, 0, C, 1, 0, True)
            ci._conv_fwd_group(r5, cw(w5), b5, y, n1 + n3, 0, nr5, 1, 2, True)
            e = torch.cuda.Event(); e.record(s2); joins.append(e)
        with torch.cuda.stream(s3):
            s3.wait_event(fork)
            L.pool_fwd(x.data_ptr(), pl.data_ptr(), arg.data_ptr(), N, H, W, C, H, W, 3, 1, 1, 1, int(ci._is32(x)), ci._st(x))
            ci._conv_fwd_group(pl, cw(wpj), bpj, y, n1 + n3 + n5, 0, C, 1, 0, True)
            e = torch.cuda.Event(); e.record(s3); joins.append(e)
        for e in joins:
            main.wait_event(e)
        ctx.save_for_backward(x, y, r3, r5, pl, arg)
        ctx.params = (w1, b1, wr3, br3, w3, b3, wr5, br5, w5, b5, wpj, bpj)
        return y

    @staticmethod
    def backward(ctx, dy):
        from . import cuda_impl as ci
        L = ci.L()
        x, y, r3, r5, pl, arg = ctx.saved_tensors
        w1, b1, wr3, br3, w3, b3, wr5, br5, w5, b5, wpj, bpj = ctx.params
        dy = ci._bf(dy).contiguous()
        N, H, W, C = x.shape
        n1, nr3, n3, nr5, n5 = w1.shape[0], wr3.shape[0], w3.shape[0], wr5.shape[0], w5.shape[0]
        need_dx = ctx.needs_input_grad[0]
        dxa, dxb, dxc, dxd = (torch.empty_like(x) for _ in range(4))
        d3, d5, dpl = torch.empty_like(r3), torch.empty_like(r5), torch.empty_like(pl)
        dx = torch.empty_like(x) if need_dx else None
        cw = compute_weight
        main = torch.cuda.current_stream(x.device)
        s1, s2, s3 = _side_streams(x.device)
        fork = torch.cuda.Event(); fork.record(main)
        out = {}
        out["1"] = ci._conv_bwd_group(x, cw(w1), y, dy, dxa, 0, 0, C, 1, 0, True, need_dx, _gout(w1), _gout(b1))
        joins = []
        with torch.cuda.stream(s1):
            s1.wait_event(fork)
            out["3"] = ci._conv_bwd_group(r3, cw(w3), y, dy, d3, n1, 0, nr3, 1, 1, True, True, _gout(w3), _gout(b3))
            out["r3"] = ci._conv_bwd_group(x, cw(wr3), r3, d3, dxb, 0, 0, C, 1, 0, True, need_dx, _gout(wr3), _gout(br3))
            e = torch.cuda.Event(); e.record(s1); joins.append(e)
        with torch.cuda.stream(s2):
            s2.wait_event(fork)
            out["5"] = ci._conv_bwd_group(r5, cw(w5), y, dy, d5, n1 + n3, 0, nr5, 1, 2, True, True, _gout(w5), _gout(b5))
            out["r5"] = ci._conv_bwd_group(x, cw(wr5), r5, d5, dxc, 0, 0, C, 1, 0, True, need_dx, _gout(wr5), _gout(br5))
            e = torch.cuda.Event(); e.record(s2); joins.append(e)
        with torch.cuda.stream(s3):
            s3.wait_event(fork)
            out["pj"] = ci._conv_bwd_group(pl, cw(wpj), y, dy, dpl, n1 + n3 + n5, 0, C, 1, 0, True, True, _gout(wpj), _gout(bpj))
            if need_dx:
                L.pool_bwd(dpl.data_ptr(), arg.data_ptr(), dxd.data_ptr(), N, H, W, C, H, W, 3, 1, 1, 1, int(ci._is32(x)), ci._st(x))
            e = torch.cuda.Event(); e.record(s3); joins.append(e)
        for e in joins:
            main.wait_event(e)
        if need_dx:
            L.add4_tensors(dxa.data_ptr(), dxb.data_ptr(), dxc.data_ptr(), dxd.data_ptr(), dx.data_ptr(), dx.numel(), int(ci._is32(x)), ci._st(x))
        # parameter gradients are delivered on the main stream, after the join (the exchanger's grad-ready callbacks order
        # their side stream behind the CURRENT stream)
        grads = []
        for (w, b), k in (((w1, b1), "1"), ((wr3, br3), "r3"), ((w3, b3), "3"), ((wr5, br5), "r5"), ((w5, b5), "5"), ((wpj, bpj), "pj")):
            dw, db = out[k]
            gb = _sink(b, db)
            gw = _sink(w, dw)
            grads += [gw, gb]
        return (dx,) + tuple(grads)


def inception(x, params):
    """``params`` = (w1, b1, wr3, br3, w3, b3, wr5, br5, w5, b5, wpj, bpj) — OHWI filters and biases of the 1x1 / 3x3-reduce /
    3x3 / 5x5-reduce / 5x5 / pool-projection convolutions.  Returns the channel-concatenated output
    ``[1x1 | 3x3 | 5x5 | pool-proj]``."""
    ws = params[0::2]
    if _cuda_ok(x, ws):
        return _InceptFn.apply(x, *params)
    from . import functional as F_
    w1, b1, wr3, br3, w3, b3, wr5, br5, w5, b5, wpj, bpj = params
    a = F_.conv2d_bias_act(x, w1, b1, 1, 0, 1, True)
    b = F_.conv2d_bias_act(F_.conv2d_bias_act(x, wr3, br3, 1, 0, 1, True), w3, b3, 1, 1, 1, True)
    c = F_.conv2d_bias_act(F_.conv2d_bias_act(x, wr5, br5, 1, 0, 1, True), w5, b5, 1, 2, 1, True)
    d = F_.conv2d_bias_act(F_.pool2d(x, 3, 1, 1, "max"), wpj, bpj, 1, 0, 1, True)
    return torch.cat([a, b, c, d], dim=-1)
