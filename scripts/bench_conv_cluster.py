"""Operand-bandwidth check of the implicit-GEMM convolutions on the AlexNet-128b passes, and the bytes 2-CTA clusters would save.

For each of the 14 AlexNet-128b convolution passes (fprop, dgrad, wgrad; two-group layers as one launch, the shapes of
``gemm_probe.py``) it prints:

* ``normal``: the kernel time with L2 flushed (``gemm_probe.timeit``), in us;
* ``load``: the same launch with ``gemm_set_debug(4)`` (no MMAs: the TMA loads and barrier hand-offs only) and its share
  of ``normal``.  A pass whose load-only time is close to its normal time is bound by moving its operands, not by wgmma;
* ``TF``: issued TFLOP/s (the MACs the wgmmas issue under the tile plan, zero fill included);
* ``GB`` / ``TB/s``: the operand bytes TMA moves from L2 into shared memory under the tile plan, and the rate they imply;
* the 2-CTA pairing plan (``axis``: M pairs tiles that share the weight / activation B tile, N pairs tiles that share the A
  tile) and the bytes it saves.

The card's name, power limit and the SM clock sampled during the timed passes are printed with the table.

What it showed on an H100 SXM (700 W, SM clock 1980 MHz): the load-only time is 91 % of the normal time summed over the 14
passes (70-97 % per pass), at an implied 5.5 TB/s of L2->SMEM operand traffic, so the passes are bound by feeding their
operands.  Pairing tiles in 2-CTA clusters and multicasting the shared half-boxes cuts that traffic by 19 % (the ``saved``
column), but a bit-exact implementation of it (each CTA loading half the shared box, both CTAs' consumers releasing every
ring slot, rings in lock step) was 1.7 % SLOWER per pass sum and 0.05 ms slower per bench.py step: the bound is the
per-k-block load and hand-off latency of each CTA, not L2 bandwidth, and the cluster coupling adds to that latency.
The fixed costs of a tile matter as much: with ``gemm_set_debug(7)`` (no loads and no MMAs) the passes still took 45 % of
their time.  Hoisting the epilogue's per-column bias loads to the start of each tile (DESIGN §3) cut the fprop passes by
10-18 %.  The ``normal`` column after that change sums to 1460 us, against 1550 us before it.

    python scripts/bench_conv_cluster.py [--rounds 3] [--plan-only]

``--plan-only`` prints the byte arithmetic alone (host code of the extension, no GPU needed).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SMS = 132                                                    # H100 SXM
# (name, batch, H, W, C per group, O per group, k, stride, pad, groups, dgrad): gemm_probe.py's AlexNet-128b conv layers
LAYERS = [
    ("conv1", 128, 57, 57, 48, 96, 3, 1, 0, 1, False),
    ("conv2", 128, 27, 27, 48, 128, 5, 1, 2, 2, True),
    ("conv3", 128, 13, 13, 256, 384, 3, 1, 1, 1, True),
    ("conv4", 128, 13, 13, 192, 192, 3, 1, 1, 2, True),
    ("conv5", 128, 13, 13, 192, 128, 3, 1, 1, 2, True),
]
AXES = {0: "none", 1: "M", 2: "N"}


def cdiv(a, b):
    return -(-a // b)


def passes():
    """(layer, pass, kind, M, N, Cg, taps, groups) of every pass in ``gemm_probe.issued_macs``'s convention."""
    out = []
    for name, B, H, W, C, O, k, s, p, G, dgrad in LAYERS:
        Ho = (H + 2 * p - k) // s + 1
        M = B * Ho * Ho
        out.append((name, "fprop", 0, M, O, C, k * k, G))
        if dgrad:
            out.append((name, "dgrad", 1, M, C, O, k * k, G))
        out.append((name, "wgrad", 2, O, M, C, k * k, G))
    return out


def launch_geometry(L, kind, M, N, Cg, taps, groups, sms=SMS, f32=False):
    """The launch the host code plans for one pass: GEMM rows / columns, k-blocks, (BN, MT, splits), and the bytes per k-block
    of each operand of a tile.  Returns a dict."""
    BK, ATOM = (32, 32) if f32 else (64, 64)
    if kind == 2:                                            # wgrad: rows = out-channels, columns = (tap, chunk) boxes
        boxes = taps * cdiv(Cg, ATOM)
        num_kb = cdiv(N, BK)
        bn, mt, splits = L.gemm_plan_conv(2, M, boxes * ATOM, groups, num_kb, 0, sms)
        nbox = bn // ATOM
        mtiles, ntiles = cdiv(M, 128), cdiv(boxes, nbox)
        a_bytes = lambda mti: 128 * 128
        b_bytes = lambda nti: min(nbox, boxes - nti * nbox) * BK * 128
    else:
        num_kb = taps * cdiv(Cg, BK)
        bn, mt, splits = L.gemm_plan_conv(kind, M, N, groups, num_kb, 0 if (f32 and kind == 1) else 1, sms)
        mtiles, ntiles = cdiv(M, mt * 128), cdiv(N, bn)
        a_bytes = lambda mti: (2 if (mt == 2 and mti * 256 + 128 < M) else 1) * 128 * 128
        b_bytes = lambda nti: bn * 128
    kb_per = cdiv(num_kb, splits)
    splits = cdiv(num_kb, kb_per)
    kb = lambda s: min(num_kb, (s + 1) * kb_per) - s * kb_per
    return dict(kind=kind, N=boxes * ATOM if kind == 2 else N, num_kb=num_kb, bn=bn, mt=mt, splits=splits, mtiles=mtiles, ntiles=ntiles,
                groups=groups, kb=kb, a_bytes=a_bytes, b_bytes=b_bytes)


def tile_order(g, axis):
    """Tiles (group, split, mti, nti) in the order the kernel walks them: m fastest, except n fastest when pairing along N."""
    out = []
    for grp in range(g["groups"]):
        for s in range(g["splits"]):
            for i in range(g["mtiles"] * g["ntiles"]):
                if axis == 2:
                    out.append((grp, s, i // g["ntiles"], i % g["ntiles"]))
                else:
                    out.append((grp, s, i % g["mtiles"], i // g["mtiles"]))
    return out


def operand_bytes(g, axis):
    """(bytes TMA moves into shared memory, bytes of it saved by pairing) for one launch: tiles (2q, 2q + 1) of the walk form a
    pair; a pair on the same group and split whose two tiles share the n-tile (axis M) or the m-tile (axis N) loads the shared
    operand once for both CTAs."""
    tiles = tile_order(g, axis)
    total = saved = 0
    for t in tiles:
        total += g["kb"](t[1]) * (g["a_bytes"](t[2]) + g["b_bytes"](t[3]))
    if axis:
        for q in range(len(tiles) // 2):
            t0, t1 = tiles[2 * q], tiles[2 * q + 1]
            if t0[:2] == t1[:2] and t0[4 - axis] == t1[4 - axis]:
                saved += g["kb"](t0[1]) * (g["b_bytes"](t0[3]) if axis == 1 else g["a_bytes"](t0[2]))
    return total, saved


def pair_plan(g, clusters, sms=SMS):
    """Pairing axis of a 2-CTA cluster launch: the axis with the most
    bytes saved (wgrad: N only), or none when nothing is saved or the paired launch would need more waves than the unicast one."""
    n = g["groups"] * g["splits"] * g["mtiles"] * g["ntiles"]
    if clusters <= 0 or cdiv(cdiv(n, 2), clusters) > cdiv(n, sms):
        return 0
    best, best_saved = 0, 0
    for axis in ((2,) if g["kind"] == 2 else (1, 2)):
        saved = operand_bytes(g, axis)[1]
        if saved > best_saved:
            best, best_saved = axis, saved
    return best


def plan_rows(L, clusters, sms=SMS):
    rows = []
    for layer, kind_name, kind, M, N, Cg, taps, G in passes():
        g = launch_geometry(L, kind, M, N, Cg, taps, G, sms)
        axis = pair_plan(g, clusters, sms)
        total, saved = operand_bytes(g, axis)
        best_saved = max(operand_bytes(g, a)[1] for a in ((2,) if kind == 2 else (1, 2)))
        rows.append(dict(name="%s %s" % (layer, kind_name), kind=kind, M=M, N=N, Cg=Cg, taps=taps, groups=G,
                         tile="%dx%d" % (g["bn"], 128 * g["mt"]), splits=g["splits"], tiles=len(tile_order(g, 0)),
                         axis=AXES[axis], bytes=total, saved=saved, best_saved=best_saved))
    return rows


def smi(q):
    r = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], stdout=subprocess.PIPE, text=True)
    return r.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3, help="timings per pass (median reported)")
    ap.add_argument("--plan-only", action="store_true")
    ap.add_argument("--clusters", type=int, default=0, help="--plan-only: 2-CTA clusters that fit at once (default SMS / 2)")
    ap.add_argument("--json", default="", help="also write the rows to this file")
    args = ap.parse_args()

    if args.plan_only:
        from theanompi_b200.ops import native
        L = native.lib()
        assert L is not None, native.load_error()
        rows = plan_rows(L, args.clusters or SMS // 2)
        print("%-14s %8s %6s %5s %4s %8s %8s %6s" % ("pass", "tile", "splits", "tiles", "axis", "GB", "saved", "best"))
        for r in rows:
            print("%-14s %8s %6d %5d %4s %8.3f %7.1f%% %5.1f%%" % (r["name"], r["tile"], r["splits"], r["tiles"], r["axis"], r["bytes"] / 1e9,
                                                                100.0 * r["saved"] / r["bytes"], 100.0 * r["best_saved"] / r["bytes"]))
        tb = sum(r["bytes"] for r in rows)
        ts = sum(r["saved"] for r in rows)
        print("total %.3f GB, paired %.3f GB (-%.1f %%)" % (tb / 1e9, (tb - ts) / 1e9, 100.0 * ts / tb))
        return

    import torch
    from scripts import gemm_probe as gp
    from bench import ClockSampler
    L = gp.L
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    rows = plan_rows(L, sms // 2, sms)
    fns = {}
    for layer in LAYERS:
        name, B, H, W, C, O, k, s, p, G, dgrad = layer
        for case_name, fn, useful, issued in gp.conv_case(name, B, H, W, C, O, k, s, p, groups=G, dgrad=dgrad):
            fns[case_name.split(" ")[0] + " " + case_name.split(" ")[-1]] = (fn, useful, issued)
    print("gpu: %s | sms %d" % (smi("name,power.limit,clocks.max.sm"), sms), flush=True)
    sampler = ClockSampler(torch.cuda.current_device())
    sampler.start()
    for r in rows:
        fn, useful, issued = fns[r["name"]]
        r["useful"], r["issued"] = useful, issued
        L.gemm_set_debug(0)
        r["normal"] = statistics.median(gp.timeit(fn) for _ in range(args.rounds))
        L.gemm_set_debug(4)
        r["load"] = gp.timeit(fn)
        L.gemm_set_debug(0)
    clocks = sampler.stop()
    print("SM clock during the passes: %s MHz median (max %s), throttle reasons %s; %s" % (
        clocks.get("sm_mhz"), clocks.get("sm_max_mhz"), clocks.get("reasons"), smi("name,power.limit")))
    hdr = "%-13s %9s %6s %5s %4s | %8s %8s %5s | %6s %7s %6s %6s" % (
        "pass", "tile", "splits", "tiles", "axis", "normal", "load", "load%", "TF", "GB", "TB/s", "saved")
    print(hdr)
    sums = dict(normal=0.0, load=0.0)
    for r in rows:
        t = r["normal"]
        line = "%-13s %9s %6d %5d %4s | %8.1f %8.1f %4.0f%% | %6.1f %7.3f %6.2f %5.1f%%" % (
            r["name"], r["tile"], r["splits"], r["tiles"], r["axis"], t, r["load"], 100.0 * r["load"] / t,
            2.0 * (r["issued"] or r["useful"]) / t / 1e6, r["bytes"] / 1e9, r["bytes"] / t / 1e6, 100.0 * r["saved"] / r["bytes"])
        sums["normal"] += t
        sums["load"] += r["load"]
        print(line)
    tb = sum(r["bytes"] for r in rows)
    ts = sum(r["saved"] for r in rows)
    print("sum: normal %.1f us, load-only %.1f us (%.0f %%); operand bytes %.3f GB -> %.2f TB/s; pairing saves %.1f %% of them"
          % (sums["normal"], sums["load"], 100.0 * sums["load"] / sums["normal"], tb / 1e9, tb / sums["normal"] / 1e6, 100.0 * ts / tb))
    if args.json:
        for r in rows:
            r.pop("kind", None)
        with open(args.json, "w") as f:
            json.dump(dict(gpu=smi("name,power.limit"), clocks=clocks, rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
