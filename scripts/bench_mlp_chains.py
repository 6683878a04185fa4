"""Time every MLP chain launch of the RPN backbone forward at B = 16 x 16384 points, resident weights against streamed.

    python scripts/bench_mlp_chains.py [--iters 20] [--reps 5] [--json OUT]

One eval forward runs with the chain entry points wrapped: each call is timed where it happens, with its real inputs,
under `prb_options.mlp_resident = 1` (resident where the chain fits, the default) and `= 0` (always streamed), the two
settings alternated `--reps` times after a warm-up, `--iters` back-to-back launches per CUDA-event window.  Per launch it
prints the median ms of each setting, TF/s over padded MACs (rows x K padded to 32 x N padded to 32, summed over layers)
and the L2 weight traffic the streaming kernel needs (every 64-row tile reads the whole packed image).
Then each chain call runs once more under torch.profiler, and every kernel it launches is listed with its device time:
the gather, the fused segments and each layer wider than 256 on mlp_wide_kernel, which gets its TF/s over padded MACs
and the L2 bytes its tiles read (per 128-row tile and column block, every K chunk of A, 16 KB, and of the column
block's weights).
Random weights, synthetic scenes: the work is that of a real batch.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth  # noqa: E402
from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.backbone import Pointnet2MSG  # noqa: E402

TM, KC = 64, 32
WM, WN = 128, 256     # mlp_wide_kernel's tile rows and widest column block


def _ru(a, b):
    return (a + b - 1) // b * b


def geometry(segs, c_out):
    """padded K and N of every layer, as chain_geometry packs them"""
    ks, ns = [], []
    for l, co in enumerate(c_out):
        ks.append(sum(_ru(s, KC) for s in segs) if l == 0 else ns[-1])
        ns.append(_ru(co, 32))
    return ks, ns


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # the numbers still stand; say the card could not be read
        q = "%s (nvidia-smi: %s)" % (torch.cuda.get_device_name(0), e)
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mlp_chains: needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = C.lib()
    results = []

    def timed(name, fn, cargs, label, rows, segs, c_out):
        def launch():
            C.check(fn(*cargs), name)
        for resident in (1, 0):                 # warm both kernels at this shape
            with C.options(mlp_resident=resident):
                for _ in range(2):
                    launch()
        ms = {1: [], 0: []}
        for _ in range(args.reps):
            for resident in (1, 0):
                with C.options(mlp_resident=resident):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record()
                    for _ in range(args.iters):
                        launch()
                    b.record()
                    b.synchronize()
                    ms[resident].append(a.elapsed_time(b) / args.iters)
        ks, ns = geometry(segs, c_out)
        macs = rows * sum(k * n for k, n in zip(ks, ns))
        image = sum(k * n for k, n in zip(ks, ns)) * 4
        tiles = (rows + TM - 1) // TM
        r = dict(chain=label, rows=rows, image_kb=image / 1024, stream_l2_mb=tiles * image / 1e6,
                 resident_ms=statistics.median(ms[1]), stream_ms=statistics.median(ms[0]),
                 resident_spread_ms=max(ms[1]) - min(ms[1]), stream_spread_ms=max(ms[0]) - min(ms[0]))
        r["resident_tfs"] = 2 * macs / (r["resident_ms"] * 1e-3) / 1e12
        r["stream_tfs"] = 2 * macs / (r["stream_ms"] * 1e-3) / 1e12
        r["launches"] = launches(launch, rows, ks, ns)
        results.append(r)

    def launches(launch, rows, ks, ns):
        """(kernel, ms per call, and for a wide layer TF/s and L2 MB) of every kernel one call launches, in order"""
        torch.cuda.synchronize()
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.iters):
                launch()
            torch.cuda.synchronize()
        evs = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "mlp_" in e.name),
                     key=lambda e: e.time_range.start)
        per = len(evs) // args.iters
        wide = [(k, n) for k, n in zip(ks, ns) if n > WN]
        out = []
        for i in range(per):
            name = evs[i].name.split("(")[0].replace("void ", "")
            ms = statistics.median(e.device_time_total for e in evs[i::per]) / 1e3
            row = dict(kernel=name, ms=ms)
            if "mlp_wide_kernel" in name and wide:
                k, n = wide.pop(0)
                bw = 32 * ((n // 32 + 1) // 2)     # two column blocks of equal width
                blocks = [min(bw, n - c) for c in range(0, n, bw)]
                row["layer"] = "%d->%d" % (k, n)
                row["tfs"] = 2 * rows * k * n / (ms * 1e-3) / 1e12
                row["l2_mb"] = _ru(rows, WM) // WM * (k // KC) * sum(WM * KC * 4 + b * KC * 4 for b in blocks) / 1e6
            out.append(row)
        return out

    def c_out_of(d):
        return [d.c_out[i] for i in range(d.num_layers)]

    sa, fp, rows_fn = lib.prb_sa_group_mlp_max_ws, lib.prb_fp_interp_mlp_ws, lib.prb_mlp_rows2

    class Wrap:
        """stands in for the CDLL while the forward runs: the three chain entry points are timed, the rest pass through"""
        def __getattr__(self, k):
            return getattr(lib, k)

        def prb_sa_group_mlp_max_ws(self, *a):
            B, N, npoint, ns, c_feat = (int(v) for v in a[:5])
            d = a[9]._obj
            co = c_out_of(d)
            segs = [3 + c_feat] if 0 < c_feat <= 5 else ([c_feat, 3] if c_feat else [3])
            timed("sa", sa, a, "sa %dx%d [%d]+%s" % (B * npoint, ns, 3 + c_feat, co), B * npoint * ns, segs, co)
            return sa(*a)

        def prb_fp_interp_mlp_ws(self, *a):
            B, n, m, c_known, c_skip = (int(v) for v in a[:5])
            d = a[9]._obj
            co = c_out_of(d)
            timed("fp", fp, a, "fp %d [%d+%d]+%s" % (B * n, c_known, c_skip, co), B * n, [c_known] + ([c_skip] if c_skip else []), co)
            return fp(*a)

        def prb_mlp_rows2(self, *a):
            rws, c_a, c_b = a[0].value, int(a[1]), int(a[4])
            d = a[7]._obj
            co = c_out_of(d)
            timed("rows", rows_fn, a, "rows %d [%d+%d]+%s" % (rws, c_a, c_b, co), rws, [c_a] + ([c_b] if c_b else []), co)
            return rows_fn(*a)

    torch.manual_seed(0)
    net = Pointnet2MSG(input_channels=1).to(dev).eval()
    x = torch.from_numpy(synth.u_kitti(16, 16384, 7, channels=4)).to(dev)
    with torch.no_grad():
        net(x)                                   # packs the weights, warms everything else
        torch.cuda.synchronize()
        C._lib = Wrap()
        try:
            net(x)
        finally:
            C._lib = lib
        torch.cuda.synchronize()

    print("card: %s; iters %d x reps %d per setting, alternated" % (card(), args.iters, args.reps))
    print("%-34s %8s %8s %9s %9s %7s %7s %9s %12s" % ("chain launch", "res ms", "str ms", "res sprd", "str sprd", "res TF/s",
                                                    "str TF/s", "image KB", "str L2 MB"))
    tot = {1: 0.0, 0: 0.0}
    for r in results:
        print("%-34s %8.4f %8.4f %9.4f %9.4f %7.1f %7.1f %9.0f %12.0f" % (
            r["chain"], r["resident_ms"], r["stream_ms"], r["resident_spread_ms"], r["stream_spread_ms"], r["resident_tfs"],
            r["stream_tfs"], r["image_kb"], r["stream_l2_mb"]))
        tot[1] += r["resident_ms"]
        tot[0] += r["stream_ms"]
    print("total: resident-where-fits %.3f ms, streamed %.3f ms" % (tot[1], tot[0]))
    print("\nkernels per chain call (default options, torch.profiler device time, median of %d calls)" % args.iters)
    for r in results:
        for i, k in enumerate(r["launches"]):
            extra = ("  layer %-9s %6.1f TF/s  L2 %7.1f MB" % (k["layer"], k["tfs"], k["l2_mb"])) if "tfs" in k else ""
            print("%-34s %-44s %8.4f ms%s" % (r["chain"] if i == 0 else "", k["kernel"][:44], k["ms"], extra))
    if args.json:
        with open(args.json, "w") as f:
            json.dump(dict(card=card(), results=results), f, indent=1)


if __name__ == "__main__":
    main()
