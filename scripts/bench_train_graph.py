"""Eager vs CUDA-graph training steps: RPNTrainer.step at B = 2, 4, 16 and RCNNTrainer.step at B = 2, 4 (device SA / FP,
loss and target paths; RPN B = 2 also with the SA / FP modules on the torch path), OneCycle Adam, gradient clip 1.0,
eager and graphed alternating, 3 repeats of 10 steps.  Per case: ms per step (median of the repeats, and all repeats),
host launches per step (torch.profiler: kernel and graph launches, memcpy / memset calls of the CUDA runtime and driver),
peak memory, and the time of the call that captures.
Also the GPU-busy fraction of one eager B = 2 RPN step (the union of its kernel intervals over the step's wall time),
from a profiler trace of its own.  Reads the card's name and power limit in the same run.

    python scripts/bench_train_graph.py [--out DIR]      -> one JSON document on stdout (and DIR/bench_train_graph.json)
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import synth  # noqa: E402
from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, synthetic_labels  # noqa: E402

# rpn_torch: the SA / FP modules on the op-by-op torch path (cuDNN MLPs), the trainers' default switches
CASES = [("rpn", 2), ("rpn_torch", 2), ("rpn", 4), ("rpn", 16), ("rcnn", 2), ("rcnn", 4)]
REPEATS, STEPS = 3, 10
LAUNCH_CALLS = ("cudaLaunchKernel", "cuLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernelEx", "cudaGraphLaunch",
                "cudaMemcpyAsync", "cudaMemsetAsync", "cuMemsetD8Async", "cuMemsetD32Async")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(0)


def make(kind, B, graph, dev):
    pc = torch.from_numpy(synth.u_kitti(B, 16384, 123, channels=4)).to(dev)
    common = dict(device=dev, loss_impl="device", optimizer="adam_onecycle", total_steps=10000, cuda_graph=graph)
    if kind.startswith("rpn"):
        sw = "torch" if kind == "rpn_torch" else "device"
        return RPNTrainer(seed=3, sa_train=sw, fp_train=sw, **common), (pc,) + synthetic_labels(pc, seed=1)
    gts = torch.from_numpy(synth.boxes3d(4 * B, 7)[0].reshape(B, 4, 7).copy()).to(dev)
    return RCNNTrainer(seed=5, sa_train="device", target_draw="device", gt_rows=8, **common), (pc, gts)


def run(tr, batch, it0, n):
    for it in range(it0, it0 + n):
        tr.schedule_iteration(it, 0, 10000)
        tr.step(*batch, grad_norm_clip=1.0)
    return it0 + n


def timed(tr, batch, it0):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    it = run(tr, batch, it0, STEPS)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / STEPS, it


def launches(tr, batch, it0):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU]) as prof:
        run(tr, batch, it0, 2)
        torch.cuda.synchronize()
    n = sum(e.count for e in prof.key_averages() if e.key in LAUNCH_CALLS)
    return n / 2, it0 + 2


def busy_fraction(out):
    """one eager B = 2 RPN step under the profiler: union of kernel intervals / wall time of the step"""
    from torch.profiler import ProfilerActivity, profile
    dev = torch.device("cuda:0")
    tr, batch = make("rpn", 2, False, dev)
    it = run(tr, batch, 0, 3)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        t0 = time.perf_counter()
        run(tr, batch, it, 1)
        torch.cuda.synchronize()
        wall = (time.perf_counter() - t0) * 1e6
    if out:
        prof.export_chrome_trace(os.path.join(out, "rpn_b2_eager_step.json"))
    iv = sorted((e.time_range.start, e.time_range.end) for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    busy, cur = 0.0, None
    for s, e in iv:
        if cur is None or s > cur[1]:
            if cur:
                busy += cur[1] - cur[0]
            cur = [s, e]
        else:
            cur[1] = max(cur[1], e)
    if cur:
        busy += cur[1] - cur[0]
    span = (iv[-1][1] - iv[0][0]) if iv else 0.0
    return dict(kernels=len(iv), busy_us=busy, wall_us=wall, busy_over_wall=busy / wall, busy_over_kernel_span=busy / span if span else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_train_graph: no CUDA device")
    if a.out:
        os.makedirs(a.out, exist_ok=True)
    dev = torch.device("cuda:0")
    res = dict(card=card(), repeats=REPEATS, steps=STEPS, cases=[])
    for kind, B in CASES:
        row = dict(trainer=kind, B=B)
        pair = {}
        for name, graph in (("eager", False), ("graph", True)):
            tr, batch = make(kind, B, graph, dev)
            it = run(tr, batch, 0, 1)                          # eager first step (both)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            it = run(tr, batch, it, 1)                         # graph: capture + one replay
            torch.cuda.synchronize()
            row[name + "_second_call_ms"] = (time.perf_counter() - t0) * 1e3
            it = run(tr, batch, it, 2)
            pair[name] = [tr, batch, it]
        times = {"eager": [], "graph": []}
        torch.cuda.reset_peak_memory_stats(dev)
        for _ in range(REPEATS):
            for name in ("eager", "graph"):
                tr, batch, it = pair[name]
                ms, pair[name][2] = timed(tr, batch, it)
                times[name].append(round(ms, 3))
        for name in ("eager", "graph"):
            tr, batch, it = pair[name]
            row[name + "_ms"] = statistics.median(times[name])
            row[name + "_ms_repeats"] = times[name]
            row[name + "_launches_per_step"], pair[name][2] = launches(tr, batch, it)
        row["peak_memory_gb_both"] = torch.cuda.max_memory_allocated(dev) / 1e9
        row["capture_ms"] = row["graph_second_call_ms"] - row["graph_ms"]
        res["cases"].append(row)
        pair.clear()
        torch.cuda.empty_cache()
        for name, graph in (("eager", False), ("graph", True)):         # peak memory of each mode alone
            torch.cuda.reset_peak_memory_stats(dev)
            tr, batch = make(kind, B, graph, dev)
            run(tr, batch, 0, 4)
            torch.cuda.synchronize()
            row[name + "_peak_memory_gb"] = torch.cuda.max_memory_allocated(dev) / 1e9
            del tr, batch
            torch.cuda.empty_cache()
        print(json.dumps(row), flush=True)
    res["rpn_b2_eager_gpu_busy"] = busy_fraction(a.out)
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        with open(os.path.join(a.out, "bench_train_graph.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
