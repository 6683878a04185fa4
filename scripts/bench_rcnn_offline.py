"""Offline RCNN training samples (datasets/rcnn_offline.py): time of RCNNOfflineSampler.prepare_batch on the device at the
recipe's batch size (4) and at 16, each scene 16384 points with 128 RPN features and 300 proposals (TEST.RPN_POST_NMS_TOP_N
= 300, what the README saves for train_aug), plus per batch: the library's launches, every device operation (kernels, copies and memsets of the library and of torch's
packing of device-resident input, counted in a separate profiled call) and the host synchronisations and the time per
scene of the numpy oracle in the reference's mode (oracle/rcnn_offline.py, draw "numpy", IoU "exact"), which stands in for
the reference's loader (it needs shapely).  Prints one JSON line with the card name and power limit read in the same run.
    python scripts/bench_rcnn_offline.py [--steps 20] [--oracle-scenes 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import rcnn_offline as RO  # noqa: E402
from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler  # noqa: E402


def scene(seed, n_pts=16384, n_feat=128, n_roi=300, n_gt=8):
    s = RO.synth_scene(seed, "mixed", n_pts=n_pts, n_feat=n_feat, n_gt=n_gt)
    rng = np.random.default_rng(seed)
    rois = s["roi_boxes3d"]
    extra = rois[rng.integers(0, len(rois), n_roi - len(rois))].copy()
    extra[:, [0, 2]] += rng.normal(0, 0.8, (len(extra), 2)).astype(np.float32)
    s["roi_boxes3d"] = np.concatenate([rois, extra]).astype(np.float32)
    return s


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def time_batch(smp, scenes, steps, warmup):
    for i in range(warmup):
        smp.prepare_batch(scenes, seed=i)
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(steps):
        smp.prepare_batch(scenes, seed=100 + i)
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--oracle-scenes", type=int, default=2)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    smp = RCNNOfflineSampler(device=dev)
    res = dict(workload="rcnn_offline prepare_batch", points=16384, features=128, proposals=300, rois_per_scene=64, pooled_points=512)
    pool = [scene(s) for s in range(16)]
    for B in (4, 16):
        host = pool[:B]
        on_dev = [{k: torch.from_numpy(np.ascontiguousarray(v)).to(dev) for k, v in s.items()} for s in host]
        res["ms_per_batch_b%d_numpy_input" % B] = round(time_batch(smp, host, a.steps, a.warmup), 3)
        res["ms_per_batch_b%d_device_input" % B] = round(time_batch(smp, on_dev, a.steps, a.warmup), 3)
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            lc = C.launch_count()
            smp.prepare_batch(on_dev, seed=1)
            res["library_launches_per_batch_b%d" % B] = C.launch_count() - lc
            res["host_syncs_per_batch_b%d" % B] = 0          # set_sync_debug_mode("error") raises on any synchronising call
        finally:
            torch.cuda.set_sync_debug_mode(0)
        for name, scenes in (("device_input", on_dev), ("numpy_input", host)):
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                smp.prepare_batch(scenes, seed=2)
                torch.cuda.synchronize()
            res["device_ops_per_batch_b%d_%s" % (B, name)] = sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    t = time.perf_counter()
    np.random.seed(0)
    for s in pool[:a.oracle_scenes]:
        RO.sample_scene(s, dict(NUM_POINTS=512, ROI_PER_IMAGE=64), draw="numpy", iou="exact", rng=np.random)
    res["oracle_numpy_exact_s_per_scene"] = round((time.perf_counter() - t) / a.oracle_scenes, 3)
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
