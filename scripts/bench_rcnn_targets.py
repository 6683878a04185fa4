"""RCNN target layer of the in-network recipe (ROI_SAMPLE_JIT): ProposalTargetLayer with draw="torch" (the reference's random
calls: host reads per step, a per-scene loop, up to ROI_FG_AUG_TIMES jitter rounds) against draw="device" (csrc/rcnn_sample.cu),
at B = 4 and 16 scenes of 16384 points with 128 RPN features, 512 TRAIN proposals and 64 sampled RoIs each; and
RCNNTrainer.step (fixed RPN + targets + RCNN forward / backward + Adam) with either target layer at B = 2.  Per call: time
(CUDA events around a window that ends in a synchronise), and from a separate profiled call the kernel launches and the
host synchronisations (cudaStreamSynchronize / cudaDeviceSynchronize calls; every .item() / .tolist() makes one).  Prints
one JSON line with the card name and power limit read in the same run.
    python scripts/bench_rcnn_targets.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import synth  # noqa: E402
from oracle import rcnn_offline as RO  # noqa: E402
from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler  # noqa: E402
from pointrcnn_b200.rpn.proposal_target_layer import ProposalTargetLayer  # noqa: E402


def scene(seed, n_pts=16384, n_feat=128, n_roi=512, n_gt=8):
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


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return round(start.elapsed_time(end) / steps, 3)


def _profiled(fn):
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        fn()
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    launches = sum(1 for n in names if n in ("cudaLaunchKernel", "cuLaunchKernel", "cudaLaunchKernelExC", "cuLaunchKernelEx"))
    syncs = sum(1 for n in names if n in ("cudaStreamSynchronize", "cudaDeviceSynchronize"))
    return launches, syncs


def counted(fn):
    """-> (kernel launches, host synchronisations) of one call: the profiled call minus an empty profiled window (the
    closing synchronise and whatever the profiler adds itself)"""
    base = _profiled(lambda: None)
    got = _profiled(fn)
    return got[0] - base[0], got[1] - base[1]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    res = dict(workload="rcnn target layer (ROI_SAMPLE_JIT)", points=16384, features=128, proposals=512, rois_per_scene=64, pooled_points=512)
    smp = RCNNOfflineSampler(device=dev)
    pool = [scene(s) for s in range(16)]
    np.random.seed(0)
    torch.manual_seed(0)
    with torch.no_grad():
        for B in (4, 16):
            batch = smp.prepare_jit_batch(pool[:B])
            for draw in ("torch", "device"):
                layer = ProposalTargetLayer(draw=draw)
                res["ms_b%d_%s" % (B, draw)] = timed(lambda: layer(batch), a.steps, a.warmup)
                res["launches_b%d_%s" % (B, draw)], res["host_syncs_b%d_%s" % (B, draw)] = counted(lambda: layer(batch))
    # the training step with the RPN fixed, both target layers (tests/test_gpu_train.py's set-up at B = 2)
    from pointrcnn_b200.train.step import RCNNTrainer
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 321, channels=4)).to(dev)
    for draw in ("torch", "device"):
        tr = RCNNTrainer(input_channels=1, device=dev, seed=5, target_draw=draw)
        with torch.no_grad():
            tr.rpn.rpn_reg_layer[-1].conv.weight.mul_(0.2)
            rois = tr.rpn_outputs(pc, None)["roi_boxes3d"]
        gt = torch.zeros((2, 12, 7), device=dev)
        gt[:, :8] = rois[:, ::40][:, :8]
        res["train_step_ms_b2_%s" % draw] = timed(lambda: tr.step(pc, gt, grad_norm_clip=1.0), a.steps, a.warmup)
        res["train_step_launches_b2_%s" % draw], res["train_step_host_syncs_b2_%s" % draw] = counted(lambda: tr.step(pc, gt, grad_norm_clip=1.0))
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
