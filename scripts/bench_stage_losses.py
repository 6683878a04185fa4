"""Stage losses: the torch mirror (train.losses, impl="torch": boolean-mask selections, dozens of small kernels forward and
backward) against the device path (impl="device", csrc/stage_loss.cu), as loss forward + backward at the RPN size
(B = 16 x 16384 points, 76 channels, about 3 % foreground) and the RCNN size (R = 256 = 4 x 64 RoIs, 46 channels), and
inside RPNTrainer.step (B = 2) and RCNNTrainer.step_jit with the device target layer (B = 2).  Per call: time (CUDA
events around a window that ends in a synchronise), and from a separate profiled call the kernel launches and the host
synchronisations (cudaStreamSynchronize / cudaDeviceSynchronize calls).  Prints one JSON line with the card name and power
limit read in the same run.
    python scripts/bench_stage_losses.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import synth  # noqa: E402
from bench_rcnn_targets import card, counted, timed  # noqa: E402
from oracle import rcnn_offline as RO  # noqa: E402
from pointrcnn_b200.rpn.stage import CLS_MEAN_SIZE  # noqa: E402
from pointrcnn_b200.train import losses as L  # noqa: E402


def rpn_batch(dev, B=16, N=16384, C=76, seed=0):
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(B, N, 1, generator=g)
    reg = torch.randn(B, N, C, generator=g) * 0.5
    lab = (torch.rand(B, N, generator=g) < 0.03).long()
    lab[torch.rand(B, N, generator=g) < 0.01] = -1
    rl = torch.randn(B, N, 7, generator=g) * torch.tensor([1.2, 0.3, 1.2, 0.15, 0.15, 0.4, 1.5]) + torch.tensor([0, 0, 0, 1.5, 1.6, 3.9, 0.0])
    return [t.to(dev) for t in (cls, reg, lab, rl)]


def rcnn_batch(dev, R=256, C=46, seed=1):
    g = torch.Generator().manual_seed(seed)
    cls = torch.randn(R, 1, generator=g)
    reg = torch.randn(R, C, generator=g) * 0.5
    lab = torch.randint(-1, 2, (R,), generator=g)
    valid = ((lab == 1) & (torch.rand(R, generator=g) < 0.8)).long()
    roi = torch.randn(R, 7, generator=g) * torch.tensor([10, 1, 20, 0.15, 0.15, 0.4, 1.5]) + torch.tensor([0, 1.6, 30, 1.5, 1.6, 3.9, 0.0])
    gt = torch.randn(R, 7, generator=g) * torch.tensor([0.6, 0.2, 0.6, 0.15, 0.15, 0.4, 0.5]) + torch.tensor([0, 0, 0, 1.5, 1.6, 3.9, 0.0])
    return [t.to(dev) for t in (cls, reg, lab, valid, roi, gt)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    mean = torch.from_numpy(CLS_MEAN_SIZE[0]).to(dev)
    res = dict(workload="stage losses forward + backward", rpn_rows=16 * 16384, rpn_channels=76, rcnn_rows=256, rcnn_channels=46)
    cls, reg, lab, rl = rpn_batch(dev)
    res["rpn_fg_fraction"] = round(float((lab > 0).float().mean()), 4)
    rc, rr, rlab, valid, roi, gt = rcnn_batch(dev)
    cls.requires_grad_(True)
    reg.requires_grad_(True)
    rc.requires_grad_(True)
    rr.requires_grad_(True)
    for impl in ("torch", "device"):
        def rpn():
            total, _ = L.rpn_loss(cls, reg, lab, rl, mean, impl=impl)
            total.backward()

        def rcnn():
            total, _ = L.rcnn_loss(rc, rr, rlab.clamp(min=0), valid, roi, gt, mean, impl=impl)
            total.backward()
        res["rpn_loss_ms_%s" % impl] = timed(rpn, a.steps, a.warmup)
        res["rpn_loss_launches_%s" % impl], res["rpn_loss_host_syncs_%s" % impl] = counted(rpn)
        res["rcnn_loss_ms_%s" % impl] = timed(rcnn, a.steps, a.warmup)
        res["rcnn_loss_launches_%s" % impl], res["rcnn_loss_host_syncs_%s" % impl] = counted(rcnn)
    # RPNTrainer.step at B = 2 (tests/test_gpu_train.py's set-up)
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, synthetic_labels
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 123, channels=4)).to(dev)
    pl, rg = synthetic_labels(pc, seed=1)
    for impl in ("torch", "device"):
        tr = RPNTrainer(input_channels=1, device=dev, seed=3, loss_impl=impl)
        res["rpn_step_ms_b2_%s" % impl] = timed(lambda: tr.step(pc, pl, rg, grad_norm_clip=1.0), a.steps, a.warmup)
        res["rpn_step_launches_b2_%s" % impl], res["rpn_step_host_syncs_b2_%s" % impl] = counted(lambda: tr.step(pc, pl, rg, grad_norm_clip=1.0))
    # RCNNTrainer.step_jit with the device target layer at B = 2, on saved-feature scenes
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    np.random.seed(0)
    batch = RCNNOfflineSampler(device=dev).prepare_jit_batch([RO.synth_scene(s, "mixed", n_pts=16384, n_feat=128) for s in (0, 1)])
    for impl in ("torch", "device"):
        tr = RCNNTrainer(input_channels=1, device=dev, seed=5, target_draw="device", loss_impl=impl)
        res["rcnn_step_jit_ms_b2_%s" % impl] = timed(lambda: tr.step_jit(batch), a.steps, a.warmup)
        res["rcnn_step_jit_launches_b2_%s" % impl], res["rcnn_step_jit_host_syncs_b2_%s" % impl] = counted(lambda: tr.step_jit(batch))
    res["card"] = card()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
