"""Evaluation statistics (datasets/eval_stats.py): time of EvalStats.add_rcnn over a split the size of KITTI val (3769
scenes, 100 proposals each, 0-20 GT boxes), in batches, against the reference's per-scene composition (eval_rcnn.py:
337-367: boxes_iou3d for the refined boxes and the RoIs, the max reductions, the classification-accuracy lines, and their
`.item()` calls), here with the library's prb_boxes_iou3d standing in for boxes_iou3d_gpu.  Also times
RCNNOfflineSampler.prepare_eval_batch against prepare_batch on the same scenes.  Prints one JSON line with the card name
and power limit read in the same run.
    python scripts/bench_eval_stats.py [--scenes 3769] [--batch 16]
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
from pointrcnn_b200.datasets.eval_stats import EvalStats  # noqa: E402
from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def split(n, m, dev, seed=0):
    """n scenes: m proposals around 0-20 GT boxes, refined boxes jittered from the proposals, scores, gt_iou from the kernel"""
    rng = np.random.default_rng(seed)
    G = 20
    gt_count = rng.integers(0, G + 1, n).astype(np.int32)
    gt = np.stack([rng.uniform(-20, 20, (n, G)), rng.uniform(0.5, 2, (n, G)), rng.uniform(5, 60, (n, G)), rng.uniform(1.3, 1.8, (n, G)),
                   rng.uniform(1.4, 1.9, (n, G)), rng.uniform(3.2, 4.8, (n, G)), rng.uniform(-3, 3, (n, G))], -1).astype(np.float32)
    src = gt[np.arange(n)[:, None], rng.integers(0, G, (n, m))]
    rois = (src + rng.normal(0, 1, (n, m, 7)) * np.array([0.4, 0.1, 0.4, 0.1, 0.1, 0.3, 0.2])).astype(np.float32)
    pred = (rois + rng.normal(0, 1, (n, m, 7)) * np.array([0.2, 0.05, 0.2, 0.05, 0.05, 0.1, 0.1])).astype(np.float32)
    t = lambda a: torch.from_numpy(a).to(dev)
    d = dict(gt=t(gt), gt_count=t(gt_count), rois=t(rois), pred=t(pred), pred_cls=t(rng.integers(0, 2, (n, m)).astype(np.int64)),
             select=t(rng.random((n, m)) < 0.05))
    st = EvalStats(device=dev)
    d["gt_iou"] = torch.empty((n, m), device=dev)
    st._recall(d["rois"], None, d["gt"], d["gt_count"], None, None, d["gt_iou"])
    return d


def batched(d, n, batch, dev):
    st = EvalStats(device=dev)
    for i in range(0, n, batch):
        s = slice(i, i + batch)
        st.add_rcnn(d["pred"][s], d["rois"][s], d["gt"][s], d["gt_count"][s], pred_classes=d["pred_cls"][s], gt_iou=d["gt_iou"][s],
                    select=d["select"][s])
    return st.result()


def per_scene(d, n, gt_count_host, dev):
    """eval_one_epoch_rcnn's statistics lines, one scene at a time, with their host round trips"""
    L, stream = C.lib(), C.stream()
    rec, roi_rec, total_gt, acc_sum, acc_r_sum = [0] * 5, [0] * 5, 0, 0.0, 0.0
    for k in range(n):
        g = int(gt_count_host[k])
        gt_iou = d["gt_iou"][k]
        pred_classes = d["pred_cls"][k]
        if g > 0:
            gt = d["gt"][k, :g].contiguous()
            for boxes, out in ((d["pred"][k], rec), (d["rois"][k], roi_rec)):
                iou = torch.empty((boxes.shape[0], g), device=dev)
                C.check(L.prb_boxes_iou3d(1, boxes.shape[0], C.ptr(boxes), g, C.ptr(gt), C.ptr(iou), stream), "boxes_iou3d")
                gt_max_iou, _ = iou.max(dim=0)
                for idx, thresh in enumerate((0.1, 0.3, 0.5, 0.7, 0.9)):
                    out[idx] += (gt_max_iou > thresh).sum().item()
            total_gt += g
        cls_label = (gt_iou > 0.6).float()
        cls_valid_mask = ((gt_iou >= 0.6) | (gt_iou <= 0.45)).float()
        cls_acc = ((pred_classes == cls_label.long()).float() * cls_valid_mask).sum() / max(cls_valid_mask.sum(), 1.0)
        cls_label_refined = (gt_iou >= 0.7).float()
        cls_acc_refined = (pred_classes == cls_label_refined.long()).float().sum() / max(cls_label_refined.shape[0], 1.0)
        acc_sum += cls_acc.item()
        acc_r_sum += cls_acc_refined.item()
    return rec, roi_rec, total_gt, acc_sum, acc_r_sum


def timed(fn, reps=1):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        r = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3, r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", type=int, default=3769)
    ap.add_argument("--proposals", type=int, default=100)
    ap.add_argument("--batch", type=int, default=16)
    ap.add_argument("--pool-batch", type=int, default=4)
    ap.add_argument("--pool-steps", type=int, default=10)
    a = ap.parse_args()
    dev = torch.device("cuda")
    n, m = a.scenes, a.proposals
    d = split(n, m, dev)
    gt_count_host = d["gt_count"].cpu().numpy()
    batched(d, min(n, 64), a.batch, dev)                     # warm-up
    per_scene(d, min(n, 16), gt_count_host, dev)
    t_batched, r = timed(lambda: batched(d, n, a.batch, dev), reps=3)
    t_scene, (rec, roi_rec, total_gt, _, _) = timed(lambda: per_scene(d, n, gt_count_host, dev))
    for key, counts in (("rcnn_recall(thresh=%.2f)", rec), ("rpn_recall(thresh=%.2f)", roi_rec)):   # both paths count the same
        assert [round(r[key % t] * max(total_gt, 1)) for t in (0.1, 0.3, 0.5, 0.7, 0.9)] == counts, key

    # prepare_eval_batch against prepare_batch: device-resident scenes, 16384 points, 128 features, 100 proposals
    scenes = []
    for k in range(a.pool_batch):
        s = RO.synth_scene(50 + k, "mixed", n_pts=16384, n_feat=128, n_gt=8)
        rng = np.random.default_rng(k)
        rois = s["roi_boxes3d"]
        s["roi_boxes3d"] = rois[rng.integers(0, len(rois), m)] + rng.normal(0, 0.5, (m, 7)).astype(np.float32) * np.float32([1, 0, 1, 0, 0, 0, 0])
        s["roi_scores"] = rng.random(m).astype(np.float32)
        scenes.append({k2: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float32)).to(dev) for k2, v in s.items()})
    smp = RCNNOfflineSampler(device=dev)
    smp.prepare_eval_batch(scenes)
    smp.prepare_batch(scenes, seed=0)
    t_eval, _ = timed(lambda: smp.prepare_eval_batch(scenes), reps=a.pool_steps)
    t_train, _ = timed(lambda: smp.prepare_batch(scenes, seed=1), reps=a.pool_steps)
    print(json.dumps({"card": card(), "scenes": n, "proposals": m, "batch": a.batch,
                      "add_rcnn_split_ms": round(t_batched, 3), "per_scene_split_ms": round(t_scene, 3),
                      "per_scene_over_batched": round(t_scene / t_batched, 2),
                      "pool_batch": a.pool_batch, "prepare_eval_batch_ms": round(t_eval, 3), "prepare_batch_ms": round(t_train, 3)}))


if __name__ == "__main__":
    main()
