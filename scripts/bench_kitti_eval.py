"""Time the device KITTI AP evaluation on a synthetic split the size of KITTI val.

    python scripts/bench_kitti_eval.py [--images 3769] [--repeats 5] [--oracle-images 100] [--out result.json]

The split: 3769 images with about as many label rows per image as KITTI's (Car / Van / Pedestrian / Cyclist / DontCare)
and about 30 detections per image, added batch by batch (8 scenes per batch, the evaluation loop's batch) through
KittiEvaluator.add_batch.  Reports the median wall time of result() (device stages + the one device-to-host copy), the
add_batch time per batch, the library's launch count per result(), the card's name and power limit, and for context the
numpy oracle's time on a subset of the images (CPU, not comparable to the GPU number).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def synth(n_img, seed=0):
    """GT annotation dicts (~7 rows per image, one in six DontCare, about KITTI's label mix) and (n_img, 40, 7) detection
    boxes, most of them near a GT box, with ~30 selected per image"""
    from oracle import kitti_eval as OK
    rng = np.random.default_rng(seed)
    gts, _ = OK.synth_split(seed, n_img, 14, 0, classes=("Car",) * 6 + ("Van", "Pedestrian", "Pedestrian", "Cyclist", "DontCare", "DontCare"))
    m = 40
    det = np.zeros((n_img, m, 7), np.float32)
    det[..., 0] = rng.uniform(-20, 20, (n_img, m))
    det[..., 1] = rng.uniform(1.4, 2.0, (n_img, m))
    det[..., 2] = rng.uniform(5, 60, (n_img, m))
    det[..., 3:6] = np.array([1.5, 1.6, 3.9], np.float32) * rng.uniform(0.4, 1.1, (n_img, m, 1))
    det[..., 6] = rng.uniform(-np.pi, np.pi, (n_img, m))
    for k, g in enumerate(gts):                 # most detections near a GT box
        n = len(g["name"])
        if n:
            src = rng.integers(0, n, m)
            near = rng.random(m) < 0.7
            loc, dim = g["location"][src], g["dimensions"][src]
            det[k, near, 0:3] = (loc + rng.normal(0, 0.2, (m, 3)))[near]
            det[k, near, 3], det[k, near, 4], det[k, near, 5] = dim[near, 1], dim[near, 2], dim[near, 0]
            det[k, near, 6] = g["rotation_y"][src][near]
    scores = rng.normal(0, 2, (n_img, m)).astype(np.float32)
    select = rng.random((n_img, m)) < 0.75
    return gts, det, scores, select


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=3769)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--oracle-images", type=int, default=100)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from oracle import kitti_eval as OK
    from oracle import kitti_io as KO
    from pointrcnn_b200 import _cabi as C
    from pointrcnn_b200.datasets import kitti_eval as KE
    from pointrcnn_b200.datasets.kitti_rcnn_dataset import Calibration
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_eval: needs a CUDA device")
    dev = torch.device("cuda:0")
    gts, det, scores, select = synth(a.images)
    B = 8
    P2 = torch.from_numpy(np.stack([Calibration(KO.CALIB).P2] * B).astype(np.float32)).to(dev)
    hw = torch.tensor([KO.IMG_SHAPE[:2]] * B, dtype=torch.float32, device=dev)
    bx, sc, se = torch.from_numpy(det).to(dev), torch.from_numpy(scores).to(dev), torch.from_numpy(select).to(dev)

    def fill(ev):
        for b0 in range(0, a.images, B):
            n = min(B, a.images - b0)
            ev.add_batch(list(range(b0, b0 + n)), bx[b0:b0 + n], sc[b0:b0 + n], se[b0:b0 + n], P2[:n], hw[:n])

    ev = KE.KittiEvaluator(gts, [0, 1, 2], dev)
    fill(ev)                                     # warm-up: allocation, module load
    r = ev.result()
    torch.cuda.synchronize()
    add_ms = []
    for _ in range(a.repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fill(ev)
        torch.cuda.synchronize()
        add_ms.append((time.perf_counter() - t0) * 1e3 / ((a.images + B - 1) // B))
    res_ms, launches = [], []
    for _ in range(a.repeats):
        torch.cuda.synchronize()
        l0 = C.launch_count()
        t0 = time.perf_counter()
        r = ev.result()                           # ends in the device-to-host copy
        res_ms.append((time.perf_counter() - t0) * 1e3)
        launches.append(C.launch_count() - l0)
    n_dt = int(ev._dt_count.sum().item())
    sub = min(a.oracle_images, a.images)
    # the oracle evaluates the same detections, read back from the device table
    table = ev._dt.cpu().numpy()
    counts = ev._dt_count.cpu().numpy()
    dt_annos = []
    for k in range(sub):
        t = table[k, :counts[k]]
        dt_annos.append(dict(name=np.array(["Car"] * len(t)), truncated=t[:, 5], occluded=t[:, 6], alpha=t[:, 4], bbox=t[:, 0:4],
                             dimensions=t[:, 7:10], location=t[:, 10:13], rotation_y=t[:, 13], score=t[:, 14]))
    t0 = time.perf_counter()
    OK.evaluate(gts[:sub], dt_annos, [0, 1, 2])
    oracle_s = time.perf_counter() - t0
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    out = dict(images=a.images, gt_rows=int(sum(len(g["name"]) for g in gts)), detections=n_dt, classes=[0, 1, 2],
               result_ms_median=float(np.median(res_ms)), result_ms=[round(x, 3) for x in res_ms],
               add_batch_ms_per_batch_of_8=float(np.median(add_ms)), launches_per_result=launches[0],
               cpu_oracle_s=round(oracle_s, 2), cpu_oracle_images=sub, gpu=torch.cuda.get_device_name(0),
               nvidia_smi=smi.stdout.strip(), car_moderate_3d_ap=float(r.ret_dict["Car_3d_moderate"]))
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
