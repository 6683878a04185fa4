"""BASELINE configs[3]: RCNN stage-2 -- roipool3d on 512 proposals/scene x 512 points (+ canonical transform) + the RCNN
PointNet++ stack (xyz_up / merge, 3 SA modules, cls / reg heads; tools/cfgs/default.yaml:78-110), batch 4, 1 GPU.
Synthetic RPN outputs (uniform KITTI-scope points, N(0,1) features, proposals sitting on points).  Prints one JSON object."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import synth  # noqa: E402
from pointrcnn_b200 import prof  # noqa: E402
from pointrcnn_b200.rcnn.stage import RCNNStage  # noqa: E402


def make_inputs(dev, B=4, N=16384, M=512, seed=70):
    rng = np.random.default_rng(seed)
    xyz = synth.u_kitti(B, N, seed)
    boxes = np.stack([synth.boxes3d(M, seed + 1 + b)[0] for b in range(B)]).astype(np.float32)
    for b in range(B):          # RoIs sit on points (as RPN proposals do)
        pick = rng.integers(0, N, M)
        boxes[b, :, 0], boxes[b, :, 2], boxes[b, :, 1] = xyz[b, pick, 0], xyz[b, pick, 2], xyz[b, pick, 1] + 0.8
    x = torch.from_numpy(xyz).to(dev)
    return dict(rpn_xyz=x, rpn_features=torch.randn(B, N, 128, device=dev), seg_mask=(torch.rand(B, N, device=dev) > 0.5).float(),
                pts_depth=torch.norm(x, p=2, dim=2), roi_boxes3d=torch.from_numpy(boxes).to(dev))


def flops_per_roi(net):
    c = net.cfg
    f = 512 * sum(a * b for a, b in zip([net.rcnn_input_channel] + c["XYZ_UP_LAYER"][:-1], c["XYZ_UP_LAYER"]))
    f += 512 * 2 * c["XYZ_UP_LAYER"][-1] * c["XYZ_UP_LAYER"][-1]
    npts = [512] + [n if n != -1 else 1 for n in c["NPOINTS"]]
    cin = 128
    for k, mlp in enumerate(c["MLPS"]):
        rows = npts[k + 1] * (c["NSAMPLE"][k] if c["NPOINTS"][k] != -1 else npts[k])
        dims = [cin + 3] + list(mlp)
        f += rows * sum(a * b for a, b in zip(dims[:-1], dims[1:]))
        cin = mlp[-1]
    for fc in (c["CLS_FC"] + [1], c["REG_FC"] + [net.reg_channel]):
        dims = [cin] + list(fc)
        f += sum(a * b for a, b in zip(dims[:-1], dims[1:]))
    return 2 * f


def measure(dev, steps=10, warm=5):
    torch.manual_seed(0)
    net = RCNNStage().to(dev).eval()
    inp = make_inputs(dev)
    B, M = inp["roi_boxes3d"].shape[:2]
    flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)
    peaks = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}   # H100 SXM data sheet (700 W card), dense
    with torch.no_grad():
        for _ in range(warm):
            net(inp)
        torch.cuda.synchronize()
        t_pool = t_net = 0.0
        mallocs0 = torch.cuda.memory_stats(dev).get("num_device_alloc", 0)
        prof.enable()
        for _ in range(steps):
            flush.fill_(0.0)
            a, b, c = (torch.cuda.Event(enable_timing=True) for _ in range(3))
            a.record()
            pts_input, empty = net.pool(inp["rpn_xyz"], inp["rpn_features"], inp["seg_mask"], inp["pts_depth"], inp["roi_boxes3d"])
            b.record()
            cls, reg = net.forward_pts(pts_input)
            c.record()
            torch.cuda.synchronize()
            t_pool += a.elapsed_time(b)
            t_net += b.elapsed_time(c)
            n_nonempty, checksum = int((empty == 0).sum()), float(cls.double().mean() + reg.double().mean())
            del pts_input, empty, cls, reg       # the next step's 558 MB pooled block reuses this one (no cudaMalloc in the loop)
        prof.disable()
        mallocs = torch.cuda.memory_stats(dev).get("num_device_alloc", 0) - mallocs0
    fam = {k: v[0] / steps for k, v in prof.collect().items()}
    t_pool /= steps
    t_net /= steps
    N, C = inp["rpn_xyz"].shape[1], 130
    pool_bytes = B * N * C * 4 + B * N * 12 + B * M * 512 * (3 + C) * 4
    fl = flops_per_roi(net) * B * M
    out = {"config": "BASELINE configs[3]: B=%d scenes x %d RoIs x 512 points, 130 pooled channels" % (B, M),
           "ms_roipool3d_incl_feature_cat": t_pool, "ms_rcnn_net": t_net, "ms_total": t_pool + t_net,
           "rois_per_s": B * M / ((t_pool + t_net) * 1e-3), "scenes_per_s": B / ((t_pool + t_net) * 1e-3),
           "roipool3d": {"algorithmic_MB": pool_bytes / 1e6, "achieved_GBs_incl_cat": pool_bytes / t_pool / 1e6, "peak_GBs": peaks["hbm_gbs"]},
           "rcnn_net": {"algorithmic_TFLOP": fl / 1e12, "achieved_TFLOPs": fl / t_net / 1e9, "peak_TFLOPs_tf32": peaks["bf16_tflops"] / 2,
                        "frac": fl / t_net / 1e9 / (peaks["bf16_tflops"] / 2)},
           "families_ms": fam, "non_empty_rois": n_nonempty, "checksum": checksum, "cudaMallocs_in_timed_loop": mallocs}
    return out


if __name__ == "__main__":
    print(json.dumps(measure(torch.device("cuda", 0))))
