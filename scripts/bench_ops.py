"""Secondary measurements for SURVEY 8 rows a12-a16 (BASELINE configs 4/5 shapes): roipool3d, IoU matrices, NMS --
this repo's kernels next to the reference's own kernels (oracle/_ref), CUDA events, inputs resident on the device.
Prints one JSON object."""
import json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np, torch
import synth
from oracle import refgpu as R
from pointrcnn_b200.ext import iou3d_cuda, roipool3d_cuda
from pointrcnn_b200.iou3d import iou3d_utils

dev = torch.device("cuda:0")
peaks = {"hbm_gbs": 3350.0}   # H100 SXM data sheet (700 W card)
flush = torch.empty(256 * 1024 * 1024 // 4, device=dev)


def timeit(fn, iters=10, warm=3, sync_each=False):
    for _ in range(warm): fn()
    torch.cuda.synchronize()
    tot = 0.0
    for _ in range(iters):
        flush.fill_(0.0)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    return tot / iters


out = {}
# ---- C4: roipool3d, B=4, 16384 pts, 512 RoIs, 130 feature channels, 512 samples
B, N, M, C, S = 4, 16384, 512, 130, 512
rng = np.random.default_rng(0)
xyz = synth.u_kitti(B, N, 40)
boxes = np.stack([synth.boxes3d(M, 41 + b)[0] for b in range(B)]).astype(np.float32)
for b in range(B):   # RoIs sit on points, pooled with the 1 m context margin the RCNN stage uses
    pick = rng.integers(0, N, M)
    boxes[b, :, 0], boxes[b, :, 2], boxes[b, :, 1] = xyz[b, pick, 0], xyz[b, pick, 2], xyz[b, pick, 1] + 0.8
    boxes[b, :, 3:6] += 2.0; boxes[b, :, 1] += 1.0
x, bx = torch.from_numpy(xyz).to(dev), torch.from_numpy(boxes).to(dev)
f = torch.randn(B, N, C, device=dev)
pooled = torch.zeros((B, M, S, 3 + C), device=dev); empty = torch.zeros((B, M), dtype=torch.int32, device=dev)
ms = timeit(lambda: roipool3d_cuda.forward(x, bx, f, pooled, empty))
ms_c = timeit(lambda: roipool3d_cuda.forward(x, bx, f, pooled, empty, bx))
ms_1p = timeit(lambda: roipool3d_cuda.forward_one_pass(x, bx, f, pooled, empty))
ms_memset = timeit(lambda: pooled.zero_())
from pointrcnn_b200.roipool3d import roipool3d_utils
ms_util = timeit(lambda: roipool3d_utils.roipool3d_gpu(x, f, bx, 0.0, S))
ms_ref = timeit(lambda: R.roipool3d(x, f, bx, S), iters=5)
alg = (B * N * C * 4 + B * N * 12 + B * M * S * (3 + C) * 4)
nonempty = int((empty == 0).sum())
out["roipool3d_C4"] = {"ms": ms, "ms_with_canonical": ms_c, "ms_one_pass_kernel": ms_1p, "ms_memset_of_output": ms_memset,
                       "ms_roipool3d_gpu_wrapper_incl_alloc": ms_util, "ms_reference_kernels": ms_ref, "speedup": ms_ref / ms,
                       "algorithmic_MB": alg / 1e6, "achieved_GBs": alg / ms / 1e6, "peak_GBs": peaks["hbm_gbs"],
                       "frac": alg / ms / 1e6 / peaks["hbm_gbs"], "non_empty_boxes": nonempty, "of": B * M}
# ---- NMS (C++-boundary semantics: sorted boxes in, keep list on the host out)
for n, thr, normal in ((6300, 0.8, True), (2700, 0.8, True), (1000, 0.3, False), (100, 0.1, False)):
    bev = torch.from_numpy(synth.sorted_bev(n, 50 + n)).to(dev)
    keep = torch.zeros(n, dtype=torch.int64)
    fn = (iou3d_cuda.nms_normal_gpu if normal else iou3d_cuda.nms_gpu)
    ms = timeit(lambda: fn(bev, keep, thr))
    ms_ref = timeit(lambda: R.nms(bev, thr, normal), iters=5)
    out["nms_%s_%d" % ("normal" if normal else "rotated", n)] = {"ms": ms, "ms_reference": ms_ref, "speedup": ms_ref / ms}
# ---- IoU matrices
b3, _ = synth.boxes3d(2048, 60)
a5 = torch.from_numpy(synth.to_bev(b3[:512])).to(dev); b5 = torch.from_numpy(synth.to_bev(b3[512:])).to(dev)
o = torch.zeros((512, 1536), device=dev)
ms = timeit(lambda: iou3d_cuda.boxes_iou_bev_gpu(a5, b5, o))
ms_ref = timeit(lambda: R.boxes_iou_bev(a5, b5), iters=5)
out["boxes_iou_bev_512x1536"] = {"ms": ms, "ms_reference": ms_ref, "speedup": ms_ref / ms}
print(json.dumps(out))
