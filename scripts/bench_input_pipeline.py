"""input pipeline / KITTI output (SURVEY 8(f) rank 4): a batch of 16 raw scans of ~120 k points -> network input + RPN labels on
the device (pinned host scans, H2D inside the timed region) against the per-scene numpy path (oracle/kitti_io.py, one host
thread, the reference's order of operations with exact-geometry labels -- the reference's Delaunay labels are slower still).
The paste_* fields time the same batch with GT-paste augmentation from a synthetic 400-entry database."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch
from oracle import gt_paste as GP
from oracle import kitti_io as KO
from pointrcnn_b200.datasets.kitti_rcnn_dataset import RPNInputPipeline
from pointrcnn_b200.datasets import kitti_output

dev = torch.device("cuda:0")
B, RAW, NPOINTS = 16, 120000, 16384
scans = []
for i in range(B):
    lidar, gt, alpha = KO.synth_scan(500 + i, RAW, 8)
    scans.append(dict(lidar=torch.from_numpy(lidar).pin_memory(), calib=KO.CALIB, img_shape=KO.IMG_SHAPE, gt_boxes3d=gt, gt_alpha=alpha))
res = {"batch": B, "raw_points_per_scan": int(scans[0]["lidar"].shape[0]), "npoints": NPOINTS}
pipe = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=dev)
for _ in range(3):
    out = pipe.prepare_batch(scans, seed=1)
torch.cuda.synchronize()
ts = []
for it in range(10):
    t0 = time.perf_counter()
    out = pipe.prepare_batch(scans, seed=it)
    torch.cuda.synchronize()
    ts.append(time.perf_counter() - t0)
ts.sort()
res["device_ms_per_batch"] = 1e3 * ts[len(ts) // 2]
res["device_scenes_per_s"] = B / ts[len(ts) // 2]
res["valid_points"] = out["valid_counts"][:, 0].tolist()
res["fg_points"] = int((out["rpn_cls_label"] == 1).sum())
# device-only part (inputs resident): events
from pointrcnn_b200 import _cabi as C
lc0 = C.launch_count()
pipe.prepare_batch(scans, seed=0)
res["launches_per_batch"] = C.launch_count() - lc0
# host path, one thread
rng = np.random.RandomState(0)
t0 = time.perf_counter()
for s in scans[:4]:
    KO.rpn_sample(s["lidar"].numpy(), KO.CALIB, KO.IMG_SHAPE, s["gt_boxes3d"], s["gt_alpha"], NPOINTS, rng, train=True)
host = (time.perf_counter() - t0) / 4
res["numpy_ms_per_scene"] = 1e3 * host
res["numpy_scenes_per_s"] = 1.0 / host
res["speedup_vs_numpy_thread"] = res["device_scenes_per_s"] * host
# GT-paste leg: the same scans with a synthetic database (default.yaml's GT_AUG_* settings), device draw
from pointrcnn_b200.datasets.kitti_rcnn_dataset import GTDatabase
db = GP.synth_gt_database(31, 400)
gdb = GTDatabase.from_arrays(np.stack([e["gt_box3d"] for e in db]), [np.concatenate([e["points"], e["intensity"][:, None]], 1) for e in db],
                             np.array([e["alpha"] for e in db], np.float32))
plane = GP.road_plane()
for s in scans:
    s["road_plane"] = plane
paste = RPNInputPipeline(npoints=NPOINTS, mode="TRAIN", draw="device", device=dev, gt_database=gdb)
for _ in range(3):
    out = paste.prepare_batch(scans, seed=1)
torch.cuda.synchronize()
ts = []
for it in range(10):
    t0 = time.perf_counter()
    out = paste.prepare_batch(scans, seed=it)
    torch.cuda.synchronize()
    ts.append(time.perf_counter() - t0)
ts.sort()
res["paste_device_ms_per_batch"] = 1e3 * ts[len(ts) // 2]
res["paste_pasted_objects_per_scene"] = float(out["gt_paste"]["stats"][:, 0].float().mean())
lc0 = C.launch_count()
paste.prepare_batch(scans, seed=0)
res["paste_launches_per_batch"] = C.launch_count() - lc0
# the device stages alone (CUDA events around one batch; host candidate draw excluded)
ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
torch.cuda.synchronize()
ev[0].record(); pipe.prepare_batch(scans, seed=0); ev[1].record()
ev[2].record(); paste.prepare_batch(scans, seed=0); ev[3].record()
torch.cuda.synchronize()
res["gpu_ms_span_without_paste"] = ev[0].elapsed_time(ev[1])
res["gpu_ms_span_with_paste"] = ev[2].elapsed_time(ev[3])
t0 = time.perf_counter()
for b in range(B):
    paste._draw_candidates(scans[b:b + 1], b, np.random)
res["paste_host_draw_ms_per_batch"] = 1e3 * (time.perf_counter() - t0)
# the numpy restatement of apply_gt_aug_to_one_scene + get_rpn_sample (shapely replaced by the exact clip)
rng = np.random.RandomState(0)
t0 = time.perf_counter()
for s in scans[:4]:
    GP.rpn_sample_with_paste(s["lidar"].numpy(), KO.CALIB, KO.IMG_SHAPE, s["gt_boxes3d"], s["gt_alpha"], NPOINTS, rng, train=True, gt_db=db,
                             road_plane=plane)
host = (time.perf_counter() - t0) / 4
res["paste_numpy_ms_per_scene"] = 1e3 * host
res["paste_speedup_vs_numpy_thread"] = B / (res["paste_device_ms_per_batch"] / 1e3) * host
# KITTI output: 100 detections per scene
det_rng = np.random.default_rng(3)
boxes = np.concatenate([s["gt_boxes3d"] for s in scans])[det_rng.integers(0, 8 * B, 100)] + det_rng.normal(0, 0.1, (100, 7)).astype(np.float32)
boxes_t, scores_t = torch.from_numpy(boxes.astype(np.float32)).to(dev), torch.randn(100, device=dev)
import tempfile
with tempfile.TemporaryDirectory() as d:
    for _ in range(3):
        kitti_output.save_kitti_format(1, KO.CALIB, boxes_t, d, scores_t, KO.IMG_SHAPE)
    t0 = time.perf_counter()
    for i in range(50):
        kitti_output.save_kitti_format(i, KO.CALIB, boxes_t, d, scores_t, KO.IMG_SHAPE)
    res["save_kitti_ms_per_scene"] = 1e3 * (time.perf_counter() - t0) / 50
    t0 = time.perf_counter()
    for i in range(10):
        open(os.path.join(d, "x%d.txt" % i), "w").write(KO.kitti_lines(boxes.astype(np.float32), scores_t.cpu().numpy(), KO.CALIB["P2"], KO.IMG_SHAPE))
    res["numpy_save_kitti_ms_per_scene"] = 1e3 * (time.perf_counter() - t0) / 10
print(json.dumps(res))
os.makedirs(os.path.join(ROOT, "gpurun_out"), exist_ok=True)
json.dump(res, open(os.path.join(ROOT, "gpurun_out", "r2_input_pipeline.json"), "w"), indent=1)
