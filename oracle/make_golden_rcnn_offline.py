"""oracle/make_golden_rcnn_offline.py -- golden vectors for offline RCNN training samples.

Runs the reference's OWN lib/datasets/kitti_rcnn_dataset.py (get_rcnn_training_sample_batch, imported unchanged from
/root/reference through dropin.activate(compat=True)) on small synthetic scenes (oracle/rcnn_offline.py::synth_scene) whose
RPN features and proposals are written to a temporary directory the way tools/eval_rcnn.py --save_rpn_feature and the
proposal writer leave them, and writes tests/golden/rcnn_offline.npz.  TEST INFRASTRUCTURE ONLY.
    python oracle/make_golden_rcnn_offline.py

Stand-ins:
  - kitti_utils.get_iou3d needs shapely, which is not installed: oracle/gt_paste.py::iou3d (exact float64 clip) replaces it;
  - the dataset object is built without the KITTI tree (labels come from memory);
  - aug_roi_by_noise_batch and roipool3d_cpu are wrapped to record what they see: the wrapper calls the reference's
    aug_roi_by_noise_batch one row at a time (its rows are independent and draw in row order, so the stream is the same)
    and counts the IoU calls of each row (its jitter tries);
  - save_rpn_features is taken from tools/eval_rcnn.py's source (that module parses the command line when imported).
The fg-only branch cannot come from here: kitti_rcnn_dataset.py:923 calls torch.from_numpy(...).type_as(<ndarray>), which
raises.  The oracle implements what the line evidently means, and the tests cover that branch against the device only.
"""
import ast
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"

# (synth seed, kind, REG_AUG_METHOD); one np.random stream over the runs, in this order
RUNS = [(11, "mixed", "multiple"), (12, "hard", "multiple"), (13, "easy", "single"), (14, "bg", "normal"), (15, "mixed", "normal"),
        (16, "mixed", "single")]
SEED = 2026
CFG = dict(ROI_PER_IMAGE=32, NUM_POINTS=32)
FILE_SCENE = (21, 64, 5)        # (seed, points, features) of the save_rpn_features byte check
KEYS = ("pts_input", "pts_features", "cls_label", "reg_valid_mask", "gt_boxes3d_ct", "roi_boxes3d", "gt_boxes3d")


def fmt(v):
    return repr(float(v))


def label_line(cls, box, score=None):
    x, y, z, h, w, l, ry = box
    vals = [cls, "0.00", "0", "-10", "0.0", "0.0", "100.0", "100.0"] + [fmt(v) for v in (h, w, l, x, y, z, ry)]
    return " ".join(vals + ([fmt(score)] if score is not None else []))


def save_rpn_features_fn():
    src = open(os.path.join(REF, "tools", "eval_rcnn.py")).read()
    node = next(n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name == "save_rpn_features")
    ns = dict(os=os, np=np)
    exec(compile(ast.Module(body=[node], type_ignores=[]), "eval_rcnn.py", "exec"), ns)
    return ns["save_rpn_features"]


def file_scene():
    seed, n, c = FILE_SCENE
    rng = np.random.default_rng(seed)
    return dict(seg=(rng.random(n) < 0.4).astype(np.float32), rawscore=rng.standard_normal(n).astype(np.float32),
                pts_features=rng.random((n, 1)).astype(np.float32), xyz=rng.standard_normal((n, 3)).astype(np.float32),
                features=rng.standard_normal((c, n)).astype(np.float32))


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, REF)
    from pointrcnn_b200 import dropin
    dropin.activate(compat=True)
    import lib.datasets.kitti_rcnn_dataset as K
    from lib.config import cfg
    from lib.utils import kitti_utils, object3d
    from oracle import gt_paste as GP
    from oracle import rcnn_offline as RO
    cfg.INCLUDE_SIMILAR_TYPE, cfg.PC_REDUCE_BY_RANGE = False, False
    cfg.AUG_DATA, cfg.AUG_METHOD_LIST, cfg.AUG_METHOD_PROB, cfg.AUG_ROT_RANGE = True, ["rotation", "scaling", "flip"], [1.0, 1.0, 0.5], 18
    for k, v in dict(RO.CFG, **CFG).items():
        if not k.startswith("AUG"):
            setattr(cfg.RCNN, k, v)
    cfg.RCNN.USE_SEG_SCORE = False
    calls = []

    def iou3d(a, b, need_bev=False):
        calls.append(1)
        return GP.iou3d(a, b)
    kitti_utils.get_iou3d = iou3d

    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        feat_dir, roi_dir = os.path.join(tmp, "features"), os.path.join(tmp, "rois")
        os.makedirs(feat_dir)
        os.makedirs(roi_dir)
        scenes = {}
        for sid, (seed, kind, _) in enumerate(RUNS):
            s = RO.synth_scene(seed, kind)
            scenes[sid] = s
            for suffix, v in (("", s["rpn_features"]), ("_xyz", s["rpn_xyz"]), ("_intensity", s["rpn_intensity"]), ("_seg", s["seg_mask"])):
                np.save(os.path.join(feat_dir, "%06d%s.npy" % (sid, suffix)), v)
            with open(os.path.join(roi_dir, "%06d.txt" % sid), "w") as f:
                f.write("\n".join(label_line("Car", b, 0.5) for b in s["roi_boxes3d"]) + "\n")

        ds = object.__new__(K.KittiRCNNDataset)
        ds.mode, ds.classes = "TRAIN", ("Background", "Car")
        ds.sample_id_list = list(range(len(RUNS)))
        ds.rcnn_training_feature_dir, ds.rcnn_training_roi_dir = feat_dir, roi_dir
        ds.get_label = lambda sid: [object3d.Object3d(label_line("Car", b)) for b in scenes[sid]["gt_boxes3d"]]
        record = {}
        orig_aug = ds.aug_roi_by_noise_batch

        def aug_rows(roi_boxes3d, gt_boxes3d, aug_times=10):
            ious, tries = [], []
            record.setdefault("src", []).append(roi_boxes3d.copy())
            record.setdefault("gt", []).append(gt_boxes3d.copy())
            for k in range(len(roi_boxes3d)):
                n0 = len(calls)
                ious.append(orig_aug(roi_boxes3d[k:k + 1], gt_boxes3d[k:k + 1], aug_times=aug_times)[1])
                tries.append(len(calls) - n0)
            record.setdefault("tries", []).append(np.array(tries))
            record.setdefault("iou", []).append(np.concatenate(ious))
            record.setdefault("rois", []).append(roi_boxes3d.copy())
            return roi_boxes3d, np.concatenate(ious)
        ds.aug_roi_by_noise_batch = aug_rows
        orig_pool = K.roipool3d_utils.roipool3d_cpu

        def pool(*a, **kw):
            r = orig_pool(*a, **kw)
            record["pool"] = [np.array(v, copy=True) for v in r]
            return r
        K.roipool3d_utils.roipool3d_cpu = pool

        np.random.seed(SEED)
        for i, (seed, kind, method) in enumerate(RUNS):
            cfg.RCNN.REG_AUG_METHOD = method
            record.clear()
            r = ds.get_rcnn_training_sample_batch(i)
            s = scenes[i]
            src = np.concatenate(record["src"])
            gts = np.concatenate(record["gt"])
            sel_src = np.array([np.nonzero((s["roi_boxes3d"] == b).all(1))[0][0] for b in src], np.int32)
            sel_gt = np.array([np.nonzero((s["gt_boxes3d"] == b).all(1))[0][0] for b in gts], np.int32)
            out["run%d_sel" % i] = np.stack([sel_src, sel_gt, np.concatenate(record["tries"])], 1).astype(np.int32)
            out["run%d_iou" % i] = np.concatenate(record["iou"]).astype(np.float32)
            out["run%d_rois" % i] = np.concatenate(record["rois"]).astype(np.float32)
            out["run%d_pooled_input" % i], out["run%d_pooled_features" % i], out["run%d_empty" % i] = record["pool"]
            for k in KEYS:
                out["run%d_%s" % (i, k)] = np.asarray(r[k])
            t = out["run%d_sel" % i][:, 2]
            print("run %d (%s, %s): fg rows %d, tries %s, empty %d, cls %s" % (
                i, kind, method, int((t > 1).sum()), np.bincount(t).tolist(), int(out["run%d_empty" % i].sum()),
                np.bincount(r["cls_label"] + 1).tolist()))
        out["rng_state"] = np.random.get_state()[1]

        fs = file_scene()
        save_rpn_features_fn()(fs["seg"], fs["rawscore"], fs["pts_features"], fs["xyz"], fs["features"].T, tmp, 7)
        for suffix in ("", "_xyz", "_seg", "_intensity", "_rawscore"):
            with open(os.path.join(tmp, "%06d%s.npy" % (7, suffix)), "rb") as f:
                out["file%s" % (suffix or "_features")] = np.frombuffer(f.read(), np.uint8)
    path = os.path.join(ROOT, "tests", "golden", "rcnn_offline.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
