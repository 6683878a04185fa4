"""oracle/make_golden_gt_paste.py -- golden vectors for GT-paste augmentation in the RPN input pipeline.

Runs the reference's OWN lib/datasets/kitti_rcnn_dataset.py (get_rpn_sample with apply_gt_aug_to_one_scene, imported
unchanged from /root/reference) with cfg.GT_AUG_ENABLED = True and the GT settings of tools/cfgs/default.yaml
(GT_EXTRA_NUM 15, GT_AUG_RAND_NUM, GT_AUG_APPLY_PROB 1.0, GT_AUG_HARD_RATIO 0.6) on synthetic scans
(oracle/kitti_io.py::synth_scan) and a synthetic database (oracle/gt_paste.py::synth_gt_database), and writes
tests/golden/gt_paste.npz.  TEST INFRASTRUCTURE ONLY.
    python oracle/make_golden_gt_paste.py

Stand-ins, each for something that is not part of this environment or that would make the vectors depend on call history:
  - kitti_utils.get_iou3d needs shapely, a third-party package that is not installed: it is replaced by
    oracle/gt_paste.py::iou3d, the same 3D IoU with an exact float64 convex-polygon clip for the bottom-face overlap;
  - the database is a fresh copy per scene and every read of an entry's 'obj' returns a copy: the reference moves the
    shared obj.pos in place on every draw, so from an entry's second draw on its label box drifts from its points;
  - get_road_plane returns a slightly tilted plane (oracle/gt_paste.py::road_plane);
  - the labels hold a Pedestrian and a DontCare row besides the cars: the collision list (every class but DontCare)
    and the label list (Car) differ.
"""
import copy
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, REF)

NPOINTS = 4096
DB_SEED, DB_SIZE = 31, 40
# (seed, raw points, GT cars): a subsampled scene, a crowded one (candidates rejected), one with fewer valid points than NPOINTS
SCENES = [(21, 30000, 4), (22, 30000, 16), (23, 2500, 2)]
SEED = 2025


def fmt(v):
    return repr(float(v))


def label_line(cls, box, alpha):
    x, y, z, h, w, l, ry = box
    return " ".join([cls, "0.00", "0", fmt(alpha), "100.0", "100.0", "200.0", "200.0"] + [fmt(v) for v in (h, w, l, x, y, z, ry)])


def extra_labels(seed):
    """a Pedestrian (collision box, not a label box) and a DontCare row (neither)"""
    rng = np.random.default_rng(seed + 1000)
    ped = np.array([rng.uniform(-8, 8), 1.7, rng.uniform(12, 30), 1.75, 0.65, 0.9, rng.uniform(-3, 3)], np.float32)
    dc = np.array([3.0, 1.6, 20.0, 1.5, 1.6, 3.9, 0.0], np.float32)
    return ped, dc


class _Entry(dict):
    def __getitem__(self, key):
        v = dict.__getitem__(self, key)
        return copy.deepcopy(v) if key == "obj" else v


def main():
    from pointrcnn_b200 import dropin
    dropin.activate(compat=True)
    import lib.datasets.kitti_rcnn_dataset as K
    from lib.config import cfg
    from lib.utils import calibration, kitti_utils, object3d
    from oracle import gt_paste as GP
    from oracle import kitti_io as KO
    cfg.GT_AUG_ENABLED, cfg.GT_EXTRA_NUM, cfg.GT_AUG_RAND_NUM, cfg.GT_AUG_APPLY_PROB, cfg.GT_AUG_HARD_RATIO = True, 15, True, 1.0, 0.6
    cfg.RPN.ENABLED, cfg.RCNN.ENABLED = True, False
    kitti_utils.get_iou3d = lambda a, b, need_bev=False: GP.iou3d(a, b)

    db = GP.synth_gt_database(DB_SEED, DB_SIZE)
    ref_db = [_Entry(gt_box3d=e["gt_box3d"], points=e["points"], intensity=e["intensity"],
                     obj=object3d.Object3d(label_line("Car", e["gt_box3d"], e["alpha"]))) for e in db]
    plane = GP.road_plane()
    scans = {sid: KO.synth_scan(seed, n, g) for sid, (seed, n, g) in enumerate(SCENES)}

    def labels(sid):
        lidar, gt, alpha = scans[sid]
        ped, dc = extra_labels(SCENES[sid][0])
        return [object3d.Object3d(label_line("Car", b, a)) for b, a in zip(gt, alpha)] + \
            [object3d.Object3d(label_line("Pedestrian", ped, 0.1)), object3d.Object3d(label_line("DontCare", dc, 0.0))]

    ds = object.__new__(K.KittiRCNNDataset)
    ds.mode, ds.npoints, ds.random_select = "TRAIN", NPOINTS, True
    ds.classes = ("Background", "Car")
    ds.sample_id_list = list(range(len(SCENES)))
    ds.get_calib = lambda sid: calibration.Calibration(KO.CALIB)
    ds.get_image_shape = lambda sid: KO.IMG_SHAPE
    ds.get_lidar = lambda sid: scans[sid][0]
    ds.get_label = labels
    ds.get_road_plane = lambda sid: plane.copy()

    out = dict(plane=plane)
    np.random.seed(SEED)
    for i in range(len(SCENES)):
        dbc = [_Entry(dict.items(e)) for e in copy.deepcopy(ref_db)]
        ds.gt_database = [[e for e in dbc if e["points"].shape[0] > 100], [e for e in dbc if e["points"].shape[0] <= 100]]
        s = ds.get_rpn_sample(i)
        for k in ("pts_input", "pts_rect", "pts_features", "rpn_cls_label", "rpn_reg_label", "gt_boxes3d"):
            out["train%d_%s" % (i, k)] = s[k]
        out["train%d_aug" % i] = np.array(repr(s.get("aug_method", [])))
        print("scene %d: %d label boxes (%d cars), %d fg points, aug %s" % (i, len(s["gt_boxes3d"]), SCENES[i][2],
                                                                          int((s["rpn_cls_label"] == 1).sum()), s.get("aug_method")))
    path = os.path.join(ROOT, "tests", "golden", "gt_paste.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, os.path.getsize(path), "bytes")


if __name__ == "__main__":
    main()
