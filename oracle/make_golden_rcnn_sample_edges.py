"""oracle/make_golden_rcnn_sample_edges.py -- golden vectors of the RCNN RoI sampling decisions on the crafted IoU matrices
of tests/rcnn_sample_reference.py (ties, thresholds, NaN / inf / -0.0, every branch, quotas, counts, GT trimming).

Runs the reference's own sampling on the CPU with its IoU function replaced by the crafted matrix:
  loader  lib/datasets/kitti_rcnn_dataset.py::get_rcnn_training_sample_batch (kitti_utils.get_iou3d returns the matrix;
          the RoI and GT boxes come from memory), stopped at its first aug_roi_by_noise_batch call
  layer   lib/rpn/proposal_target_layer.py::sample_rois_for_rcnn (iou3d_utils.boxes_iou3d_gpu returns the matrix's columns
          of the trimmed GT list) with ROI_FG_AUG_TIMES = 0, run to its end
A trace function reads the sampler's locals at two lines: where the branch is chosen (max_overlaps, gt_assignment, the fg,
easy and hard lists, roi_assignment, the trimmed GT count) and where the jitter starts (the sampled fg and bg sources and
their row counts).  The draws themselves are the reference's np.random / torch streams and are not what the tests check.
Writes tests/golden/rcnn_sample_edges.npz, per case and recipe "<case>.<recipe>.<key>", with <key>.raises where the
reference stops (empty lists reduced by numpy, pdb.set_trace, the loader's fg-only line 923, the layer's all-zero GT list).
TEST INFRASTRUCTURE ONLY.   python oracle/make_golden_rcnn_sample_edges.py
"""
import inspect
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import rcnn_sample_reference as RS  # noqa: E402

REF = "/root/reference"
GOLDEN = os.path.join(ROOT, "tests", "golden", "rcnn_sample_edges.npz")
SEED = 11
BRANCH_LINE = "if fg_num_rois > 0 and bg_num_rois > 0:"
JITTER_LINE = "roi_list, roi_iou_list, roi_gt_list = [], [], []"
BRANCH_KEYS = ("max_overlaps", "gt_assignment", "fg_inds", "easy_bg_inds", "hard_bg_inds", "roi_assignment", "cur_gt")
JITTER_KEYS = ("fg_inds", "bg_inds", "fg_rois_per_this_image", "bg_rois_per_this_image")


class Stop(Exception):
    pass


def _np(v):
    return v.detach().cpu().numpy() if torch.is_tensor(v) else np.asarray(v)


def traced(fn, call):
    """runs call() and returns (dict of the locals at BRANCH_LINE and JITTER_LINE of fn, the exception or None)"""
    src, first = inspect.getsourcelines(fn)
    lines = {first + i: tag for i, s in enumerate(src) for tag, mark in (("branch", BRANCH_LINE), ("jitter", JITTER_LINE))
             if s.strip() == mark}
    assert sorted(lines.values()) == ["branch", "jitter"], lines
    seen = {}

    def local(frame, event, arg):
        tag = lines.get(frame.f_lineno) if event == "line" else None
        if tag:
            keys = BRANCH_KEYS if tag == "branch" else JITTER_KEYS
            seen[tag] = {k: _np(frame.f_locals[k]) for k in keys if k in frame.f_locals}
        return local

    def glob(frame, event, arg):
        return local if frame.f_code is fn.__code__ else None
    sys.settrace(glob)
    try:
        call()
        err = None
    except Exception as e:           # noqa: BLE001 -- every stop of the reference is recorded
        err = e
    finally:
        sys.settrace(None)
    return seen, err


def install():
    from oracle import oracle as O
    from pointrcnn_b200 import dropin
    dropin._install_compat()
    sys.path.insert(0, REF)
    cur = {}
    iou_stub = types.ModuleType("lib.utils.iou3d.iou3d_utils")
    iou_stub.boxes_iou3d_gpu = lambda a, b: torch.from_numpy(cur["iou"][:, :b.shape[0]].copy())
    rp_stub = types.ModuleType("lib.utils.roipool3d.roipool3d_utils")
    rp_stub.roipool3d_gpu = None
    rp_stub.roipool3d_cpu = None
    import lib.utils  # noqa: F401
    for name, mod in (("lib.utils.iou3d", None), ("lib.utils.iou3d.iou3d_utils", iou_stub), ("lib.utils.roipool3d", None),
                      ("lib.utils.roipool3d.roipool3d_utils", rp_stub)):
        if mod is None:
            mod = types.ModuleType(name)
            mod.__path__ = []
        sys.modules[name] = mod
    sys.modules["lib.utils.iou3d"].iou3d_utils = iou_stub
    sys.modules["lib.utils.roipool3d"].roipool3d_utils = rp_stub
    from lib.config import cfg, cfg_from_file
    cfg_from_file(os.path.join(REF, "tools/cfgs/default.yaml"))
    cfg.RCNN.ROI_FG_AUG_TIMES = 0
    cfg.AUG_DATA = False
    import lib.datasets.kitti_rcnn_dataset as K
    from lib.rpn.proposal_target_layer import ProposalTargetLayer
    K.kitti_utils.get_iou3d = lambda a, b, need_bev=False: cur["iou"].copy()
    K.kitti_utils.get_objects_from_label = lambda path: "rois"
    K.kitti_utils.objs_to_boxes3d = lambda objs: cur[objs].copy()
    ds = object.__new__(K.KittiRCNNDataset)
    ds.mode, ds.classes, ds.sample_id_list = "TRAIN", ("Background", "Car"), [0]
    ds.rcnn_training_feature_dir = ds.rcnn_training_roi_dir = "/nonexistent"
    z = np.zeros((1, 3), np.float32)
    ds.get_rpn_features = lambda d, sid: (z, z, z[:, 0], z[:, 0])
    ds.get_label = lambda sid: "gts"
    ds.filtrate_objects = lambda objs: objs

    def stop(*a, **kw):
        raise Stop()
    ds.aug_roi_by_noise_batch = stop
    import pdb
    pdb.set_trace = stop                       # the reference's "no fg and no bg" branch
    del O
    return cfg, cur, ds, ProposalTargetLayer()


def main():
    cfg, cur, ds, layer = install()
    defaults = {k: getattr(cfg.RCNN, k) for k in ("ROI_PER_IMAGE", "HARD_BG_RATIO", "CLS_BG_THRESH", "CLS_BG_THRESH_LO")}
    out = {}
    np.random.seed(SEED)
    torch.manual_seed(SEED)
    for case in RS.cases():
        for k, v in dict(defaults, ROI_PER_IMAGE=case["R"], **case["cfg"]).items():
            setattr(cfg.RCNN, k, v)
        r, t, M = RS.scene(case)
        n = r.shape[0] if case["roi_count"] is None else case["roi_count"]
        ng = t.shape[0] if case["gt_count"] is None else case["gt_count"]
        # the loader reads exactly its n RoIs and ng GT boxes
        cur.update(rois=r[:n], gts=t[:ng], iou=M[:n, :ng])
        seen, err = traced(type(ds).get_rcnn_training_sample_batch, lambda: ds.get_rcnn_training_sample_batch(0))
        _store(out, case["name"] + ".loader", seen, err)
        # the layer sees every row and trims the GT list itself
        cur.update(iou=M)
        res = {}

        def run_layer():
            res["out"] = layer.sample_rois_for_rcnn(torch.from_numpy(r[None]), torch.from_numpy(t[None]))
        seen, err = traced(type(layer).sample_rois_for_rcnn, run_layer)
        _store(out, case["name"] + ".layer", seen, err)
        if err is None:
            out[case["name"] + ".layer.iou"] = res["out"][2].numpy()[0]
            out[case["name"] + ".layer.rois"] = res["out"][0].numpy()[0]
    np.savez_compressed(GOLDEN, **out)
    print("wrote", os.path.relpath(GOLDEN, ROOT), "%d bytes" % os.path.getsize(GOLDEN))


def _store(out, key, seen, err):
    raises = err is not None and not isinstance(err, Stop)
    out[key + ".raises"] = np.array(raises)
    out[key + ".pdb"] = np.array(isinstance(err, Stop) and "jitter" not in seen)      # no fg and no bg
    for tag in ("branch", "jitter"):
        for k, v in seen.get(tag, {}).items():
            out["%s.%s.%s" % (key, tag, k)] = v
    j = seen.get("jitter", {})
    print("%-28s %s fg %s bg %s" % (key, ("raises %s" % type(err).__name__) if raises else "ok", j.get("fg_rois_per_this_image", "-"),
                                    j.get("bg_rois_per_this_image", "-")))


if __name__ == "__main__":
    main()
