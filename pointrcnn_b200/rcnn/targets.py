"""RCNN training targets on the device, for the reference's two recipes:

  loader   the offline samples of lib/datasets/kitti_rcnn_dataset.py:876-1077 (get_rcnn_training_sample_batch,
           ROI_SAMPLE_JIT=False): RCNNOfflineSampler.prepare_batch
  layer    the in-network target layer of lib/rpn/proposal_target_layer.py (ROI_SAMPLE_JIT=True):
           ProposalTargetLayer with draw="device"

Both run the same four launches (`run`); a `Recipe` holds every value in which they differ, and `loader_recipe` /
`layer_recipe` derive it from the reference's config.  include/pointrcnn_b200.h describes each value.
"""
import collections
import types

import numpy as np
import torch

from .. import _cabi as C

# tools/cfgs/default.yaml:6-9, :60-122
DEFAULT_CFG = dict(AUG_DATA=True, AUG_METHOD_LIST=["rotation", "scaling", "flip"], AUG_METHOD_PROB=[1.0, 1.0, 0.5], AUG_ROT_RANGE=18,
                   RCNN=dict(USE_INTENSITY=False, USE_DEPTH=True, USE_SEG_SCORE=False, POOL_EXTRA_WIDTH=1.0, NUM_POINTS=512,
                             REG_AUG_METHOD="multiple", ROI_FG_AUG_TIMES=10, CLS_FG_THRESH=0.6, CLS_BG_THRESH=0.45,
                             CLS_BG_THRESH_LO=0.05, REG_FG_THRESH=0.55, FG_RATIO=0.5, ROI_PER_IMAGE=64, HARD_BG_RATIO=0.8))
AUG_METHODS = {"single": 0, "multiple": 1, "normal": 2}
# aug_roi_by_noise_batch is called with aug_times=10 for the foreground rows (kitti_rcnn_dataset.py:942), not ROI_FG_AUG_TIMES
LOADER_FG_AUG_TIMES = 10


def ns(d):
    """a nested dict -> nested SimpleNamespace, read like the reference's EasyDict cfg"""
    return types.SimpleNamespace(**{k: (ns(v) if isinstance(v, dict) else v) for k, v in d.items()})


# the arguments of prb_rcnn_sample_rois and prb_rcnn_roi_targets that the recipe chooses; counts: roi_count / gt_count are
# passed (the loader) or NULL (the layer)
Recipe = collections.namedtuple("Recipe", [
    "counts", "roi_per_image", "fg_per_image", "reg_fg_thresh", "cls_fg_thresh", "cls_bg_thresh", "cls_bg_thresh_lo", "hard_bg_ratio",
    "aug_method", "gt_max_fg", "fg_aug_times", "bg_aug_times", "kept_src_iou", "pool_extra_width",
    "num_points", "aug_data", "aug_rotation", "aug_scaling", "aug_flip", "rot_lo", "rot_hi", "flip_prob", "pts_raw_ry"])


def _shared(cfg):
    r = cfg.RCNN
    if r.REG_AUG_METHOD not in AUG_METHODS:
        raise NotImplementedError(r.REG_AUG_METHOD)
    R = int(r.ROI_PER_IMAGE)
    return dict(roi_per_image=R, fg_per_image=int(np.round(r.FG_RATIO * R)), reg_fg_thresh=r.REG_FG_THRESH, cls_fg_thresh=r.CLS_FG_THRESH,
                cls_bg_thresh=r.CLS_BG_THRESH, cls_bg_thresh_lo=r.CLS_BG_THRESH_LO, hard_bg_ratio=r.HARD_BG_RATIO,
                aug_method=AUG_METHODS[r.REG_AUG_METHOD], pool_extra_width=r.POOL_EXTRA_WIDTH, num_points=int(r.NUM_POINTS))


def _rot_lo(cfg):
    """-pi / AUG_ROT_RANGE in fp32, as the device computes the angle; AUG_ROT_RANGE <= 0 gives an interval that
    prb_rcnn_roi_targets rejects"""
    with np.errstate(divide="ignore"):
        return float(-np.float32(np.pi) / np.float32(cfg.AUG_ROT_RANGE))


def loader_recipe(cfg, mode):
    """get_rcnn_training_sample_batch: GT-max RoIs in the fg list, 10 tries per fg row and 1 per bg row, the last box's
    IoU, counts given; in TRAIN mode with AUG_DATA the methods of AUG_METHOD_LIST, rotation U(-pi/R, pi/R) for
    R = AUG_ROT_RANGE, flip with p = AUG_METHOD_PROB[2]; the points rotated by ry mod 2 pi"""
    aug = bool(cfg.AUG_DATA) and mode == "TRAIN"
    methods = list(cfg.AUG_METHOD_LIST)
    lo = _rot_lo(cfg) if aug and "rotation" in methods else 0.0
    return Recipe(counts=True, gt_max_fg=1, fg_aug_times=LOADER_FG_AUG_TIMES, bg_aug_times=1, kept_src_iou=0, aug_data=int(aug),
                  aug_rotation=int("rotation" in methods), aug_scaling=int("scaling" in methods), aug_flip=int("flip" in methods),
                  rot_lo=lo, rot_hi=-lo, flip_prob=float(cfg.AUG_METHOD_PROB[2]), pts_raw_ry=0, **_shared(cfg))


def layer_recipe(cfg):
    """ProposalTargetLayer: the fg list only the RoIs over the threshold (no GT-max RoIs), ROI_FG_AUG_TIMES tries per fg
    row and min(ROI_FG_AUG_TIMES, 1) per bg row, the source IoU for a kept box, every row a candidate and GT counts from
    the trailing zero rows; with AUG_DATA rotation, scaling and flip, the rotation U[-pi/R, 0) (the reference's
    `(rand - 0.5 / 0.5) * (pi / R)`, proposal_target_layer.py:295), flip with p = 0.5; the points rotated by the raw ry"""
    fg_times = int(cfg.RCNN.ROI_FG_AUG_TIMES)
    return Recipe(counts=False, gt_max_fg=0, fg_aug_times=fg_times, bg_aug_times=min(fg_times, 1), kept_src_iou=1,
                  aug_data=int(bool(cfg.AUG_DATA)), aug_rotation=1, aug_scaling=1, aug_flip=1, rot_lo=_rot_lo(cfg), rot_hi=0.0,
                  flip_prob=0.5, pts_raw_ry=1, **_shared(cfg))


def run(recipe, xyz, feat, rois, gts, counts, seed, seed_dev=None):
    """the recipe on one batch, on the current stream and without a host synchronisation: prb_boxes_iou3d (skipped when M
    or G is 0), prb_rcnn_sample_rois, prb_roipool3d_ws on the enlarged sampled boxes, prb_rcnn_roi_targets.
    xyz (B,N,3), feat (B,N,F), rois (B,M,7), gts (B,G,7): contiguous float32 CUDA tensors; counts (2,B) int32
    [roi_count; gt_count], required by a recipe with counts and ignored otherwise.  seed_dev: None, or a CUDA int32 tensor
    whose first element the sample and targets launches read as the seed in place of `seed` (the _dseed entries: a
    captured graph that advances it draws anew on every replay).  -> dict of the raw outputs, R = ROI_PER_IMAGE, S =
    NUM_POINTS: pooled (B,R,S,3+F) transformed rows, empty (B,R) int32, pool_boxes (B,R,7) the boxes the
    rows were pooled from, rois / gts (B,R,7) after augmentation, iou (B,R) before it, sel (B,R,3) int32, status (B) int32, gt_ct (B*R,7), cls / reg (B*R) int32"""
    if recipe.counts and counts is None:
        raise ValueError("rcnn targets: this recipe takes the RoI and GT counts")
    rc = recipe
    B, M, G, N = rois.shape[0], rois.shape[1], gts.shape[1], xyz.shape[1]
    R, S, F_ = rc.roi_per_image, rc.num_points, feat.shape[2]
    W = 3 + F_
    dev = rois.device
    L, st = C.lib(), C.stream()
    f = lambda *shp: torch.empty(shp, dtype=torch.float32, device=dev)
    i32 = lambda *shp: torch.empty(shp, dtype=torch.int32, device=dev)
    iou = f(B, M, G)
    if M and G:
        C.check(L.prb_boxes_iou3d(B, M, C.ptr(rois), G, C.ptr(gts), C.ptr(iou), st), "boxes_iou3d")
    rois_out, gt_out, iou_out, pool_boxes = f(B, R, 7), f(B, R, 7), f(B, R), f(B, R, 7)
    sel, status = i32(B, R, 3), i32(B)
    roi_count, gt_count = (counts[0], counts[1]) if rc.counts else (None, None)
    if seed_dev is None:
        sample, finish, seed = L.prb_rcnn_sample_rois, L.prb_rcnn_roi_targets, seed & 0xffffffff
    else:
        sample, finish, seed = L.prb_rcnn_sample_rois_dseed, L.prb_rcnn_roi_targets_dseed, C.ptr(seed_dev)
    C.check(sample(B, M, G, C.ptr(iou), C.ptr(rois), C.ptr(roi_count), C.ptr(gts), C.ptr(gt_count), R, rc.fg_per_image, rc.reg_fg_thresh,
                   rc.cls_fg_thresh, rc.cls_bg_thresh, rc.cls_bg_thresh_lo, rc.hard_bg_ratio, rc.aug_method, rc.gt_max_fg,
                   rc.fg_aug_times, rc.bg_aug_times, rc.kept_src_iou, rc.pool_extra_width, seed, C.ptr(rois_out), C.ptr(gt_out),
                   C.ptr(iou_out), C.ptr(pool_boxes), C.ptr(sel), C.ptr(status), st), "rcnn_sample_rois")
    pooled = f(B, R, S, W)
    empty = torch.zeros((B, R), dtype=torch.int32, device=dev)
    wsb = L.prb_roipool3d_workspace_bytes(B, N, R, S)
    ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
    C.check(L.prb_roipool3d_ws(B, N, R, F_, S, C.ptr(xyz), C.ptr(pool_boxes), C.ptr(feat), C.ptr(pooled), C.ptr(empty), None, 1,
                               C.ptr(ws), C.c_size_t(wsb), st), "roipool3d")
    gt_ct, cls, reg = f(B * R, 7), i32(B * R), i32(B * R)
    C.check(finish(B, R, S, W, C.ptr(pooled), C.ptr(rois_out), C.ptr(gt_out), C.ptr(iou_out), C.ptr(empty), rc.aug_data, rc.aug_rotation,
                   rc.aug_scaling, rc.aug_flip, rc.rot_lo, rc.rot_hi, rc.flip_prob, rc.pts_raw_ry, rc.reg_fg_thresh, rc.cls_fg_thresh,
                   rc.cls_bg_thresh, seed, C.ptr(gt_ct), C.ptr(cls), C.ptr(reg), st), "rcnn_roi_targets")
    return dict(pooled=pooled, empty=empty, pool_boxes=pool_boxes, rois=rois_out, gts=gt_out, iou=iou_out, sel=sel, status=status, gt_ct=gt_ct, cls=cls, reg=reg)
