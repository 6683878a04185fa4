"""CPU restatement (numpy / torch CPU) of the in-network RCNN target layer, lib/rpn/proposal_target_layer.py with
ROI_SAMPLE_JIT, for one scene.  TEST INFRASTRUCTURE ONLY: imported by tests/ and scripts/, never by pointrcnn_b200/.

It is oracle/rcnn_offline.py's loader restatement with the parameters in which the layer differs from the loader:
  * the fg list is only the RoIs over min(REG_FG_THRESH, CLS_FG_THRESH): no GT-max RoIs (the layer's :113 is commented out);
  * fg rows run ROI_FG_AUG_TIMES jitter tries (0 allowed), bg rows 1 if ROI_FG_AUG_TIMES > 0 else 0; a row with no try, or
    whose last try kept the source box, reports the source's max IoU;
  * every row of roi_boxes3d is a candidate (zero padding: IoU 0, easy bg); trailing all-zero GT rows are trimmed;
  * stage-2 augmentation always rotates, scales and flips: angle U(-pi / AUG_ROT_RANGE, 0) (the reference's
    `rand - 0.5 / 0.5`), scale U(0.95, 1.05), flip with p = 0.5;
  * the canonical transform rotates the points by the augmented ry and the GT box by ry mod 2 pi.
IoU and pooling are oracle.boxes_iou3d / oracle.roipool3d, the fp32 op sequences of boxes_iou3d_gpu / roipool3d_gpu.
Two draw sources:
  "ref"   the layer's host random calls in its order: np.random.permutation / rand (fg), torch.randint on the CPU generator
          (bg), np.random.rand (keep), torch.rand / randint on the CPU (single / multiple jitter); with AUG_DATA off this is the
          reference run on the CPU (the augmentation draws are batch-wide there and are not restated)
  "hash"  the device's counter-based keys (csrc/rcnn_sample.cu); augmentation and canonical transform in float64
"""
import numpy as np
import torch

from oracle import oracle as O
from oracle import rcnn_offline as RO

# tools/cfgs/default.yaml
CFG = dict(AUG_DATA=True, AUG_ROT_RANGE=18, USE_INTENSITY=False, USE_DEPTH=True, POOL_EXTRA_WIDTH=1.0, NUM_POINTS=512,
           REG_AUG_METHOD="multiple", ROI_FG_AUG_TIMES=10, CLS_FG_THRESH=0.6, CLS_BG_THRESH=0.45, CLS_BG_THRESH_LO=0.05,
           REG_FG_THRESH=0.55, FG_RATIO=0.5, ROI_PER_IMAGE=64, HARD_BG_RATIO=0.8)
# the three methods of data_augmentation, always on, flip when 1 - u < 0.5 (RO._augment_f64's rule)
_AUG = dict(AUG_METHOD_LIST=["rotation", "scaling", "flip"], AUG_METHOD_PROB=[1.0, 1.0, 0.5])


class RefDraws(RO.NumpyDraws):
    """the reference layer's host random calls (numpy global state, torch CPU generator)"""

    def __init__(self):
        super().__init__(np.random)

    def bg(self, rows, size):
        return torch.randint(low=0, high=size, size=(rows,)).long().numpy()

    def jitter(self, box, method, row, t):
        b = torch.from_numpy(np.asarray(box, np.float32))
        if method == "single":
            pos = torch.rand(3) - 0.5
            hwl = (torch.rand(3) - 0.5) / (0.5 / 0.15) + 1.0
            ang = (torch.rand(1) - 0.5) / (0.5 / (np.pi / 12))
        elif method == "multiple":
            rc = RO.RANGE_CONFIG[torch.randint(low=0, high=len(RO.RANGE_CONFIG), size=(1,))[0].long()]
            pos = ((torch.rand(3) - 0.5) / 0.5) * rc[0]
            hwl = ((torch.rand(3) - 0.5) / 0.5) * rc[1] + 1.0
            ang = ((torch.rand(1) - 0.5) / 0.5) * rc[2]
        else:
            raise NotImplementedError(method)
        return torch.cat([b[0:3] + pos, b[3:6] * hwl, b[6:7] + ang]).numpy()


class JitHashDraws(RO.HashDraws):
    """the device's keys; the rotation interval [-pi / AUG_ROT_RANGE, 0)"""

    def aug(self, row, cfg):
        f = np.float32
        u = lambda slot: self._u(RO.SALT_AUG, row, 0, slot)
        lo = f(-f(np.pi) / f(cfg["AUG_ROT_RANGE"]))
        angle = float(f(lo + f(f(f(0) - lo) * u(3))))
        scale = float(f(f(0.95) + f(f(0.1) * u(4))))
        return np.array([-1.0, -1.0, float(f(1) - u(2))]), angle, scale


def trimmed_gt(gt):
    """the reference's `while cur_gt[k].sum() == 0: k -= 1` for rows that are all zero"""
    nz = np.nonzero(np.any(gt != 0, axis=1))[0]
    return gt[:nz[-1] + 1] if nz.size else gt[:0]


def sample_scene(scene, cfg=None, draw="hash", seed=0, scene_index=0):
    """scene: dict rpn_xyz (N,3), rpn_features (N,C), seg_mask (N,), pts_depth (N,) [, rpn_intensity], roi_boxes3d (M,7) (every row
    a candidate), gt_boxes3d (G,7) (trailing zero rows trimmed).  -> dict: status, branch, sel (R,3) [source RoI, GT, tries], iou
    (R,), rois / gt_of_rois (R,7) before augmentation, empty (R,), pts_feature (R,S,F), sampled_pts (R,S,3) and gt_of_rois_ct (R,7)
    after the canonical transform, roi_boxes3d (R,7) after augmentation, cls_label, reg_valid_mask"""
    c = dict(CFG, **(cfg or {}))
    R, S = c["ROI_PER_IMAGE"], c["NUM_POINTS"]
    dr = RefDraws() if draw == "ref" else JitHashDraws(seed, scene_index)
    rois_all = np.asarray(scene["roi_boxes3d"], np.float32).reshape(-1, 7)
    gts = trimmed_gt(np.asarray(scene["gt_boxes3d"], np.float32).reshape(-1, 7))
    xyz = np.asarray(scene["rpn_xyz"], np.float32)
    extra = ([np.asarray(scene["rpn_intensity"], np.float32).reshape(-1, 1)] if c["USE_INTENSITY"] else [])
    extra.append(np.asarray(scene["seg_mask"], np.float32).reshape(-1, 1))
    if c["USE_DEPTH"]:
        extra.append((np.asarray(scene["pts_depth"], np.float32) / np.float32(70.0) - np.float32(0.5)).reshape(-1, 1))
    feat_all = np.concatenate(extra + [np.asarray(scene["rpn_features"], np.float32)], axis=1)
    out = dict(status=0)
    if len(rois_all) == 0 or len(gts) == 0:
        return _ignored(out, 2, R, S, feat_all.shape[1])
    iou3d = O.boxes_iou3d(rois_all, gts)
    max_overlaps, gt_assignment = iou3d.max(axis=1), iou3d.argmax(axis=1)
    fg_thresh = min(c["REG_FG_THRESH"], c["CLS_FG_THRESH"])
    fg_inds = np.nonzero(max_overlaps >= fg_thresh)[0]
    easy = np.nonzero(max_overlaps < c["CLS_BG_THRESH_LO"])[0]
    hard = np.nonzero((max_overlaps < c["CLS_BG_THRESH"]) & (max_overlaps >= c["CLS_BG_THRESH_LO"]))[0]
    fg_num, bg_num = fg_inds.size, hard.size + easy.size
    if fg_num > 0 and bg_num > 0:
        fg_n = min(int(np.round(c["FG_RATIO"] * R)), fg_num)
        fg_sel = fg_inds[dr.fg_perm(fg_num, fg_n)]
        bg_sel = RO._bg(dr, hard, easy, fg_n, R - fg_n, c)
        out["branch"] = "fg+bg"
    elif fg_num > 0:
        fg_n = R
        fg_sel = fg_inds[dr.fg_with_replacement(R, fg_num)]
        bg_sel = np.zeros(0, np.int64)
        out["branch"] = "fg"
    elif bg_num > 0:
        fg_n, fg_sel = 0, np.zeros(0, np.int64)
        bg_sel = RO._bg(dr, hard, easy, 0, R, c)
        out["branch"] = "bg"
    else:
        return _ignored(out, 1, R, S, feat_all.shape[1])
    sel = np.concatenate([fg_sel, bg_sel]).astype(np.int64)
    A = c["ROI_FG_AUG_TIMES"]
    rois, ious, tries = np.zeros((R, 7), np.float32), np.zeros(R, np.float32), np.zeros(R, np.int64)
    gt_of_rois = gts[gt_assignment[sel]]
    for k in range(R):
        src, gt = rois_all[sel[k]].copy(), gt_of_rois[k]
        times = A if k < fg_n else (1 if A > 0 else 0)
        temp_iou, cnt, box, keep = 0, 0, src, True
        while temp_iou < fg_thresh and cnt < times:
            keep = dr.keep(k, cnt)
            box = src if keep else dr.jitter(src, c["REG_AUG_METHOD"], k, cnt)
            temp_iou = O.boxes_iou3d(np.asarray(box, np.float32).reshape(1, 7), gt.reshape(1, 7))[0, 0]
            cnt += 1
        rois[k], tries[k] = box, cnt
        ious[k] = max_overlaps[sel[k]] if cnt == 0 or keep else temp_iou
    out.update(sel=np.stack([sel, gt_assignment[sel], tries], 1).astype(np.int32), iou=ious, rois=rois.copy(), gt_of_rois=gt_of_rois.copy())
    pooled, empty = O.roipool3d(xyz[None], feat_all[None], O.enlarge_box3d(rois, c["POOL_EXTRA_WIDTH"])[None], S)
    pooled, empty = pooled[0], empty[0].astype(np.int64)
    pts = pooled[:, :, 0:3].copy()
    out.update(empty=empty, pts_feature=pooled[:, :, 3:].copy())
    valid = (empty == 0).astype(np.int32)
    reg_valid_mask = (ious > c["REG_FG_THRESH"]).astype(np.int32) & valid
    cls_label = (ious > c["CLS_FG_THRESH"]).astype(np.int32)
    cls_label[(ious > c["CLS_BG_THRESH"]) & (ious < c["CLS_FG_THRESH"])] = -1
    cls_label[valid == 0] = -1
    if draw == "ref":
        if c["AUG_DATA"]:
            raise NotImplementedError("the reference's augmentation draws are batch-wide on the device generator")
        pts_ct, gt_ct = _canonical_ref(pts, rois, gt_of_rois)
    else:
        if c["AUG_DATA"]:
            p64, r64, g64 = np.zeros((R, S, 3)), np.zeros((R, 7)), np.zeros((R, 7))
            for k in range(R):
                en, angle, scale = dr.aug(k, c)
                p64[k], r64[k], g64[k] = RO._augment_f64(pts[k], rois[k], gt_of_rois[k], en, angle, scale, _AUG)
            pts, rois, gt_of_rois = p64, r64, g64
        pts_ct, gt_ct = _canonical_f64(pts, rois, gt_of_rois)
    out.update(sampled_pts=pts_ct, gt_of_rois_ct=gt_ct, roi_boxes3d=rois, cls_label=cls_label, reg_valid_mask=reg_valid_mask)
    return out


def _ignored(out, status, R, S, F):
    z = lambda *s: np.zeros(s, np.float32)
    out.update(status=status, branch="none", sel=np.tile(np.array([-1, -1, 0], np.int32), (R, 1)), iou=z(R), rois=z(R, 7),
               gt_of_rois=z(R, 7), empty=np.ones(R, np.int64), pts_feature=z(R, S, F), sampled_pts=z(R, S, 3), gt_of_rois_ct=z(R, 7),
               roi_boxes3d=z(R, 7), cls_label=np.full(R, -1, np.int32), reg_valid_mask=np.zeros(R, np.int32))
    return out


def _canonical_ref(pts, rois, gt_of_rois):
    """proposal_target_layer.py:45-56 with the reference's torch operations, one scene"""
    p, r, g = torch.from_numpy(pts.copy()), torch.from_numpy(rois.copy()), torch.from_numpy(gt_of_rois.copy())
    roi_ry = r[:, 6] % (2 * np.pi)
    roi_center = r[:, 0:3]
    p = p - roi_center.unsqueeze(dim=1)
    g[:, 0:3] = g[:, 0:3] - roi_center
    g[:, 6] = g[:, 6] - roi_ry
    p = RO.rotate_pc_along_y_torch(p, r[:, 6])
    g = RO.rotate_pc_along_y_torch(g.unsqueeze(dim=1), roi_ry).squeeze(dim=1)
    return p.numpy(), g.numpy()


def _canonical_f64(pts, rois, gt_of_rois):
    r = np.asarray(rois, np.float64)
    roi_ry = np.mod(r[:, 6], 2 * np.pi)
    p = np.asarray(pts, np.float64) - r[:, None, 0:3]
    p[:, :, 0], p[:, :, 2] = RO._rot64(p[:, :, 0], p[:, :, 2], r[:, None, 6])        # the points: the augmented ry itself
    g = np.asarray(gt_of_rois, np.float64).copy()
    g[:, 0:3] -= r[:, 0:3]
    g[:, 0], g[:, 2] = RO._rot64(g[:, 0], g[:, 2], roi_ry)
    g[:, 6] -= roi_ry
    return p, g
