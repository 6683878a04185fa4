"""oracle/rcnn_offline.py -- CPU restatement (numpy) of one offline RCNN training sample.
TEST INFRASTRUCTURE ONLY: imported by tests/, scripts/ and oracle/make_golden_rcnn_offline.py, never by pointrcnn_b200/.

Follows lib/datasets/kitti_rcnn_dataset.py:876-1077 (get_rcnn_training_sample_batch, sample_bg_inds,
aug_roi_by_noise_batch, random_aug_box3d :746-788, data_augmentation stage 2 :513-570, rotate_box3d_along_y :396-406,
canonical_transform_batch :685-704) and lib/utils/kitti_utils.py (boxes3d_to_corners3d, rotate_pc_along_y[_torch]).

Two draw sources:
  "numpy"  the reference's np.random calls in the reference's order (rng = np.random or a RandomState)
  "hash"   the device's counter-based keys (csrc/rcnn_sample.cu), restated; the jitter arithmetic in fp32 as the kernel does it
Two IoU functions:
  "exact"  oracle/gt_paste.py::iou3d, the float64 polygon clip that stands in for shapely
  "fp32"   oracle.boxes_iou3d, prb_boxes_iou3d's op sequence compiled for the host: a few ulp (about 2e-6) from the
           device's IoU, so IoUs are compared within a bound and decisions agree unless an IoU lies that close to a threshold
and, with them, two pooling predicates: "exact" pools with roipool3d_cpu's mixed float / double test (the reference's
loader), "fp32" with roipool3d_kernel.cu's (oracle.roipool3d, the device's).  ("numpy", "exact") is the reference's loader;
("hash", "fp32") is what the device computes.  In "hash" mode the augmentation and the canonical transform are float64
numpy, which the device matches to fp32 rounding only (sinf / cosf / atan2f).
"""
import numpy as np
import torch

from oracle import gt_paste as GP
from oracle import oracle as O

# tools/cfgs/default.yaml
CFG = dict(AUG_DATA=True, AUG_METHOD_LIST=["rotation", "scaling", "flip"], AUG_METHOD_PROB=[1.0, 1.0, 0.5], AUG_ROT_RANGE=18,
           USE_INTENSITY=False, USE_DEPTH=True, POOL_EXTRA_WIDTH=1.0, NUM_POINTS=512, REG_AUG_METHOD="multiple", CLS_FG_THRESH=0.6,
           CLS_BG_THRESH=0.45, CLS_BG_THRESH_LO=0.05, REG_FG_THRESH=0.55, FG_RATIO=0.5, ROI_PER_IMAGE=64, HARD_BG_RATIO=0.8)
FG_AUG_TIMES = 10
RANGE_CONFIG = [[0.2, 0.1, np.pi / 12, 0.7], [0.3, 0.15, np.pi / 12, 0.6], [0.5, 0.15, np.pi / 9, 0.5], [0.8, 0.15, np.pi / 6, 0.3],
                [1.0, 0.15, np.pi / 3, 0.2]]

# ------------------------------------------------------------------------------------------------ hashed draws
SALT_FG, SALT_BG, SALT_JITTER, SALT_AUG = 0x3c6ef372, 0xa54ff53a, 0x510e527f, 0x9b05688c
_M = 0xffffffff


def mix32(x):
    x &= _M
    x ^= x >> 16
    x = (x * 0x7feb352d) & _M
    x ^= x >> 15
    x = (x * 0x846ca68b) & _M
    x ^= x >> 16
    return x


def draw_key(seed, scene, i, salt):
    return mix32((mix32(seed ^ ((scene * 0x9e3779b9) & _M) ^ salt) + i * 0x85ebca6b) & _M)


def rs_key(seed, scene, salt, row, t, slot):
    return draw_key(seed, scene, (row << 12) | (t << 6) | slot, salt)


def u01(h):
    return np.float32(h >> 8) * np.float32(2.0 ** -24)


def pick(h, n):
    return ((h >> 8) * n) >> 24


# ------------------------------------------------------------------------------------------------ geometry
def corners3d(boxes3d):
    """boxes3d_to_corners3d with the reference's dtypes: float32 local corners, the rotation in the box's own dtype"""
    b = np.asarray(boxes3d)
    n = b.shape[0]
    h, w, l = b[:, 3], b[:, 4], b[:, 5]
    xc = np.array([l / 2., l / 2., -l / 2., -l / 2., l / 2., l / 2., -l / 2., -l / 2.], dtype=np.float32).T
    zc = np.array([w / 2., -w / 2., -w / 2., w / 2., w / 2., -w / 2., -w / 2., w / 2.], dtype=np.float32).T
    yc = np.zeros((n, 8), dtype=np.float32)
    yc[:, 4:8] = -h.reshape(n, 1).repeat(4, axis=1)
    ry = b[:, 6]
    zeros, ones = np.zeros(ry.size, dtype=np.float32), np.ones(ry.size, dtype=np.float32)
    rot = np.transpose(np.array([[np.cos(ry), zeros, -np.sin(ry)], [zeros, ones, zeros], [np.sin(ry), zeros, np.cos(ry)]]), (2, 0, 1))
    local = np.concatenate((xc.reshape(-1, 8, 1), yc.reshape(-1, 8, 1), zc.reshape(-1, 8, 1)), axis=2)
    r = np.matmul(local, rot)
    x = b[:, 0].reshape(-1, 1) + r[:, :, 0].reshape(-1, 8)
    y = b[:, 1].reshape(-1, 1) + r[:, :, 1].reshape(-1, 8)
    z = b[:, 2].reshape(-1, 1) + r[:, :, 2].reshape(-1, 8)
    return np.concatenate((x.reshape(-1, 8, 1), y.reshape(-1, 8, 1), z.reshape(-1, 8, 1)), axis=2).astype(np.float32)


def iou_matrix(a, b, iou):
    if iou == "exact":
        return GP.iou3d(corners3d(a), corners3d(b))
    return O.boxes_iou3d(np.asarray(a, np.float32), np.asarray(b, np.float32))


def rotate_pc_along_y(pc, rot_angle):
    c, s = np.cos(rot_angle), np.sin(rot_angle)
    rotmat = np.array([[c, -s], [s, c]])
    pc[:, [0, 2]] = np.dot(pc[:, [0, 2]], np.transpose(rotmat))
    return pc


def rotate_pc_along_y_torch(pc, rot_angle):
    cosa, sina = torch.cos(rot_angle).view(-1, 1), torch.sin(rot_angle).view(-1, 1)
    R = torch.cat((torch.cat([cosa, -sina], dim=1).unsqueeze(dim=1), torch.cat([sina, cosa], dim=1).unsqueeze(dim=1)), dim=1)
    pc[:, :, [0, 2]] = torch.matmul(pc[:, :, [0, 2]], R.permute(0, 2, 1))
    return pc


def rotate_box3d_along_y(box3d, rot_angle):
    old_beta = np.arctan2(box3d[2], box3d[0])
    alpha = -np.sign(old_beta) * np.pi / 2 + old_beta + box3d[6]
    box3d = rotate_pc_along_y(box3d.reshape(1, 7), rot_angle)[0]
    new_beta = np.arctan2(box3d[2], box3d[0])
    box3d[6] = np.sign(new_beta) * np.pi / 2 + alpha - new_beta
    return box3d


def in_box_cpu(pts, box):
    """roipool3d_cpu's inside test (pt_in_box3d_cpu, roipool3d.cpp:82-95 as the CPU twin evaluates it)"""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    cx, by, cz, h, w, l, ang = [np.float32(v) for v in box]
    cy = np.float32(np.float64(by) - np.float64(h) / 2.0)
    ok = (np.abs(x - cx) <= np.float32(10.0)) & (np.abs(y - cy).astype(np.float64) <= np.float64(h) / 2.0) & \
         (np.abs(z - cz) <= np.float32(10.0))
    cosa, sina = np.float32(np.cos(ang)), np.float32(np.sin(ang))
    x_rot = (x - cx) * cosa + (z - cz) * (-sina)
    z_rot = (x - cx) * sina + (z - cz) * cosa
    hl, hw = np.float64(l) / 2.0, np.float64(w) / 2.0
    return ok & (x_rot >= -hl) & (x_rot <= hl) & (z_rot >= -hw) & (z_rot <= hw)


def enlarge_box3d(boxes3d, extra_width):
    b = np.array(boxes3d, dtype=np.float32, copy=True)
    b[:, 3:6] += extra_width * 2
    b[:, 1] += extra_width
    return b


# ------------------------------------------------------------------------------------------------ draws
class NumpyDraws:
    """the reference's np.random calls"""

    def __init__(self, rng):
        self.rng = rng

    def fg_perm(self, fg_num, fg_n):
        return self.rng.permutation(fg_num)[:fg_n]

    def fg_with_replacement(self, R, fg_num):
        return np.floor(self.rng.rand(R) * fg_num).astype(np.int64)

    def bg(self, rows, size):
        return np.floor(self.rng.rand(rows) * size).astype(np.int32)

    def keep(self, row, t):
        return self.rng.rand() < 0.2

    def jitter(self, box, method, row, t):
        r = self.rng
        if method == "single":
            pos_shift = r.rand(3) - 0.5
            hwl_scale = (r.rand(3) - 0.5) / (0.5 / 0.15) + 1.0
            angle_rot = (r.rand(1) - 0.5) / (0.5 / (np.pi / 12))
        elif method == "multiple":
            rc = RANGE_CONFIG[r.randint(len(RANGE_CONFIG))]
            pos_shift = ((r.rand(3) - 0.5) / 0.5) * rc[0]
            hwl_scale = ((r.rand(3) - 0.5) / 0.5) * rc[1] + 1.0
            angle_rot = ((r.rand(1) - 0.5) / 0.5) * rc[2]
        elif method == "normal":
            sh = [r.normal(loc=0, scale=s) for s in (0.3, 0.2, 0.3, 0.25, 0.15, 0.5)]
            ry_shift = ((r.rand() - 0.5) / 0.5) * np.pi / 12
            return np.array([box[q] + sh[q] for q in range(6)] + [box[6] + ry_shift])
        else:
            raise NotImplementedError(method)
        return np.concatenate([box[0:3] + pos_shift, box[3:6] * hwl_scale, box[6:7] + angle_rot])

    def aug(self, row, cfg):
        """-> aug_enable (3,), angle or None, scale or None (data_augmentation's draws, mustaug)"""
        r = self.rng
        en = 1 - r.rand(3)
        en[0] = en[1] = -1
        angle = scale = None
        if "rotation" in cfg["AUG_METHOD_LIST"] and en[0] < cfg["AUG_METHOD_PROB"][0]:
            angle = r.uniform(-np.pi / cfg["AUG_ROT_RANGE"], np.pi / cfg["AUG_ROT_RANGE"])
        if "scaling" in cfg["AUG_METHOD_LIST"] and en[1] < cfg["AUG_METHOD_PROB"][1]:
            scale = r.uniform(0.95, 1.05)
        return en, angle, scale


class HashDraws:
    """the device's keys; the jitter in fp32 with the kernel's roundings"""

    def __init__(self, seed, scene):
        self.seed, self.scene = seed & _M, scene

    def _u(self, salt, row, t, slot):
        return u01(rs_key(self.seed, self.scene, salt, row, t, slot))

    def fg_perm(self, fg_num, fg_n):
        keys = [draw_key(self.seed, self.scene, e, SALT_FG) for e in range(fg_num)]
        return np.array(sorted(range(fg_num), key=lambda e: (keys[e], e))[:fg_n], np.int64)

    def fg_with_replacement(self, R, fg_num):
        return np.array([pick(rs_key(self.seed, self.scene, SALT_BG, r, 0, 0), fg_num) for r in range(R)], np.int64)

    def bg_row(self, row, size):
        return pick(rs_key(self.seed, self.scene, SALT_BG, row, 0, 0), size)

    def keep(self, row, t):
        return self._u(SALT_JITTER, row, t, 0) < np.float32(0.2)

    def jitter(self, box, method, row, t):
        f = np.float32
        u = lambda slot: self._u(SALT_JITTER, row, t, slot)
        s = np.asarray(box, np.float32)
        o = np.zeros(7, np.float32)
        if method == "normal":
            sd = [0.3, 0.2, 0.3, 0.25, 0.15, 0.5]
            for p in range(3):
                rr = np.sqrt(-2.0 * np.log(1.0 - float(u(2 + 2 * p))))
                a = 2.0 * np.pi * float(u(3 + 2 * p))
                o[2 * p] = s[2 * p] + f(f(rr * np.cos(a)) * f(sd[2 * p]))
                o[2 * p + 1] = s[2 * p + 1] + f(f(rr * np.sin(a)) * f(sd[2 * p + 1]))
            o[6] = s[6] + f(f(f(u(8) - f(0.5)) * f(2)) * f(np.pi / 12))
            return o
        if method == "multiple":
            rc = RANGE_CONFIG[pick(rs_key(self.seed, self.scene, SALT_JITTER, row, t, 1), 5)]
            pos_r, hwl_r, ang_r = f(rc[0]), f(rc[1]), f(rc[2])
        elif method == "single":
            pos_r, hwl_r, ang_r = f(0.5), f(0.15), f(np.pi / 12)
        else:
            raise NotImplementedError(method)
        for q in range(3):
            d = f(f(u(2 + q) - f(0.5)) * f(2))
            o[q] = f(s[q] + f(d * pos_r))
            e = f(f(u(5 + q) - f(0.5)) * f(2))
            o[3 + q] = f(s[3 + q] * f(f(e * hwl_r) + f(1)))
        o[6] = f(s[6] + f(f(f(u(8) - f(0.5)) * f(2)) * ang_r))
        return o

    def aug(self, row, cfg):
        f = np.float32
        u = lambda slot: self._u(SALT_AUG, row, 0, slot)
        en = np.array([-1.0, -1.0, float(f(1) - u(2))])
        angle = scale = None
        if "rotation" in cfg["AUG_METHOD_LIST"]:
            lo = f(-f(np.pi) / f(cfg["AUG_ROT_RANGE"]))
            angle = float(f(lo + f(f(lo * f(-2)) * u(3))))
        if "scaling" in cfg["AUG_METHOD_LIST"]:
            scale = float(f(f(0.95) + f(f(0.1) * u(4))))
        return en, angle, scale


# ------------------------------------------------------------------------------------------------ one scene
def sample_scene(scene, cfg=None, draw="numpy", iou="exact", rng=np.random, seed=0, scene_index=0, train=True):
    """scene: dict rpn_xyz (N,3), rpn_features (N,C), rpn_intensity (N,), seg_mask (N,), roi_boxes3d (M,7), gt_boxes3d (G,7).
    -> dict: status, sel (R,3) [source RoI, GT, tries], iou (R,), rois / gt_of_rois (R,7) before augmentation,
    pooled_input / pooled_features / empty (the pool), pts_input / pts_features, cls_label, reg_valid_mask, gt_boxes3d_ct,
    roi_boxes3d, gt_boxes3d (after augmentation and the canonical transform)"""
    c = dict(CFG, **(cfg or {}))
    R, S = c["ROI_PER_IMAGE"], c["NUM_POINTS"]
    dr = NumpyDraws(rng) if draw == "numpy" else HashDraws(seed, scene_index)
    rois_all = np.asarray(scene["roi_boxes3d"], np.float32).reshape(-1, 7)
    gts_all = np.asarray(scene["gt_boxes3d"], np.float32).reshape(-1, 7)
    xyz = np.asarray(scene["rpn_xyz"], np.float32)
    extra = ([np.asarray(scene["rpn_intensity"]).reshape(-1, 1)] if c["USE_INTENSITY"] else []) + [np.asarray(scene["seg_mask"]).reshape(-1, 1)]
    if c["USE_DEPTH"]:
        extra.append(((np.linalg.norm(xyz, ord=2, axis=1) / 70.0) - 0.5).reshape(-1, 1))
    extra = np.concatenate(extra, axis=1)
    E = extra.shape[1]
    feats = np.asarray(scene["rpn_features"], np.float32)
    out = dict(status=0)
    if len(rois_all) == 0 or len(gts_all) == 0:
        return _ignored(out, 2, R, S, E, feats.shape[1])
    iou3d = iou_matrix(rois_all, gts_all, iou)
    max_overlaps, gt_assignment = iou3d.max(axis=1), iou3d.argmax(axis=1)
    max_iou_of_gt, roi_assignment = iou3d.max(axis=0), iou3d.argmax(axis=0)
    roi_assignment = roi_assignment[max_iou_of_gt > 0].reshape(-1)
    fg_thresh = min(c["REG_FG_THRESH"], c["CLS_FG_THRESH"])
    fg_inds = np.concatenate((np.nonzero(max_overlaps >= fg_thresh)[0], roi_assignment), axis=0)
    easy = np.nonzero(max_overlaps < c["CLS_BG_THRESH_LO"])[0]
    hard = np.nonzero((max_overlaps < c["CLS_BG_THRESH"]) & (max_overlaps >= c["CLS_BG_THRESH_LO"]))[0]
    fg_num, bg_num = fg_inds.size, hard.size + easy.size
    fg_quota = int(np.round(c["FG_RATIO"] * R))
    if fg_num > 0 and bg_num > 0:
        fg_n = min(fg_quota, fg_num)
        fg_sel = fg_inds[dr.fg_perm(fg_num, fg_n)]
        bg_sel = _bg(dr, hard, easy, fg_n, R - fg_n, c)
        out["branch"] = "fg+bg"
    elif fg_num > 0:
        # the reference's line 923 (torch.from_numpy(...).type_as(<ndarray>)) raises: the evident meaning is implemented
        fg_n = R
        fg_sel = fg_inds[dr.fg_with_replacement(R, fg_num)]
        bg_sel = np.zeros(0, np.int64)
        out["branch"] = "fg"
    elif bg_num > 0:
        fg_n, fg_sel = 0, np.zeros(0, np.int64)
        bg_sel = _bg(dr, hard, easy, 0, R, c)
        out["branch"] = "bg"
    else:
        return _ignored(out, 1, R, S, E, feats.shape[1])
    sel = np.concatenate([fg_sel, bg_sel]).astype(np.int64)
    pos_thresh = fg_thresh
    rois, ious, tries = np.zeros((R, 7), np.float32), np.zeros(R, np.float32), np.zeros(R, np.int64)
    gt_of_rois = gts_all[gt_assignment[sel]]
    for k in range(R):
        src, gt = rois_all[sel[k]].copy(), gt_of_rois[k]
        times = FG_AUG_TIMES if k < fg_n else 1
        temp_iou, cnt, box = 0, 0, src
        while temp_iou < pos_thresh and cnt < times:
            box = src if dr.keep(k, cnt) else dr.jitter(src, c["REG_AUG_METHOD"], k, cnt)
            temp_iou = iou_matrix(box.reshape(1, 7), gt.reshape(1, 7), iou)[0][0]
            cnt += 1
        rois[k], ious[k], tries[k] = box, temp_iou, cnt
    out.update(sel=np.stack([sel, gt_assignment[sel], tries], 1).astype(np.int32), iou=ious, rois=rois.copy(), gt_of_rois=gt_of_rois.copy())
    # pooling in the original frame
    pool_boxes = enlarge_box3d(rois, c["POOL_EXTRA_WIDTH"])
    feat_all = np.concatenate((extra, feats), axis=1).astype(np.float32)
    if iou == "exact":
        pooled = np.zeros((R, S, 3 + feat_all.shape[1]), np.float32)
        empty = np.zeros(R, np.int64)
        for k in range(R):
            idx = np.nonzero(in_box_cpu(xyz, pool_boxes[k]))[0][:S]
            if idx.size == 0:
                empty[k] = 1
                continue
            idx = idx[np.arange(S) % idx.size]
            pooled[k, :, 0:3], pooled[k, :, 3:] = xyz[idx], feat_all[idx]
    else:
        pooled, empty = O.roipool3d(xyz[None], feat_all[None], pool_boxes[None], S)
        pooled, empty = pooled[0], empty[0].astype(np.int64)
    pts_input, pts_features = pooled[:, :, :3 + E].copy(), pooled[:, :, 3 + E:].copy()
    out.update(pooled_input=pts_input.copy(), pooled_features=pts_features, empty=empty)
    if c["AUG_DATA"] and train:
        for k in range(R):
            en, angle, scale = dr.aug(k, c)
            if draw == "numpy":
                pts_input[k, :, 0:3], rois[k], gt_of_rois[k] = _augment_ref(pts_input[k, :, 0:3].copy(), rois[k], gt_of_rois[k], en, angle, scale, c)
            else:
                pts_input[k, :, 0:3], rois[k], gt_of_rois[k] = _augment_f64(pts_input[k, :, 0:3], rois[k], gt_of_rois[k], en, angle, scale, c)
    valid = (empty == 0).astype(np.int32)
    reg_valid_mask = (ious > c["REG_FG_THRESH"]).astype(np.int32) & valid
    cls_label = (ious > c["CLS_FG_THRESH"]).astype(np.int32)
    cls_label[(ious > c["CLS_BG_THRESH"]) & (ious < c["CLS_FG_THRESH"])] = -1
    cls_label[valid == 0] = -1
    if draw == "numpy":
        pts_ct, gt_ct = _canonical_ref(pts_input, rois, gt_of_rois)
    else:
        pts_ct, gt_ct = _canonical_f64(pts_input, rois, gt_of_rois)
    out.update(pts_input=pts_ct, pts_features=pts_features, cls_label=cls_label, reg_valid_mask=reg_valid_mask, gt_boxes3d_ct=gt_ct,
               roi_boxes3d=rois, gt_boxes3d=gt_of_rois)
    return out


def _ignored(out, status, R, S, E, C):
    z = lambda *s: np.zeros(s, np.float32)
    out.update(status=status, branch="none", sel=np.tile(np.array([-1, -1, 0], np.int32), (R, 1)), iou=z(R), rois=z(R, 7), gt_of_rois=z(R, 7),
               pooled_input=z(R, S, 3 + E), pooled_features=z(R, S, C), empty=np.ones(R, np.int64), pts_input=z(R, S, 3 + E),
               pts_features=z(R, S, C), cls_label=np.full(R, -1, np.int32), reg_valid_mask=np.zeros(R, np.int32), gt_boxes3d_ct=z(R, 7),
               roi_boxes3d=z(R, 7), gt_boxes3d=z(R, 7))
    return out


def _bg(dr, hard, easy, row0, rows, c):
    """sample_bg_inds; hashed draws index the output row"""
    if hard.size > 0 and easy.size > 0:
        hard_n = int(rows * c["HARD_BG_RATIO"])
    elif hard.size > 0:
        hard_n = rows
    else:
        hard_n = 0
    easy_n = rows - hard_n
    if isinstance(dr, NumpyDraws):
        parts = []
        if hard_n:
            parts.append(hard[dr.bg(hard_n, hard.size)])
        if easy_n:
            parts.append(easy[dr.bg(easy_n, easy.size)])
        return np.concatenate(parts) if parts else np.zeros(0, np.int64)
    return np.array([hard[dr.bg_row(row0 + q, hard.size)] if q < hard_n else easy[dr.bg_row(row0 + q, easy.size)]
                     for q in range(rows)], np.int64)


def _augment_ref(aug_pts, roi, gt, en, angle, scale, c):
    """data_augmentation(mustaug=True, stage=2) on one RoI with the reference's numpy operations"""
    boxes = np.concatenate([roi.reshape(1, 7), gt.reshape(1, 7)], axis=0)
    if angle is not None:
        aug_pts = rotate_pc_along_y(aug_pts, rot_angle=angle)
        boxes[0] = rotate_box3d_along_y(boxes[0], angle)
        boxes[1] = rotate_box3d_along_y(boxes[1], angle)
    if scale is not None:
        aug_pts = aug_pts * scale
        boxes[:, 0:6] = boxes[:, 0:6] * scale
    if "flip" in c["AUG_METHOD_LIST"] and en[2] < c["AUG_METHOD_PROB"][2]:
        aug_pts[:, 0] = -aug_pts[:, 0]
        boxes[:, 0] = -boxes[:, 0]
        boxes[0, 6] = np.sign(boxes[0, 6]) * np.pi - boxes[0, 6]
        boxes[1, 6] = np.sign(boxes[1, 6]) * np.pi - boxes[1, 6]
    return aug_pts, boxes[0], boxes[1]


def _canonical_ref(pts_input, rois, gt_of_rois):
    roi_ry = rois[:, 6] % (2 * np.pi)
    roi_center = rois[:, 0:3]
    pts_input[:, :, [0, 1, 2]] = pts_input[:, :, [0, 1, 2]] - roi_center.reshape(-1, 1, 3)
    gt_ct = np.copy(gt_of_rois)
    gt_ct[:, 0:3] = gt_ct[:, 0:3] - roi_center
    gt_ct = rotate_pc_along_y_torch(torch.from_numpy(gt_ct.reshape(-1, 1, 7)), torch.from_numpy(roi_ry)).numpy().reshape(-1, 7)
    gt_ct[:, 6] = gt_ct[:, 6] - roi_ry
    pts = rotate_pc_along_y_torch(torch.from_numpy(pts_input), torch.from_numpy(roi_ry)).numpy()
    return pts, gt_ct


# float64 restatements of the device's augmentation and canonical transform
def _rot64(x, z, a):
    c, s = np.cos(a), np.sin(a)
    return x * c - z * s, x * s + z * c


def _rotate_box64(b, a):
    b = b.astype(np.float64)
    beta0 = np.arctan2(b[2], b[0])
    alpha = -np.sign(beta0) * np.pi / 2 + beta0 + b[6]
    b[0], b[2] = _rot64(b[0], b[2], a)
    beta1 = np.arctan2(b[2], b[0])
    b[6] = np.sign(beta1) * np.pi / 2 + alpha - beta1
    return b


def _augment_f64(pts, roi, gt, en, angle, scale, c):
    p = pts.astype(np.float64)
    rb, gb = roi.astype(np.float64), gt.astype(np.float64)
    if angle is not None:
        p[:, 0], p[:, 2] = _rot64(p[:, 0], p[:, 2], angle)
        rb, gb = _rotate_box64(rb, angle), _rotate_box64(gb, angle)
    if scale is not None:
        p, rb[0:6], gb[0:6] = p * scale, rb[0:6] * scale, gb[0:6] * scale
    if "flip" in c["AUG_METHOD_LIST"] and en[2] < c["AUG_METHOD_PROB"][2]:
        p[:, 0], rb[0], gb[0] = -p[:, 0], -rb[0], -gb[0]
        rb[6], gb[6] = np.sign(rb[6]) * np.pi - rb[6], np.sign(gb[6]) * np.pi - gb[6]
    return p, rb, gb


def _canonical_f64(pts_input, rois, gt_of_rois):
    r = rois.astype(np.float64)
    roi_ry = np.mod(r[:, 6], 2 * np.pi)
    p = pts_input.astype(np.float64)
    p[:, :, 0:3] -= r[:, None, 0:3]
    p[:, :, 0], p[:, :, 2] = _rot64(p[:, :, 0], p[:, :, 2], roi_ry[:, None])
    g = gt_of_rois.astype(np.float64)
    g[:, 0:3] -= r[:, 0:3]
    g[:, 0], g[:, 2] = _rot64(g[:, 0], g[:, 2], roi_ry)
    g[:, 6] -= roi_ry
    return p, g


# ------------------------------------------------------------------------------------------------ synthetic scenes
THRESHOLDS = (0.05, 0.45, 0.55, 0.6)


def synth_scene(seed, kind="mixed", n_pts=2048, n_feat=3, n_gt=3):
    """saved RPN output of one scene: points around the GT cars and on the ground, features, a 0/1 mask, proposals.
    kind: "mixed" (fg over the threshold and from roi_assignment, hard and easy bg, RoIs with no point), "hard" (no easy
    bg), "easy" (no hard bg), "bg" (no RoI overlaps a GT).  No RoI's IoU lies within 1e-5 of a threshold (exact clip)."""
    rng = np.random.default_rng(seed)
    gt = np.zeros((n_gt, 7), np.float32)
    gt[:, 0] = rng.uniform(-12, 12, n_gt) + np.arange(n_gt) * 9 - 9
    gt[:, 1] = rng.uniform(1.5, 1.8, n_gt)
    gt[:, 2] = rng.uniform(12, 40, n_gt)
    gt[:, 3:6] = np.array([1.52, 1.63, 3.88]) * (1 + rng.uniform(-0.1, 0.1, (n_gt, 3)))
    gt[:, 6] = rng.uniform(-np.pi, np.pi, n_gt)
    per = n_pts // (2 * n_gt)
    pts = []
    for b in gt:
        loc = rng.uniform(-0.6, 0.6, (per, 3)) * b[[5, 3, 4]]
        c, s = np.cos(b[6]), np.sin(b[6])
        pts.append(np.stack([b[0] + loc[:, 0] * c + loc[:, 2] * s, b[1] - b[3] / 2 + loc[:, 1], b[2] - loc[:, 0] * s + loc[:, 2] * c], 1))
    rest = n_pts - per * n_gt
    pts.append(np.stack([rng.uniform(-25, 25, rest), rng.uniform(1.4, 1.9, rest), rng.uniform(5, 45, rest)], 1))
    xyz = np.concatenate(pts).astype(np.float32)
    rois = []
    for j, b in enumerate(gt):
        if kind == "bg":
            break
        scales = {"mixed": [0.05, 0.1, 0.6, 1.2], "hard": [0.05, 0.5, 0.7], "easy": [0.03, 0.08]}[kind]
        if kind == "mixed" and j == n_gt - 1:
            scales = [1.3]                                   # this GT's only overlap is poor: its roi_assignment row jitters 10 times
        for sc in scales:
            for _ in range(3):
                r = b.copy()
                r[[0, 2]] += rng.normal(0, sc, 2)
                r[3:6] *= 1 + rng.normal(0, sc / 4, 3)
                r[6] += rng.normal(0, sc / 2)
                rois.append(r)
    n_far = {"mixed": 14, "hard": 0, "easy": 10, "bg": 20}[kind]
    for q in range(n_far):
        r = gt[q % n_gt].copy()
        r[0] = rng.uniform(-30, 30)
        r[2] = rng.uniform(50, 65) if q % 3 == 0 else rng.uniform(5, 45)   # beyond the points: empty pooled RoIs
        r[6] = rng.uniform(-np.pi, np.pi)
        rois.append(r)
    rois = np.array(rois, np.float32)
    for _ in range(100):
        m = GP.iou3d(corners3d(rois), corners3d(gt))
        near = np.zeros(len(rois), bool)
        for t in THRESHOLDS:
            near |= (np.abs(m - t) < 1e-5).any(1)
        if not near.any():
            break
        rois[near, 0] += np.float32(0.013)
    if kind == "hard":
        keep = GP.iou3d(corners3d(rois), corners3d(gt)).max(1) >= 0.06
        rois = rois[keep]
    if kind == "bg":
        rois = rois[GP.iou3d(corners3d(rois), corners3d(gt)).max(1) == 0]
    return dict(rpn_xyz=xyz, rpn_features=rng.standard_normal((len(xyz), n_feat)).astype(np.float32),
                rpn_intensity=rng.random(len(xyz)).astype(np.float32), seg_mask=(rng.random(len(xyz)) < 0.3).astype(np.float32),
                roi_boxes3d=rois, gt_boxes3d=gt)
