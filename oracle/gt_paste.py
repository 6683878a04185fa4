"""oracle/gt_paste.py -- CPU restatement (numpy) of the reference's GT-paste augmentation.
TEST INFRASTRUCTURE ONLY: imported by tests/, scripts/ and oracle/make_golden_gt_paste.py, never by pointrcnn_b200/.

Follows (reference file:line):
  gt_paste_scene           lib/datasets/kitti_rcnn_dataset.py:408-511 (apply_gt_aug_to_one_scene)
  iou3d                    lib/utils/kitti_utils.py:195-235 (get_iou3d) with the bottom-face overlap computed by an exact
                           float64 convex-polygon clip instead of shapely
  paste_in_box             lib/utils/roipool3d/src/roipool3d.cpp:82-95 (pts_in_boxes3d_cpu's predicate)
  rpn_sample_with_paste    lib/datasets/kitti_rcnn_dataset.py:246-353 with GT_AUG_ENABLED (the np.random calls in the same order)
The rest of the scene pipeline (calibration, validity, npoints draw, augmentation, labels) is oracle/kitti_io.py's.
Pinned by tests/golden/gt_paste.npz, which the reference's own Python produced (oracle/make_golden_gt_paste.py).
"""
import numpy as np

from oracle import kitti_io as K


def rpn_sample_with_paste(lidar, calib, img_shape, gt, gt_alpha, npoints, rng, train=True, gt_db=None, road_plane=None, all_gt_boxes3d=None,
               gt_aug=None):
    """kitti_io.rpn_sample with GT-paste augmentation (kitti_rcnn_dataset.py:273-282, 324-331) in the reference's order:
    validity filter, apply draw and paste loop, npoints draw, data_augmentation.  Pastes only with gt_db (a list of entries
    as synth_gt_database returns them) and road_plane, in train mode; gt_alpha is extended with the pasted entries' alpha"""
    rect = K.lidar_to_rect(lidar, calib)
    uv, depth = K.rect_to_img(rect, calib)
    ok = K.get_valid_flag(rect, uv, depth, img_shape)
    rect, inten = rect[ok][:, :3], lidar[ok, 3]
    g, alpha = gt.copy(), np.asarray(gt_alpha, np.float32)
    out = dict(valid=ok)
    if gt_db is not None and train:
        kw = dict(GT_AUG_DEFAULTS, **(gt_aug or {}))
        coll = gt if all_gt_boxes3d is None else all_gt_boxes3d
        if rng.rand() < kw.pop("apply_prob"):
            rect, inten, extra, extra_alpha = gt_paste_scene(rect, inten, coll, gt_db, road_plane, rng, **kw)
            g = np.concatenate([g, extra], 0).astype(np.float32)
            alpha = np.concatenate([alpha, extra_alpha]).astype(np.float32)
            out["pasted"] = len(extra)
        out["pts_all"] = rect
    ch = K.draw_choice(rect[:, 2], npoints, rng)
    pts, feat = rect[ch], (inten[ch] - 0.5).reshape(-1, 1)
    out.update(choice=ch, pts_features=feat)
    if train:
        pts, g, out["aug_method"] = K.data_augmentation(pts, g, alpha, rng)
    out["pts_rect"], out["gt_boxes3d"] = pts, g
    out["pts_input"] = np.concatenate((pts, feat), 1)
    out["rpn_cls_label"], out["rpn_reg_label"] = K.rpn_training_labels(pts, g)
    return out


# ------------------------------------------------------------------------------------------------ GT-paste
GT_AUG_DEFAULTS = dict(apply_prob=1.0, extra_num=15, rand_num=True, hard_ratio=0.6)      # tools/cfgs/default.yaml:11-15


def synth_gt_database(seed, n=40):
    """a GT-paste database like tools/generate_gt_database.py writes (points in the rect frame, box bottom at y):
    entries {gt_box3d (7,) f32, points (n,3) f32, intensity (n,) f32, alpha}; easy (> 100 points) and hard ones, a few
    with fewer than 5 points, a few centred outside the range box"""
    rng = np.random.default_rng(seed)
    db = []
    for e in range(n):
        box = np.zeros(7, np.float32)
        box[0] = rng.uniform(-25, 25)
        box[2] = rng.uniform(6, 60)
        box[1] = rng.uniform(1.5, 1.9)
        box[3:6] = np.array([1.526, 1.629, 3.883]) * (1 + rng.uniform(-0.1, 0.1, 3))
        box[6] = rng.uniform(-np.pi, np.pi)
        if e % 13 == 5:
            box[2] = rng.uniform(72, 80)                    # centre beyond the range box
        if e % 11 == 7:
            box[0] = rng.uniform(41, 45) * (1 if e % 2 else -1)
        npts = [int(rng.integers(150, 600)), int(rng.integers(5, 100)), int(rng.integers(101, 200)), int(rng.integers(12, 60))][e % 4]
        if e % 9 == 4:
            npts = int(rng.integers(1, 5))                  # too few points
        loc = rng.uniform(-0.5, 0.5, (npts, 3)) * box[[5, 3, 4]]
        c, s = np.cos(box[6]), np.sin(box[6])
        pts = np.stack([box[0] + loc[:, 0] * c + loc[:, 2] * s, box[1] - box[3] / 2 + loc[:, 1], box[2] - loc[:, 0] * s + loc[:, 2] * c], 1)
        beta = np.arctan2(box[2], box[0])
        db.append(dict(gt_box3d=box, points=pts.astype(np.float32), intensity=rng.random(npts).astype(np.float32),
                       alpha=float(-np.sign(beta) * np.pi / 2 + beta + box[6])))
    return db


def road_plane(tilt=0.01, height=1.65):
    """a slightly tilted road plane a x + b y + c z + d = 0 with the normal facing up (b < 0), unit normal"""
    p = np.array([tilt, -1.0, 0.5 * tilt, height])
    return p / np.linalg.norm(p[:3])


def _poly_area(p):
    x, y = p[:, 0], p[:, 1]
    return 0.5 * (np.dot(x, np.roll(y, -1)) - np.dot(y, np.roll(x, -1)))


def clip_area(a, b):
    """intersection area of two convex polygons (n,2), float64 Sutherland-Hodgman"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    if _poly_area(b) < 0:
        b = b[::-1]
    out = list(a)
    for i in range(len(b)):
        p0, p1 = b[i], b[(i + 1) % len(b)]
        e = p1 - p0
        side = lambda q: e[0] * (q[1] - p0[1]) - e[1] * (q[0] - p0[0])
        inp, out = out, []
        for j in range(len(inp)):
            cur, prev = inp[j], inp[j - 1]
            sc, sp = side(cur), side(prev)
            if sc >= 0:
                if sp < 0:
                    out.append(prev + (cur - prev) * (sp / (sp - sc)))
                out.append(cur)
            elif sp >= 0:
                out.append(prev + (cur - prev) * (sp / (sp - sc)))
        if not out:
            return 0.0
    return abs(_poly_area(np.array(out))) if len(out) >= 3 else 0.0


def iou3d(corners_a, corners_b):
    """(N,8,3), (M,8,3) -> (N,M) 3D IoU as kitti_utils.get_iou3d defines it: bottom faces (x, z) intersected, height
    range [-y_bottom, -y_top] from the float32 corners; the polygon area by clip_area instead of shapely"""
    A, B = np.asarray(corners_a, np.float32), np.asarray(corners_b, np.float32)
    lo_a, hi_a = -A[:, 0:4, 1].sum(1) / 4.0, -A[:, 4:8, 1].sum(1) / 4.0
    lo_b, hi_b = -B[:, 0:4, 1].sum(1) / 4.0, -B[:, 4:8, 1].sum(1) / 4.0
    out = np.zeros((len(A), len(B)), np.float32)
    for i in range(len(A)):
        for j in range(len(B)):
            oh = max(0.0, float(min(hi_a[i], hi_b[j])) - float(max(lo_a[i], lo_b[j])))
            if oh == 0:
                continue
            pa, pb = A[i, 0:4][:, [0, 2]], B[j, 0:4][:, [0, 2]]
            ov = clip_area(pa, pb) * oh
            union = abs(_poly_area(pa.astype(np.float64))) * float(hi_a[i] - lo_a[i]) + \
                abs(_poly_area(pb.astype(np.float64))) * float(hi_b[j] - lo_b[j]) - ov
            out[i, j] = ov / union
    return out


def paste_in_box(pts, box):
    """pts_in_boxes3d_cpu's predicate (roipool3d.cpp:82-95): fp32 differences and rotation, cos / sin computed in double
    and stored to float, the half sizes and their comparisons in double"""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    cx, by, cz, h, w, l, ang = [np.float32(v) for v in box]
    cy = np.float32(np.float64(by) - np.float64(h) / 2.0)
    dx, dz = x - cx, z - cz
    # the source's rejecting form: a NaN difference or height passes these tests and leaves the decision to the rotation
    ok = ~((np.abs(dx) > np.float32(10.0)) | (np.abs(y - cy).astype(np.float64) > np.float64(h) / 2.0) | (np.abs(dz) > np.float32(10.0)))
    cosa, sina = np.float32(np.cos(np.float64(ang))), np.float32(np.sin(np.float64(ang)))
    x_rot = dx * cosa + dz * (-sina)
    z_rot = dx * sina + dz * cosa
    hl, hw = np.float64(l) / 2.0, np.float64(w) / 2.0
    return ok & (x_rot >= -hl) & (x_rot <= hl) & (z_rot >= -hw) & (z_rot <= hw)


def enlarged_wl(boxes):
    b = np.array(boxes, np.float32).reshape(-1, 7)
    b[:, 4] += np.float32(0.5)
    b[:, 5] += np.float32(0.5)
    return b


def gt_paste_scene(pts_rect, pts_intensity, all_gt_boxes3d, gt_db, plane, rng, extra_num=15, rand_num=True, hard_ratio=0.6,
                   scope=K.SCOPE, reduce_by_range=True):
    """apply_gt_aug_to_one_scene: up to 100 tries, each drawing the easy / hard list and an entry; candidates outside the
    range box or with fewer than 5 points are skipped, the rest are moved onto the road plane (float64 arithmetic,
    float32 stores), counted, and accepted when their enlarged box overlaps no current box.  The label box of a pasted
    object is the moved gt_box3d of this draw (the reference moves the shared obj.pos instead, which drifts from the
    second draw of an entry on).  -> pts_rect, pts_intensity (kept points in order, then the pasted ones), extra boxes
    (n,7), extra alpha (n,)"""
    if hard_ratio > 0:
        lists = ([e for e in gt_db if len(e["points"]) > 100], [e for e in gt_db if len(e["points"]) <= 100])
    extra = rng.randint(10, extra_num) if rand_num else extra_num
    cur = enlarged_wl(all_gt_boxes3d)
    cur_corners = K.corners3d(cur)
    keep = np.ones(len(pts_rect), bool)
    a, b, c, d = np.asarray(plane, np.float64)
    scope = np.asarray(scope, np.float64)
    cnt, new_pts, new_int, boxes, alphas = 0, [], [], [], []
    for _ in range(100):
        if cnt > extra:
            break
        if hard_ratio > 0:
            lst = lists[0] if rng.rand() > hard_ratio else lists[1]
            ent = lst[rng.randint(0, len(lst))]
        else:
            ent = gt_db[rng.randint(0, len(gt_db))]
        box = np.array(ent["gt_box3d"], np.float32).copy()
        pts = np.array(ent["points"], np.float32).copy()
        if reduce_by_range and not all(scope[k][0] <= box[k] <= scope[k][1] for k in range(3)):
            continue
        if len(pts) < 5:
            continue
        move = box[1] - (-d - a * box[0] - c * box[2]) / b
        box[1] -= move
        pts[:, 1] -= move
        cnt += 1
        big = enlarged_wl(box)
        corners = K.corners3d(big)
        if len(cur) and iou3d(corners, cur_corners).max() >= 1e-8:
            continue
        tall = box.copy()
        tall[3] += np.float32(2)
        keep &= ~paste_in_box(pts_rect, tall)
        new_pts.append(pts)
        new_int.append(np.asarray(ent["intensity"], np.float32))
        cur = np.concatenate([cur, big], 0)
        cur_corners = np.concatenate([cur_corners, corners], 0)
        boxes.append(box)
        alphas.append(ent["alpha"])
    if not new_pts:
        return pts_rect, pts_intensity, np.zeros((0, 7), np.float32), np.zeros(0, np.float32)
    return (np.concatenate([pts_rect[keep]] + new_pts, 0), np.concatenate([pts_intensity[keep]] + new_int, 0),
            np.stack(boxes).astype(np.float32), np.array(alphas, np.float32))
