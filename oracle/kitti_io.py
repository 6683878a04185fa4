"""oracle/kitti_io.py -- CPU restatement (numpy) of the reference's RPN input pipeline and KITTI result writer.
TEST INFRASTRUCTURE ONLY: imported by tests/ and oracle/make_golden_kitti_io.py, never by pointrcnn_b200/.

Follows (reference file:line):
  lidar_to_rect, rect_to_img            lib/utils/calibration.py:51-70
  get_valid_flag                        lib/datasets/kitti_rcnn_dataset.py:198-219
  rpn_sample                            lib/datasets/kitti_rcnn_dataset.py:246-353 (the np.random calls in the same order)
  data_augmentation                     lib/datasets/kitti_rcnn_dataset.py:513-570 (stage 1), lib/utils/kitti_utils.py:32-42
  rpn_training_labels                   lib/datasets/kitti_rcnn_dataset.py:355-391 with the hull test done as exact box
                                        geometry (kitti_utils.py:66-101 corner layout) instead of scipy's Delaunay
  image_boxes, kitti_lines              lib/utils/calibration.py:106-124, tools/eval_rcnn.py:69-94
Pinned by tests/golden/kitti_io.npz, which the reference's own Python produced (oracle/make_golden_kitti_io.py).
"""
import numpy as np

# a KITTI-like calibration (values of the usual magnitude; fp32 like get_calib_from_file, calibration.py:5-22)
CALIB = dict(
    P2=np.array([[721.5377, 0.0, 609.5593, 44.85728], [0.0, 721.5377, 172.854, 0.2163791], [0.0, 0.0, 1.0, 0.002745884]], np.float32),
    R0=np.array([[0.9999239, 0.00983776, -0.007445048], [-0.009869795, 0.9999421, -0.004278459],
                 [0.007402527, 0.004351614, 0.9999631]], np.float32),
    Tr_velo2cam=np.array([[0.007533745, -0.9999714, -0.000616602, -0.004069766], [0.01480249, 0.0007280733, -0.9998902, -0.07631618],
                          [0.9998621, 0.00752379, 0.01480755, -0.2717806]], np.float32))
IMG_SHAPE = (375, 1242, 3)
SCOPE = np.array([[-40.0, 40.0], [-1.0, 3.0], [0.0, 70.4]])


def synth_scan(seed, n=30000, n_gt=6):
    """a raw scan in the LIDAR frame (x forward, y left, z up) + GT boxes in the rectified camera frame with points on them"""
    rng = np.random.default_rng(seed)
    gt = np.zeros((n_gt, 7), np.float32)
    gt[:, 0] = rng.uniform(-15, 15, n_gt)
    gt[:, 2] = rng.uniform(8, 55, n_gt)
    gt[:, 1] = rng.uniform(1.4, 1.9, n_gt)
    gt[:, 3:6] = np.array([1.526, 1.629, 3.883]) * (1 + rng.uniform(-0.1, 0.1, (n_gt, 3)))
    gt[:, 6] = rng.uniform(-np.pi, np.pi, n_gt)
    # background: drawn in the camera frustum (denser near the sensor), a part of it outside the image / range box
    zb = 2.0 + 70.0 * rng.random(n) ** 4
    xb = rng.uniform(-0.95, 0.95, n) * np.minimum(zb, 45.0)
    yb = rng.uniform(-1.6, 3.4, n)
    bg = np.stack([zb + 0.27, -xb, -yb - 0.08], 1)
    # object points: sampled in the box frame (slightly larger than the box so that some fall in the ignore shell)
    per = 220
    which = np.repeat(np.arange(n_gt), per)
    loc = rng.uniform(-0.56, 0.56, (n_gt * per, 3)) * gt[which][:, [5, 3, 4]]     # l, h, w extents
    c, s = np.cos(gt[which, 6]), np.sin(gt[which, 6])
    xr = gt[which, 0] + loc[:, 0] * c + loc[:, 2] * s
    zr = gt[which, 2] - loc[:, 0] * s + loc[:, 2] * c
    yr = gt[which, 1] - gt[which, 3] / 2 + loc[:, 1]
    # rect -> lidar with the (approximate) inverse of the calibration: x_l = z_r, y_l = -x_r, z_l = -y_r
    obj = np.stack([zr + 0.27, -xr, -yr - 0.08], 1)
    pts = np.concatenate([bg, obj], 0)
    pts = pts[rng.permutation(len(pts))]
    inten = rng.random(len(pts))
    alpha = (-np.sign(np.arctan2(gt[:, 2], gt[:, 0])) * np.pi / 2 + np.arctan2(gt[:, 2], gt[:, 0]) + gt[:, 6]).astype(np.float32)
    return np.concatenate([pts, inten[:, None]], 1).astype(np.float32), gt, alpha


def lidar_to_rect(pts_lidar, calib):
    hom = np.concatenate([pts_lidar[:, :3], np.ones((len(pts_lidar), 1), np.float32)], 1)
    return hom @ (calib["Tr_velo2cam"].T @ calib["R0"].T)


def rect_to_img(pts_rect, calib):
    hom = np.concatenate([pts_rect, np.ones((len(pts_rect), 1), np.float32)], 1)
    proj = hom @ calib["P2"].T
    uv = proj[:, :2] / hom[:, 2:3]
    return uv, proj[:, 2] - calib["P2"][2, 3]


def get_valid_flag(pts_rect, uv, depth, img_shape, scope=SCOPE):
    ok = (uv[:, 0] >= 0) & (uv[:, 0] < img_shape[1]) & (uv[:, 1] >= 0) & (uv[:, 1] < img_shape[0]) & (depth >= 0)
    if scope is not None:
        for a in range(3):
            ok &= (pts_rect[:, a] >= scope[a][0]) & (pts_rect[:, a] <= scope[a][1])
    return ok


def in_box(pts, box):
    """exact geometry of the hull kitti_utils.boxes3d_to_corners3d builds: bottom face at y, top at y - h"""
    x, y, z, h, w, l, ry = [np.float32(v) for v in box]
    dx, dy, dz = pts[:, 0] - x, pts[:, 1] - y, pts[:, 2] - z
    c, s = np.float32(np.cos(ry)), np.float32(np.sin(ry))
    xc, zc = dx * c - dz * s, dx * s + dz * c
    # the y tests in the device kernel's rejecting form, so a NaN height leaves the decision to x and z as on the device (the
    # reference's Delaunay hull has no defined answer for a non-finite box)
    return ~((dy > 0) | (dy < -h)) & (np.abs(xc) <= l * np.float32(0.5)) & (np.abs(zc) <= w * np.float32(0.5))


def rpn_training_labels(pts_rect, gt_boxes3d, extra=0.2):
    n = len(pts_rect)
    cls = np.zeros(n, np.int32)
    reg = np.zeros((n, 7), np.float32)
    for box in gt_boxes3d:
        big = box.copy()
        big[3:6] += np.float32(2 * extra)
        big[1] += np.float32(extra)
        fg, fg_big = in_box(pts_rect, box), in_box(pts_rect, big)
        cls[fg] = 1
        cls[fg ^ fg_big] = -1
        centre = box[0:3].copy()
        centre[1] -= box[3] / 2
        reg[fg, 0:3] = centre - pts_rect[fg]
        reg[fg, 3:7] = box[3:7]
    return cls, reg


def draw_choice(depth_valid, npoints, rng):
    n = len(depth_valid)
    if npoints < n:
        near = depth_valid < 40.0
        far_i, near_i = np.where(~near)[0], np.where(near)[0]
        pick = rng.choice(near_i, npoints - len(far_i), replace=False)
        ch = np.concatenate((pick, far_i)) if len(far_i) else pick
    else:
        ch = np.arange(n, dtype=np.int32)
        if npoints > n:
            ch = np.concatenate((ch, rng.choice(ch, npoints - n, replace=False)))
    rng.shuffle(ch)
    return ch


def data_augmentation(pts, gt, gt_alpha, rng, probs=(0.5, 0.5, 0.5), rot_range=18):
    pts, gt = pts.copy(), gt.copy()
    en = 1 - rng.rand(3)
    method = []
    if en[0] < probs[0]:
        ang = rng.uniform(-np.pi / rot_range, np.pi / rot_range)
        R = np.array([[np.cos(ang), -np.sin(ang)], [np.sin(ang), np.cos(ang)]])
        pts[:, [0, 2]] = pts[:, [0, 2]] @ R.T
        gt[:, [0, 2]] = gt[:, [0, 2]] @ R.T
        beta = np.arctan2(gt[:, 2], gt[:, 0])
        gt[:, 6] = np.sign(beta) * np.pi / 2 + gt_alpha - beta
        method.append(["rotation", ang])
    if en[1] < probs[1]:
        sc = rng.uniform(0.95, 1.05)
        pts = pts * sc
        gt[:, 0:6] = gt[:, 0:6] * sc
        method.append(["scaling", sc])
    if en[2] < probs[2]:
        pts[:, 0] = -pts[:, 0]
        gt[:, 0] = -gt[:, 0]
        gt[:, 6] = np.sign(gt[:, 6]) * np.pi - gt[:, 6]
        method.append("flip")
    return pts, gt, method


def rpn_sample(lidar, calib, img_shape, gt, gt_alpha, npoints, rng, train=True):
    """one scene through the reference's get_rpn_sample order of operations (GT-paste augmentation off)"""
    rect = lidar_to_rect(lidar, calib)
    uv, depth = rect_to_img(rect, calib)
    ok = get_valid_flag(rect, uv, depth, img_shape)
    rect, inten = rect[ok][:, :3], lidar[ok, 3]
    ch = draw_choice(rect[:, 2], npoints, rng)
    pts, feat = rect[ch], (inten[ch] - 0.5).reshape(-1, 1)
    out = dict(valid=ok, choice=ch, pts_features=feat)
    g = gt.copy()
    if train:
        pts, g, out["aug_method"] = data_augmentation(pts, g, gt_alpha, rng)
    out["pts_rect"], out["gt_boxes3d"] = pts, g
    out["pts_input"] = np.concatenate((pts, feat), 1)
    out["rpn_cls_label"], out["rpn_reg_label"] = rpn_training_labels(pts, g)
    return out


def corners3d(boxes):
    b = np.asarray(boxes, np.float32)
    h, w, l = b[:, 3], b[:, 4], b[:, 5]
    sx = np.array([1, 1, -1, -1, 1, 1, -1, -1], np.float32) / np.float32(2)
    sz = np.array([1, -1, -1, 1, 1, -1, -1, 1], np.float32) / np.float32(2)
    xc, zc = l[:, None] * sx, w[:, None] * sz
    yc = np.concatenate([np.zeros((len(b), 4), np.float32), -np.repeat(h[:, None], 4, 1)], 1)
    c, s = np.cos(b[:, 6])[:, None], np.sin(b[:, 6])[:, None]
    x = b[:, 0:1] + (xc * c + zc * s)
    z = b[:, 2:3] + (-xc * s + zc * c)
    return np.stack([x, b[:, 1:2] + yc, z], 2).astype(np.float32)


def image_boxes(boxes, P2, img_shape):
    cr = corners3d(boxes).astype(np.float64)
    hom = np.concatenate([cr, np.ones(cr.shape[:2] + (1,))], 2) @ P2.T.astype(np.float64)
    u, v = hom[:, :, 0] / hom[:, :, 2], hom[:, :, 1] / hom[:, :, 2]
    ib = np.stack([u.min(1), v.min(1), u.max(1), v.max(1)], 1)
    ib[:, [0, 2]] = np.clip(ib[:, [0, 2]], 0, img_shape[1] - 1)
    ib[:, [1, 3]] = np.clip(ib[:, [1, 3]], 0, img_shape[0] - 1)
    valid = ((ib[:, 2] - ib[:, 0]) < img_shape[1] * 0.8) & ((ib[:, 3] - ib[:, 1]) < img_shape[0] * 0.8)
    beta = np.arctan2(boxes[:, 2], boxes[:, 0])
    alpha = -np.sign(beta) * np.pi / 2 + beta + boxes[:, 6]
    return ib, alpha, valid


def kitti_lines(boxes, scores, P2, img_shape, cls_name="Car"):
    ib, alpha, valid = image_boxes(boxes, P2, img_shape)
    out = []
    for k in range(len(boxes)):
        if valid[k]:
            b = boxes[k]
            out.append("%s -1 -1 %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f %.4f\n" % (
                cls_name, alpha[k], ib[k, 0], ib[k, 1], ib[k, 2], ib[k, 3], b[3], b[4], b[5], b[0], b[1], b[2], b[6], scores[k]))
    return "".join(out)


def parse_kitti_text(text):
    rows = [ln.split() for ln in text.strip().split("\n") if ln.strip()]
    return [r[0] for r in rows], np.array([[float(v) for v in r[1:]] for r in rows], np.float64).reshape(len(rows), -1)
