"""oracle/oracle.py -- numpy front-end of the CPU restatement (liboracle.so) + module-level oracles.

TEST INFRASTRUCTURE ONLY.  May be imported by tests/, __graft_entry__.smoke() and bench.py's
cpu_baseline / --impl reference legs; never by anything under pointrcnn_b200/.

Op-level functions wrap oracle/pointops_oracle.c one-to-one (see that file's header for the
reference file:line each one follows).  Module-level functions restate the Python orchestration:
  sa_module_msg   pointnet2_lib/pointnet2/pointnet2_modules.py:19-55 + pointnet2_utils.py:241-264
  fp_module       pointnet2_lib/pointnet2/pointnet2_modules.py:127-156
  shared_mlp      pointnet2_lib/pointnet2/pytorch_utils.py:5-101 (eval-mode BN folded to scale/shift)
  canonical       lib/net/rcnn_net.py:146-152 + lib/utils/kitti_utils.py:45-63
  boxes_iou3d     lib/utils/iou3d/iou3d_utils.py:21-53, kitti_utils.py:134-147
  enlarge_box3d   lib/utils/kitti_utils.py:150-160
The MLP arithmetic of the reference is third-party (torch.nn.Conv2d -> cuDNN, version unpinned,
SURVEY.md 8c); its oracle here is an fp32 numpy matmul of the same weights (tolerance stated in tests).
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

c_int, c_float, c_void_p = ctypes.c_int, ctypes.c_float, ctypes.c_void_p


def build(force=False):
    """Compile liboracle.so with gcc (seconds).  Building the checker is not using it."""
    so = os.path.join(_HERE, "liboracle.so")
    src = os.path.join(_HERE, "pointops_oracle.c")
    if force or not os.path.exists(so) or os.path.getmtime(so) < os.path.getmtime(src):
        subprocess.check_call(["make", "-C", _HERE, "oracle"], stdout=subprocess.DEVNULL)
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(build())
        _LIB.orc_box_overlap.restype = c_float
        _LIB.orc_iou_bev.restype = c_float
        _LIB.orc_iou_normal.restype = c_float
    return _LIB


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _p(a):
    return a.ctypes.data_as(c_void_p)


def num_threads():
    return int(lib().orc_num_threads())


def opt_n_threads(n):
    return int(lib().orc_opt_n_threads(int(n)))


# ------------------------------------------------------------------ pointnet2 ops
def dist2(a, b):
    """fp32 squared distance of aligned point pairs (..., 3) in the reference kernels' FMA order"""
    a, b = np.broadcast_arrays(_f32(a), _f32(b))
    shape = a.shape[:-1]
    a, b = _f32(a.reshape(-1, 3)), _f32(b.reshape(-1, 3))
    out = np.empty(a.shape[0], dtype=np.float32)
    lib().orc_dist2(a.shape[0], _p(a), _p(b), _p(out))
    return out.reshape(shape)


def fps(xyz, npoint, return_temp=False, temp0=None):
    """temp0: caller-initialised running minima (the reference's temp tensor is in/out); default 1e10 everywhere"""
    xyz = _f32(xyz)
    B, N, _ = xyz.shape
    temp = np.full((B, N), 1e10, dtype=np.float32) if temp0 is None else np.ascontiguousarray(temp0, dtype=np.float32).copy()
    idx = np.zeros((B, npoint), dtype=np.int32)
    lib().orc_fps(B, N, int(npoint), _p(xyz), _p(temp), _p(idx))
    return (idx, temp) if return_temp else idx


def gather(features, idx):
    features, idx = _f32(features), _i32(idx)
    B, C, N = features.shape
    M = idx.shape[1]
    out = np.empty((B, C, M), dtype=np.float32)
    lib().orc_gather(B, C, N, M, _p(features), _p(idx), _p(out))
    return out


def gather_grad(grad_out, idx, N):
    grad_out, idx = _f32(grad_out), _i32(idx)
    B, C, M = grad_out.shape
    g = np.zeros((B, C, N), dtype=np.float32)
    lib().orc_gather_grad(B, C, N, M, _p(grad_out), _p(idx), _p(g))
    return g


def ball_query(radius, nsample, xyz, new_xyz):
    xyz, new_xyz = _f32(xyz), _f32(new_xyz)
    B, N, _ = xyz.shape
    M = new_xyz.shape[1]
    idx = np.zeros((B, M, nsample), dtype=np.int32)
    lib().orc_ball_query(B, N, M, c_float(radius), int(nsample), _p(new_xyz), _p(xyz), _p(idx))
    return idx


def group(features, idx):
    features, idx = _f32(features), _i32(idx)
    B, C, N = features.shape
    _, M, S = idx.shape
    out = np.empty((B, C, M, S), dtype=np.float32)
    lib().orc_group(B, C, N, M, S, _p(features), _p(idx), _p(out))
    return out


def group_grad(grad_out, idx, N):
    grad_out, idx = _f32(grad_out), _i32(idx)
    B, C, M, S = grad_out.shape
    g = np.zeros((B, C, N), dtype=np.float32)
    lib().orc_group_grad(B, C, N, M, S, _p(grad_out), _p(idx), _p(g))
    return g


def three_nn(unknown, known):
    """returns (dist2, idx): the raw kernel outputs; the Python wrapper takes sqrt afterwards"""
    unknown, known = _f32(unknown), _f32(known)
    B, N, _ = unknown.shape
    M = known.shape[1]
    dist2 = np.empty((B, N, 3), dtype=np.float32)
    idx = np.empty((B, N, 3), dtype=np.int32)
    lib().orc_three_nn(B, N, M, _p(unknown), _p(known), _p(dist2), _p(idx))
    return dist2, idx


def three_interpolate(features, idx, weight):
    features, idx, weight = _f32(features), _i32(idx), _f32(weight)
    B, C, M = features.shape
    N = idx.shape[1]
    out = np.empty((B, C, N), dtype=np.float32)
    lib().orc_three_interpolate(B, C, M, N, _p(features), _p(idx), _p(weight), _p(out))
    return out


def three_interpolate_grad(grad_out, idx, weight, M):
    grad_out, idx, weight = _f32(grad_out), _i32(idx), _f32(weight)
    B, C, N = grad_out.shape
    g = np.zeros((B, C, M), dtype=np.float32)
    lib().orc_three_interpolate_grad(B, C, N, M, _p(grad_out), _p(idx), _p(weight), _p(g))
    return g


def interp_weights(dist2):
    """pointnet2_modules.py:140-142 applied to sqrt(dist2) (pointnet2_utils.py:98)"""
    dist = np.sqrt(dist2.astype(np.float32))
    recip = (np.float32(1.0) / (dist + np.float32(1e-8))).astype(np.float32)
    norm = recip.sum(axis=2, keepdims=True, dtype=np.float32)
    return (recip / norm).astype(np.float32)


# ------------------------------------------------------------------ roipool3d
def enlarge_box3d(boxes3d, extra_width):
    out = np.array(boxes3d, dtype=np.float32, copy=True)
    out[..., 3:6] += np.float32(extra_width * 2)
    out[..., 1] += np.float32(extra_width)
    return out


def pts_in_boxes3d(pts, boxes3d):
    pts, boxes3d = _f32(pts), _f32(boxes3d)
    N, M = pts.shape[0], boxes3d.shape[0]
    flag = np.zeros((M, N), dtype=np.int64)
    lib().orc_pts_in_boxes3d(N, M, _p(pts), _p(boxes3d), _p(flag))
    return flag


def roipool3d(xyz, pts_feature, boxes3d, sampled_pt_num=512):
    """boxes3d are the ALREADY ENLARGED boxes (the C++ boundary, roipool3d.cpp:48)"""
    xyz, pts_feature, boxes3d = _f32(xyz), _f32(pts_feature), _f32(boxes3d)
    B, N, _ = xyz.shape
    M, C = boxes3d.shape[1], pts_feature.shape[2]
    pooled = np.zeros((B, M, sampled_pt_num, 3 + C), dtype=np.float32)
    empty = np.zeros((B, M), dtype=np.int32)
    lib().orc_roipool3d(B, N, M, C, int(sampled_pt_num), _p(xyz), _p(boxes3d), _p(pts_feature), _p(pooled), _p(empty))
    return pooled, empty


def canonical_transform(pooled, rois):
    """rcnn_net.py:146-152: xyz -= roi centre; rotate (x,z) by roi ry (kitti_utils.py:45-63), fp32"""
    out = np.array(pooled, dtype=np.float32, copy=True)
    rois = _f32(rois)
    out[..., 0:3] -= rois[:, :, None, 0:3]
    ry = rois[..., 6]
    cosa, sina = np.cos(ry).astype(np.float32), np.sin(ry).astype(np.float32)
    x, z = out[..., 0].copy(), out[..., 2].copy()
    # pc[:, [0,2]] @ [[cos, -sin],[sin, cos]]^T  ->  x' = x*cos - z*sin ; z' = x*sin + z*cos
    out[..., 0] = x * cosa[..., None] + z * (-sina[..., None])
    out[..., 2] = x * sina[..., None] + z * cosa[..., None]
    return out


# ------------------------------------------------------------------ iou3d
def boxes3d_to_bev(boxes3d):
    b = _f32(boxes3d)
    out = np.empty((b.shape[0], 5), dtype=np.float32)
    half_l, half_w = b[:, 5] / np.float32(2), b[:, 4] / np.float32(2)
    out[:, 0], out[:, 1] = b[:, 0] - half_l, b[:, 2] - half_w
    out[:, 2], out[:, 3] = b[:, 0] + half_l, b[:, 2] + half_w
    out[:, 4] = b[:, 6]
    return out


def boxes_overlap_bev(a, b):
    a, b = _f32(a), _f32(b)
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float32)
    lib().orc_boxes_overlap_bev(a.shape[0], _p(a), b.shape[0], _p(b), _p(out))
    return out


def box_overlap_pairs(a, b, mutant=0):
    """aligned pairs (n,5) -> (overlap (n,) f32, polygon vertex count (n,) int32); mutant: see pointops_oracle.c"""
    a, b = _f32(a), _f32(b)
    n = a.shape[0]
    out = np.empty(n, dtype=np.float32)
    cnt = np.empty(n, dtype=np.int32)
    lib().orc_box_overlap_pairs(n, _p(a), _p(b), int(mutant), _p(out), _p(cnt))
    return out, cnt


def boxes_iou_bev(a, b):
    a, b = _f32(a), _f32(b)
    out = np.empty((a.shape[0], b.shape[0]), dtype=np.float32)
    lib().orc_boxes_iou_bev(a.shape[0], _p(a), b.shape[0], _p(b), _p(out))
    return out


def boxes_iou3d(boxes_a, boxes_b):
    a, b = _f32(boxes_a), _f32(boxes_b)
    ov_bev = boxes_overlap_bev(boxes3d_to_bev(a), boxes3d_to_bev(b))
    a_min, a_max = (a[:, 1] - a[:, 3])[:, None], a[:, 1][:, None]
    b_min, b_max = (b[:, 1] - b[:, 3])[None, :], b[:, 1][None, :]
    ov_h = np.clip(np.minimum(a_max, b_max) - np.maximum(a_min, b_min), 0, None).astype(np.float32)
    ov3d = ov_bev * ov_h
    vol_a = (a[:, 3] * a[:, 4] * a[:, 5])[:, None]
    vol_b = (b[:, 3] * b[:, 4] * b[:, 5])[None, :]
    return (ov3d / np.clip(vol_a + vol_b - ov3d, 1e-7, None)).astype(np.float32)


def nms_mask(boxes, thresh, normal=False):
    boxes = _f32(boxes)
    n = boxes.shape[0]
    cb = (n + 63) // 64
    mask = np.zeros((n, cb), dtype=np.uint64)
    lib().orc_nms_mask(_p(boxes), n, c_float(thresh), int(bool(normal)), _p(mask))
    return mask


def nms_scan(mask):
    mask = np.ascontiguousarray(mask, dtype=np.uint64)
    n = mask.shape[0]
    keep = np.zeros((max(n, 1),), dtype=np.int64)
    num = lib().orc_nms_scan(_p(mask), n, _p(keep))
    return keep[:num]


def nms(boxes, thresh, normal=False):
    """C++-boundary semantics: boxes already score-sorted; returns kept positions (int64)"""
    boxes = _f32(boxes)
    n = boxes.shape[0]
    keep = np.zeros((max(n, 1),), dtype=np.int64)
    num = lib().orc_nms(_p(boxes), n, c_float(thresh), int(bool(normal)), _p(keep))
    return keep[:num]


# ------------------------------------------------------------------ module level
def fold_bn(conv_w, conv_b, bn):
    """(W (Co,Ci), scale (Co), shift (Co)) with y = relu(scale * (W x) + shift); bn = dict or None"""
    W = np.asarray(conv_w, dtype=np.float32).reshape(conv_w.shape[0], -1)
    Co = W.shape[0]
    if bn is None:
        scale = np.ones(Co, dtype=np.float32)
        shift = np.zeros(Co, dtype=np.float32) if conv_b is None else np.asarray(conv_b, dtype=np.float32)
        return W, scale, shift
    inv = (np.asarray(bn["weight"], np.float32) / np.sqrt(np.asarray(bn["running_var"], np.float32) + np.float32(bn["eps"]))).astype(np.float32)
    shift = (np.asarray(bn["bias"], np.float32) - np.asarray(bn["running_mean"], np.float32) * inv).astype(np.float32)
    if conv_b is not None:
        shift = shift + inv * np.asarray(conv_b, np.float32)
    return W, inv, shift


def shared_mlp(x_rows, layers):
    """x_rows (R, C_in) fp32; layers = [(W, scale, shift), ...]; ReLU after every layer (pytorch_utils.py:20-32)"""
    h = np.asarray(x_rows, dtype=np.float32)
    for W, scale, shift in layers:
        h = h @ W.T.astype(np.float32)
        h = np.maximum(h * scale[None, :] + shift[None, :], 0).astype(np.float32)
    return h


def query_and_group(radius, nsample, xyz, new_xyz, features, use_xyz=True):
    idx = ball_query(radius, nsample, xyz, new_xyz)
    xyz_t = np.ascontiguousarray(np.transpose(_f32(xyz), (0, 2, 1)))
    g_xyz = group(xyz_t, idx)
    g_xyz = g_xyz - np.transpose(_f32(new_xyz), (0, 2, 1))[..., None]
    if features is not None:
        g_f = group(features, idx)
        return np.concatenate([g_xyz, g_f], axis=1) if use_xyz else g_f
    return g_xyz


def sa_module_msg(xyz, features, npoint, radii, nsamples, mlps, use_xyz=True, new_xyz=None):
    """mlps = list (per scale) of folded layer lists; returns (new_xyz (B,npoint,3), feats (B,sumC,npoint), fps_idx)"""
    xyz = _f32(xyz)
    B = xyz.shape[0]
    fidx = None
    if new_xyz is None:
        fidx = fps(xyz, npoint)
        new_xyz = np.stack([xyz[b][fidx[b]] for b in range(B)], axis=0)
    outs = []
    for r, ns, layers in zip(radii, nsamples, mlps):
        g = query_and_group(r, ns, xyz, new_xyz, features, use_xyz)          # (B, C, npoint, ns)
        Bc, C, M, S = g.shape
        rows = np.transpose(g, (0, 2, 3, 1)).reshape(-1, C)
        h = shared_mlp(rows, layers).reshape(Bc, M, S, -1)
        outs.append(np.transpose(h.max(axis=2), (0, 2, 1)))
    return new_xyz, np.ascontiguousarray(np.concatenate(outs, axis=1)), fidx


def fp_module(unknown, known, unknow_feats, known_feats, layers):
    d2, idx = three_nn(unknown, known)
    w = interp_weights(d2)
    interp = three_interpolate(known_feats, idx, w)
    x = np.concatenate([interp, _f32(unknow_feats)], axis=1) if unknow_feats is not None else interp
    B, C, n = x.shape
    h = shared_mlp(np.transpose(x, (0, 2, 1)).reshape(-1, C), layers).reshape(B, n, -1)
    return np.ascontiguousarray(np.transpose(h, (0, 2, 1)))
