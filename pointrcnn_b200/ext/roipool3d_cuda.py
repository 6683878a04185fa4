"""`roipool3d_cuda` -- same exports as lib/utils/roipool3d/src/roipool3d.cpp:198-203.

`forward` / `forward_slow` run the one-pass H100 kernel.  The two CPU twins the reference exports for its
dataloader (`pts_in_boxes3d_cpu`, `roipool3d_cpu`, roipool3d.cpp:97-195) are host functions by contract;
they are restated here in numpy on top of the same predicate arithmetic.
"""
import numpy as np
import torch

from .. import _cabi as C


def forward(xyz, boxes3d, pts_feature, pooled_features, pooled_empty_flag, rois_canonical=None, zero_fill_empty=False):
    """reference signature (roipool3d.cpp:48): the caller pre-zeroes `pooled_features` / `pooled_empty_flag`.
    zero_fill_empty=True (extra): the kernel zeroes the rows of empty boxes, `pooled_features` may be torch.empty"""
    for t, nm in ((xyz, "xyz"), (boxes3d, "boxes3d"), (pts_feature, "pts_feature"), (pooled_features, "pooled_features"),
                  (pooled_empty_flag, "pooled_empty_flag")):
        if not (t.is_cuda and t.is_contiguous()):
            raise RuntimeError("%s must be a contiguous CUDA tensor" % nm)  # CHECK_INPUT, roipool3d.cpp:21-25
    B, N = int(xyz.size(0)), int(xyz.size(1))
    M, Cf, S = int(boxes3d.size(1)), int(pts_feature.size(2)), int(pooled_features.size(2))
    for t, nm, dt in ((xyz, "xyz", torch.float32), (boxes3d, "boxes3d", torch.float32), (pts_feature, "pts_feature", torch.float32),
                      (pooled_features, "pooled_features", torch.float32), (pooled_empty_flag, "pooled_empty_flag", torch.int32)):
        if t.dtype != dt:
            raise RuntimeError("%s must be %s" % (nm, dt))     # the reference's .data<float>() / .data<int>() throw as well
    if tuple(pooled_features.shape) != (B, M, S, 3 + Cf) or pooled_empty_flag.numel() != B * M or boxes3d.size(0) != B or \
            pts_feature.size(0) != B or pts_feature.size(1) != N:
        raise RuntimeError("roipool3d: inconsistent tensor shapes")
    lib = C.lib()
    with torch.cuda.device(xyz.device):
        wsb = lib.prb_roipool3d_workspace_bytes(B, N, M, S)
        ws = torch.empty(wsb, dtype=torch.uint8, device=xyz.device)
        C.check(lib.prb_roipool3d_ws(B, N, M, Cf, S, C.ptr(xyz), C.ptr(boxes3d), C.ptr(pts_feature), C.ptr(pooled_features),
                                     C.ptr(pooled_empty_flag), C.ptr(rois_canonical), int(bool(zero_fill_empty)), C.ptr(ws),
                                     C.c_size_t(wsb), C.stream()), "roipool3d")
    return 1


def forward_one_pass(xyz, boxes3d, pts_feature, pooled_features, pooled_empty_flag, rois_canonical=None):
    """the one-kernel form (prb_roipool3d: no scratch, every box rescans the scene) -- kept for A/B measurements"""
    B, N = int(xyz.size(0)), int(xyz.size(1))
    M, Cf, S = int(boxes3d.size(1)), int(pts_feature.size(2)), int(pooled_features.size(2))
    with torch.cuda.device(xyz.device):
        C.check(C.lib().prb_roipool3d(B, N, M, Cf, S, C.ptr(xyz), C.ptr(boxes3d), C.ptr(pts_feature), C.ptr(pooled_features),
                                      C.ptr(pooled_empty_flag), C.ptr(rois_canonical), C.stream()), "roipool3d")
    return 1


forward_slow = forward


def _in_box_np(pts, box):
    """pt_in_box3d_cpu (roipool3d.cpp:82-95), vectorised over points; mixed float/double as in the source"""
    x, y, z = pts[:, 0], pts[:, 1], pts[:, 2]
    cx, by, cz, h, w, l, ang = [np.float32(v) for v in box]
    cy = np.float32(np.float64(by) - np.float64(h) / 2.0)
    # the source's rejecting form: a NaN difference or height passes these tests and leaves the decision to the rotation
    ok = ~((np.abs(x - cx) > np.float32(10.0)) | (np.abs(y - cy).astype(np.float64) > np.float64(h) / 2.0) |
           (np.abs(z - cz) > np.float32(10.0)))
    cosa, sina = np.float32(np.cos(ang)), np.float32(np.sin(ang))
    x_rot = (x - cx) * cosa + (z - cz) * (-sina)
    z_rot = (x - cx) * sina + (z - cz) * cosa
    hl, hw = np.float64(l) / 2.0, np.float64(w) / 2.0
    return ok & (x_rot >= -hl) & (x_rot <= hl) & (z_rot >= -hw) & (z_rot <= hw)


def pts_in_boxes3d_cpu(pts_flag, pts, boxes3d):
    p, b = pts.numpy().astype(np.float32), boxes3d.numpy().astype(np.float32)
    out = pts_flag.numpy()
    for i in range(b.shape[0]):
        out[i, :] = _in_box_np(p, b[i]).astype(np.int64)
    return 1


def roipool3d_cpu(pts, boxes3d, pts_feature, pooled_pts, pooled_features, pooled_empty_flag):
    p, b, f = pts.numpy(), boxes3d.numpy(), pts_feature.numpy()
    op, of, oe = pooled_pts.numpy(), pooled_features.numpy(), pooled_empty_flag.numpy()
    S = op.shape[1]
    oe[:] = 0
    for i in range(b.shape[0]):
        sel = np.nonzero(_in_box_np(p.astype(np.float32), b[i]))[0][:S]
        if sel.size == 0:
            oe[i] = 1
            continue
        sel = sel[np.arange(S) % sel.size] if sel.size < S else sel
        op[i] = p[sel]
        of[i] = f[sel]
    return 1
