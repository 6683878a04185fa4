"""Mirror of lib/utils/roipool3d/roipool3d_utils.py (reference :7-108): roipool3d_gpu, pts_in_boxes3d_cpu,
roipool_pc_cpu, roipool3d_cpu -- same signatures, on top of the H100 `roipool3d_cuda` natives.

Extra: roipool3d_gpu(..., canonical_rois=rois) fuses the canonical transform of lib/net/rcnn_net.py:146-152
into the pooling kernel's store.
"""
import numpy as np
import torch

from ..ext import roipool3d_cuda

try:
    import lib.utils.kitti_utils as kitti_utils
except ImportError:
    from .. import kitti_utils


def roipool3d_gpu(pts, pts_feature, boxes3d, pool_extra_width, sampled_pt_num=512, canonical_rois=None):
    """pts (B,N,3), pts_feature (B,N,C), boxes3d (B,M,7) -> pooled (B,M,S,3+C), empty_flag (B,M) int32"""
    batch_size, boxes_num, feature_len = pts.shape[0], boxes3d.shape[1], pts_feature.shape[2]
    pooled_boxes3d = kitti_utils.enlarge_box3d(boxes3d.view(-1, 7), pool_extra_width).view(batch_size, -1, 7)
    # the kernel zeroes the rows of empty boxes itself: no 558 MB memset in front of it (values equal the reference's)
    pooled_features = torch.empty((batch_size, boxes_num, sampled_pt_num, 3 + feature_len), dtype=torch.float32,
                                  device=pts.device)
    pooled_empty_flag = torch.zeros((batch_size, boxes_num), dtype=torch.int32, device=pts.device)
    roipool3d_cuda.forward(pts.contiguous(), pooled_boxes3d.contiguous(), pts_feature.contiguous(), pooled_features,
                           pooled_empty_flag, None if canonical_rois is None else canonical_rois.contiguous(), zero_fill_empty=True)
    return pooled_features, pooled_empty_flag


def pts_in_boxes3d_cpu(pts, boxes3d):
    """pts (N,3), boxes3d (M,7) -> list of M bool masks (N)"""
    if not pts.is_cuda:
        pts = pts.float().contiguous()
        boxes3d = boxes3d.float().contiguous()
        pts_flag = torch.zeros((boxes3d.size(0), pts.size(0)), dtype=torch.int64)
        roipool3d_cuda.pts_in_boxes3d_cpu(pts_flag, pts, boxes3d)
        return [pts_flag[k] > 0 for k in range(boxes3d.shape[0])]
    raise NotImplementedError


def roipool_pc_cpu(pts, pts_feature, boxes3d, sampled_pt_num):
    pts = pts.cpu().float().contiguous()
    pts_feature = pts_feature.cpu().float().contiguous()
    boxes3d = boxes3d.cpu().float().contiguous()
    assert pts.shape[0] == pts_feature.shape[0] and pts.shape[1] == 3, '%s %s' % (pts.shape, pts_feature.shape)
    pooled_pts = torch.zeros((boxes3d.shape[0], sampled_pt_num, 3), dtype=torch.float32)
    pooled_features = torch.zeros((boxes3d.shape[0], sampled_pt_num, pts_feature.shape[1]), dtype=torch.float32)
    pooled_empty_flag = torch.zeros(boxes3d.shape[0], dtype=torch.int64)
    roipool3d_cuda.roipool3d_cpu(pts, boxes3d, pts_feature, pooled_pts, pooled_features, pooled_empty_flag)
    return pooled_pts, pooled_features, pooled_empty_flag


def roipool3d_cpu(boxes3d, pts, pts_feature, pts_extra_input, pool_extra_width, sampled_pt_num=512,
                  canonical_transform=True):
    pooled_boxes3d = kitti_utils.enlarge_box3d(boxes3d, pool_extra_width)
    pts_feature_all = np.concatenate((pts_extra_input, pts_feature), axis=1)
    pooled_pts, pooled_features, pooled_empty_flag = roipool_pc_cpu(
        torch.from_numpy(pts), torch.from_numpy(pts_feature_all), torch.from_numpy(pooled_boxes3d), sampled_pt_num)
    extra_input_len = pts_extra_input.shape[1]
    sampled_pts_input = torch.cat((pooled_pts, pooled_features[:, :, 0:extra_input_len]), dim=2).numpy()
    sampled_pts_feature = pooled_features[:, :, extra_input_len:].numpy()
    if canonical_transform:
        roi_ry = boxes3d[:, 6] % (2 * np.pi)
        roi_center = boxes3d[:, 0:3]
        sampled_pts_input[:, :, 0:3] = sampled_pts_input[:, :, 0:3] - roi_center[:, np.newaxis, :]
        for k in range(sampled_pts_input.shape[0]):
            c, s = np.cos(roi_ry[k]), np.sin(roi_ry[k])
            rot = np.array([[c, -s], [s, c]])
            sampled_pts_input[k][:, [0, 2]] = np.dot(sampled_pts_input[k][:, [0, 2]], rot.T)
        return sampled_pts_input, sampled_pts_feature
    return sampled_pts_input, sampled_pts_feature, pooled_empty_flag.numpy()
