"""Mirror of lib/utils/iou3d/iou3d_utils.py (reference :6-87): boxes_iou_bev, boxes_iou3d_gpu, nms_gpu,
nms_normal_gpu -- same signatures and return values, on top of the H100 `iou3d_cuda` natives.

nms_gpu / nms_normal_gpu keep the reference contract (sorted by score, returns original indices of the kept
boxes, int64 on the GPU) but run the greedy scan on the device: one 4-byte D2H for the count instead of a
5 MB mask copy + host loop + H2D of the keep list (iou3d.cpp:86-116, iou3d_utils.py:85-87).
"""
import torch

from ..ext import iou3d_cuda

try:  # inside the reference tree use its own helpers, as the reference module does
    import lib.utils.kitti_utils as kitti_utils
except ImportError:  # standalone
    from .. import kitti_utils


def boxes_iou_bev(boxes_a, boxes_b):
    """boxes_a (M,5), boxes_b (N,5) -> (M,N) rotated BEV IoU"""
    ans_iou = torch.zeros((boxes_a.shape[0], boxes_b.shape[0]), dtype=torch.float32, device=boxes_a.device)
    iou3d_cuda.boxes_iou_bev_gpu(boxes_a.contiguous(), boxes_b.contiguous(), ans_iou)
    return ans_iou


def boxes_iou3d_gpu(boxes_a, boxes_b):
    """boxes_a (N,7), boxes_b (M,7) [x,y,z,h,w,l,ry] -> (N,M) 3D IoU"""
    boxes_a_bev = kitti_utils.boxes3d_to_bev_torch(boxes_a)
    boxes_b_bev = kitti_utils.boxes3d_to_bev_torch(boxes_b)
    overlaps_bev = torch.zeros((boxes_a.shape[0], boxes_b.shape[0]), dtype=torch.float32, device=boxes_a.device)
    iou3d_cuda.boxes_overlap_bev_gpu(boxes_a_bev.contiguous(), boxes_b_bev.contiguous(), overlaps_bev)

    boxes_a_height_min = (boxes_a[:, 1] - boxes_a[:, 3]).view(-1, 1)
    boxes_a_height_max = boxes_a[:, 1].view(-1, 1)
    boxes_b_height_min = (boxes_b[:, 1] - boxes_b[:, 3]).view(1, -1)
    boxes_b_height_max = boxes_b[:, 1].view(1, -1)
    max_of_min = torch.max(boxes_a_height_min, boxes_b_height_min)
    min_of_max = torch.min(boxes_a_height_max, boxes_b_height_max)
    overlaps_h = torch.clamp(min_of_max - max_of_min, min=0)

    overlaps_3d = overlaps_bev * overlaps_h
    vol_a = (boxes_a[:, 3] * boxes_a[:, 4] * boxes_a[:, 5]).view(-1, 1)
    vol_b = (boxes_b[:, 3] * boxes_b[:, 4] * boxes_b[:, 5]).view(1, -1)
    return overlaps_3d / torch.clamp(vol_a + vol_b - overlaps_3d, min=1e-7)


def _nms(boxes, scores, thresh, normal):
    order = scores.sort(0, descending=True)[1]
    boxes = boxes[order].contiguous()
    keep, num = iou3d_cuda.nms_device(boxes, thresh, normal)
    num_out = int(num.item())
    return order[keep[:num_out]].contiguous()


def nms_gpu(boxes, scores, thresh):
    """rotated NMS: boxes (N,5) [x1,y1,x2,y2,ry], scores (N) -> kept original indices (int64, cuda)"""
    return _nms(boxes, scores, thresh, 0)


def nms_normal_gpu(boxes, scores, thresh):
    """axis-aligned NMS with the same interface"""
    return _nms(boxes, scores, thresh, 1)
