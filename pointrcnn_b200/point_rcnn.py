"""Two-stage inference on the H100 path without the reference tree: the eval branch of lib/net/point_rcnn.py:26-70 (RPN ->
proposal layer -> RCNN) and the detection post-processing of tools/eval_rcnn.py:485-620 (decode -> score threshold ->
rotated NMS) with the NMS scan on the device.  Sub-module names are the reference's (`rpn.*` = lib.net.rpn.RPN keys,
`rcnn_net.*` = lib.net.rcnn_net.RCNNNet keys), so a PointRCNN checkpoint loads as it is.
"""
import torch
import torch.nn as nn

from . import kitti_utils
from .bbox_transform import decode_bbox_target
from .iou3d import iou3d_utils
from .rcnn.stage import RCNNStage
from .rpn.stage import CLS_MEAN_SIZE, RPNStage


class PointRCNNInference(nn.Module):
    def __init__(self, input_channels=1, rpn_score_thresh=0.3, rcnn_score_thresh=0.3, rcnn_nms_thresh=0.1, rpn_cfg=None, rcnn_cfg=None):
        super().__init__()
        self.rpn = RPNStage(input_channels=input_channels, mode="TEST", cfg=rpn_cfg)
        self.rcnn_net = RCNNStage(num_classes=2, input_channels=128, cfg=rcnn_cfg)
        self.rpn_score_thresh = rpn_score_thresh            # cfg.RPN.SCORE_THRESH (default.yaml:59)
        self.rcnn_score_thresh = rcnn_score_thresh          # cfg.RCNN.SCORE_THRESH (default.yaml:125)
        self.rcnn_nms_thresh = rcnn_nms_thresh              # cfg.RCNN.NMS_THRESH (default.yaml:126)
        self.register_buffer("mean_size", torch.from_numpy(CLS_MEAN_SIZE[0]).clone(), persistent=False)

    def forward(self, pts_input):
        """pts_input (B,N,3+C) -> dict like PointRCNN.forward's eval output (point_rcnn.py:26-70)"""
        rois, roi_scores_raw, rpn_cls, rpn_reg, xyz, feats = self.rpn(pts_input, with_features=True)
        rpn_scores_raw = rpn_cls[:, :, 0]
        seg_mask = (torch.sigmoid(rpn_scores_raw) > self.rpn_score_thresh).float()
        pts_depth = torch.norm(xyz, p=2, dim=2)
        out = self.rcnn_net({"rpn_xyz": xyz, "rpn_features": feats.permute((0, 2, 1)), "seg_mask": seg_mask,
                             "roi_boxes3d": rois, "pts_depth": pts_depth})
        out.update(rois=rois, roi_scores_raw=roi_scores_raw, seg_result=seg_mask, rpn_cls=rpn_cls, rpn_reg=rpn_reg,
                   backbone_xyz=xyz, backbone_features=feats)
        return out

    def detections(self, out):
        """eval_rcnn.py:485-620: decode the RCNN regression relative to the RoIs, keep norm score > thresh, rotated NMS on
        the raw scores.  Returns per scene (boxes (K,7), raw scores (K)) on the device, plus the decoded (B,M,7) boxes."""
        rois = out["rois"]
        B, M = rois.shape[0], rois.shape[1]
        c = self.rcnn_net.cfg
        rcnn_cls = out["rcnn_cls"].view(B, M, -1)
        rcnn_reg = out["rcnn_reg"].view(B, M, -1)
        pred = decode_bbox_target(rois.reshape(-1, 7), rcnn_reg.reshape(-1, rcnn_reg.shape[-1]), anchor_size=self.mean_size,
                                  loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"],
                                  get_xz_fine=True, get_y_by_bin=c["LOC_Y_BY_BIN"], loc_y_scope=c["LOC_Y_SCOPE"],
                                  loc_y_bin_size=c["LOC_Y_BIN_SIZE"], get_ry_fine=True).view(B, M, 7)
        raw = rcnn_cls[:, :, 0]
        keep_mask = torch.sigmoid(raw) > self.rcnn_score_thresh
        res = []
        for k in range(B):
            sel = keep_mask[k]
            boxes_k, raw_k = pred[k][sel], raw[k][sel]
            if boxes_k.shape[0] == 0:
                res.append((boxes_k, raw_k))
                continue
            keep = iou3d_utils.nms_gpu(kitti_utils.boxes3d_to_bev_torch(boxes_k), raw_k, self.rcnn_nms_thresh).view(-1)
            res.append((boxes_k[keep], raw_k[keep]))
        return res, pred

    def detections_device(self, out):
        """detections() without a host round trip: the same decode / score threshold / rotated NMS, batched, results left
        on the device: (boxes (B,M,7) in descending raw-score order, raw scores (B,M), select (B,M) bool = the detections).
        Boxes under the score threshold are ordered LAST (score -inf) instead of being compacted away: greedy NMS visits
        boxes in order, so they cannot change which of the boxes above the threshold survive, and they are masked out
        afterwards -- the selected rows equal detections()'s per-scene lists, in the same order."""
        from .ext import iou3d_cuda
        rois = out["rois"]
        B, M = rois.shape[0], rois.shape[1]
        c = self.rcnn_net.cfg
        rcnn_cls = out["rcnn_cls"].view(B, M, -1)
        rcnn_reg = out["rcnn_reg"].view(B, M, -1)
        pred = decode_bbox_target(rois.reshape(-1, 7), rcnn_reg.reshape(-1, rcnn_reg.shape[-1]), anchor_size=self.mean_size,
                                  loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"],
                                  get_xz_fine=True, get_y_by_bin=c["LOC_Y_BY_BIN"], loc_y_scope=c["LOC_Y_SCOPE"],
                                  loc_y_bin_size=c["LOC_Y_BIN_SIZE"], get_ry_fine=True).view(B, M, 7)
        raw = rcnn_cls[:, :, 0]
        above = torch.sigmoid(raw) > self.rcnn_score_thresh
        order = torch.where(above, raw, torch.full_like(raw, float("-inf"))).sort(dim=1, descending=True)[1]
        boxes = torch.gather(pred, 1, order.unsqueeze(2).expand(B, M, 7)).contiguous()
        raw_s = torch.gather(raw, 1, order)
        n_above = above.sum(dim=1, keepdim=True)
        bev = kitti_utils.boxes3d_to_bev_torch(boxes.view(-1, 7)).view(B, M, 5).contiguous()
        select = torch.zeros((B, M), dtype=torch.bool, device=rois.device)
        pos = torch.arange(M, device=rois.device)
        for k in range(B):                                   # launches only; nothing comes back to the host
            keep, num = iou3d_cuda.nms_device(bev[k], self.rcnn_nms_thresh, 0)
            kept = (pos < num.to(torch.int64)).float()       # keep[:num] are the surviving positions; the tail of keep is undefined
            select[k] = torch.zeros(M, device=rois.device).scatter_add_(0, keep.clamp(0, M - 1), kept) > 0
        select &= pos.unsqueeze(0) < n_above
        return boxes, raw_s, select
