"""The RCNN (stage-2) network of lib/net/rcnn_net.py:14-190 on the H100 path, eval / inference branch, without the
reference tree or its global EasyDict:

    roipool3d (+ canonical transform, fused) -> xyz_up_layer + merge_down_layer -> 3 PointnetSAModule -> cls / reg heads

Same sub-module and parameter names as lib.net.rcnn_net.RCNNNet (`xyz_up_layer.layer0.conv`, `merge_down_layer`,
`SA_modules.k.mlps.0.layer{j}.conv`, `cls_layer.{0,2,3}.conv`, `reg_layer...`), so a reference RCNN checkpoint loads as
it is.  With the reference tree present, `dropin.activate()` + the unchanged lib/net/rcnn_net.py build the same thing on
the same natives; this class exists so benches and GPU tests run on the box, where /root/reference does not exist.
"""
import contextlib

import torch
import torch.nn as nn

from .. import config
from ..pointnet2 import pointnet2_modules as pn2
from ..pointnet2 import pytorch_utils as pt_utils
from ..pointnet2.pointnet2_modules import PointnetSAModule
from ..roipool3d import roipool3d_utils

# tools/cfgs/default.yaml:78-110
RCNN_DEFAULT = dict(
    USE_RPN_FEATURES=True, USE_INTENSITY=False, USE_MASK=True, USE_DEPTH=True, USE_BN=False, DP_RATIO=0.0,
    XYZ_UP_LAYER=[128, 128], NUM_POINTS=512, POOL_EXTRA_WIDTH=1.0,
    NPOINTS=[128, 32, -1], RADIUS=[0.2, 0.4, 100], NSAMPLE=[64, 64, 64],
    MLPS=[[128, 128, 128], [128, 128, 256], [256, 256, 512]],
    CLS_FC=[256, 256], REG_FC=[256, 256],
    LOC_SCOPE=1.5, LOC_BIN_SIZE=0.5, NUM_HEAD_BIN=9, LOC_Y_BY_BIN=False, LOC_Y_SCOPE=0.5, LOC_Y_BIN_SIZE=0.25,
)


class RCNNStage(nn.Module):
    def __init__(self, num_classes=2, input_channels=128, use_xyz=True, cfg=None):
        super().__init__()
        c = dict(RCNN_DEFAULT, **(cfg or {}))
        self.cfg = c
        self._fused_rows = None
        self.SA_modules = nn.ModuleList()
        channel_in = input_channels
        if c["USE_RPN_FEATURES"]:
            self.rcnn_input_channel = 3 + int(c["USE_INTENSITY"]) + int(c["USE_MASK"]) + int(c["USE_DEPTH"])
            self.xyz_up_layer = pt_utils.SharedMLP([self.rcnn_input_channel] + c["XYZ_UP_LAYER"], bn=c["USE_BN"])
            c_out = c["XYZ_UP_LAYER"][-1]
            self.merge_down_layer = pt_utils.SharedMLP([c_out * 2, c_out], bn=c["USE_BN"])
        for k in range(len(c["NPOINTS"])):
            mlps = [channel_in] + list(c["MLPS"][k])
            npoint = c["NPOINTS"][k] if c["NPOINTS"][k] != -1 else None
            self.SA_modules.append(PointnetSAModule(npoint=npoint, radius=c["RADIUS"][k], nsample=c["NSAMPLE"][k], mlp=mlps,
                                                    use_xyz=use_xyz, bn=c["USE_BN"]))
            channel_in = mlps[-1]
        cls_channel = 1 if num_classes == 2 else num_classes
        self.cls_layer = self._head(channel_in, c["CLS_FC"], cls_channel, c)
        per_loc_bin_num = int(c["LOC_SCOPE"] / c["LOC_BIN_SIZE"]) * 2
        loc_y_bin_num = int(c["LOC_Y_SCOPE"] / c["LOC_Y_BIN_SIZE"]) * 2
        reg_channel = per_loc_bin_num * 4 + c["NUM_HEAD_BIN"] * 2 + 3 + (1 if not c["LOC_Y_BY_BIN"] else loc_y_bin_num * 2)
        self.reg_channel = reg_channel
        self.reg_layer = self._head(channel_in, c["REG_FC"], reg_channel, c)
        for m in self.modules():                                   # rcnn_net.py:86-105 (xavier)
            if isinstance(m, (nn.Conv2d, nn.Conv1d)):
                nn.init.xavier_normal_(m.weight)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
        nn.init.normal_(self.reg_layer[-1].conv.weight, mean=0, std=0.001)

    @staticmethod
    def _head(pre, fcs, out_ch, c):
        layers = []
        for k in fcs:
            layers.append(pt_utils.Conv1d(pre, k, bn=c["USE_BN"]))
            pre = k
        layers.append(pt_utils.Conv1d(pre, out_ch, activation=None))
        if c["DP_RATIO"] >= 0:
            layers.insert(1, nn.Dropout(c["DP_RATIO"]))
        return nn.Sequential(*layers)

    def _apply(self, fn, *args, **kwargs):
        self._fused_rows = None
        return super()._apply(fn, *args, **kwargs)

    def invalidate_fused(self):
        """call after editing weights without bumping their versions (`.data` edits, CUDA graph replays): drops the packed
        row chains and every SA module's chain"""
        self._fused_rows = None
        for m in self.SA_modules:
            m.invalidate_fused()

    def _rows_fusable(self, pts_input):
        if config.get("disable_fused") or not pts_input.is_cuda or pts_input.dtype != torch.float32 or not pts_input.is_contiguous():
            return False
        if pn2._needs_graph(self, pts_input):
            return False
        return pn2._FusedMLP.supported(self.xyz_up_layer) and pn2._FusedMLP.supported(self.merge_down_layer)

    def pool(self, rpn_xyz, rpn_features, seg_mask, pts_depth, roi_boxes3d, rpn_intensity=None):
        """rcnn_net.py:127-152: pts_feature = [intensity?, seg_mask, depth/70-0.5, rpn features]; roipool3d; canonical
        transform (fused into the pooling kernel).  -> pts_input (B*M, NUM_POINTS, 3 + extra + C), empty flags (B,M)"""
        c = self.cfg
        extra = ([rpn_intensity.unsqueeze(2)] if c["USE_INTENSITY"] else []) + [seg_mask.unsqueeze(2)]
        if c["USE_DEPTH"]:
            extra.append((pts_depth / 70.0 - 0.5).unsqueeze(2))
        pts_feature = torch.cat(extra + [rpn_features], dim=2)
        pooled, empty = roipool3d_utils.roipool3d_gpu(rpn_xyz, pts_feature, roi_boxes3d, c["POOL_EXTRA_WIDTH"],
                                                      sampled_pt_num=c["NUM_POINTS"], canonical_rois=roi_boxes3d)
        return pooled.view(-1, pooled.shape[2], pooled.shape[3]), empty

    def forward_pts(self, pts_input):
        """rcnn_net.py:165-190 on pooled, canonical points (R, NUM_POINTS, 3 + extra + C) -> rcnn_cls (R, cls), rcnn_reg (R, reg)"""
        xyz = pts_input[..., 0:3].contiguous()
        if self.cfg["USE_RPN_FEATURES"] and self._rows_fusable(pts_input):
            # tensor-core row chains straight on the pooled rows: xyz_up reads the first columns of every row, merge reads
            # [xyz feature | the row's RPN feature columns]; the result is already the point-major layout SA 1 gathers from
            R, P, W = pts_input.shape
            rows = pts_input.view(R * P, W)
            ci = self.rcnn_input_channel
            if self._fused_rows is None:
                self._fused_rows = (pn2._FusedMLP(), pn2._FusedMLP())
            up = pn2.rows_mlp(self._fused_rows[0], self.xyz_up_layer, rows[:, :ci], tag="rcnn_rows_mlp")
            merged = pn2.rows_mlp(self._fused_rows[1], self.merge_down_layer, up, rows[:, ci:], tag="rcnn_rows_mlp").view(R, P, -1)
            l_xyz, l_features = [xyz], [pn2._attach_pm(merged.transpose(1, 2), merged)]
        elif self.cfg["USE_RPN_FEATURES"]:
            xyz_input = pts_input[..., 0:self.rcnn_input_channel].transpose(1, 2).unsqueeze(dim=3)
            xyz_feature = self.xyz_up_layer(xyz_input)
            rpn_feature = pts_input[..., self.rcnn_input_channel:].transpose(1, 2).unsqueeze(dim=3)
            merged = self.merge_down_layer(torch.cat((xyz_feature, rpn_feature), dim=1))
            l_xyz, l_features = [xyz], [merged.squeeze(dim=3)]
        else:
            l_xyz, l_features = [xyz], [pts_input[..., 3:].transpose(1, 2).contiguous() if pts_input.size(-1) > 3 else None]
        for i in range(len(self.SA_modules)):
            li_xyz, li_features = self.SA_modules[i](l_xyz[i], l_features[i])
            l_xyz.append(li_xyz)
            l_features.append(li_features)
        rcnn_cls = self.cls_layer(l_features[-1]).transpose(1, 2).contiguous().squeeze(dim=1)
        rcnn_reg = self.reg_layer(l_features[-1]).transpose(1, 2).contiguous().squeeze(dim=1)
        return rcnn_cls, rcnn_reg

    def forward_train(self, input_data, target_layer=None, target_draw=None):
        """training branch of RCNNNet.forward with cfg.RCNN.ROI_SAMPLE_JIT (rcnn_net.py:119-126, :165-190): the target layer
        (RoI sampling, pooling, augmentation, canonical transform, labels -- no grad) then the network on the sampled RoIs.
        input_data: the eval keys + gt_boxes3d (B,G,7).  target_draw: "torch" / "device" for this call (the config switch
        target_draw, which a layer built with draw=None follows), None leaves the switch as it is.  -> the reference's
        ret_dict: rcnn_cls, rcnn_reg + the target dict (cls_label, reg_valid_mask, gt_of_rois, roi_boxes3d, pts_input, ...)."""
        if target_layer is None:
            if getattr(self, "proposal_target_layer", None) is None:
                from ..rpn.proposal_target_layer import ProposalTargetLayer
                self.proposal_target_layer = ProposalTargetLayer()
            target_layer = self.proposal_target_layer
        # the targets are geometry, not network: fp32 under autocast too (the canonical rotation is a matmul)
        fp32 = torch.autocast("cuda", enabled=False) if torch.is_autocast_enabled("cuda") else contextlib.nullcontext()
        with torch.no_grad(), fp32, config.override(**({"target_draw": target_draw} if target_draw is not None else {})):
            target = target_layer(input_data)
            target["pts_input"] = torch.cat((target["sampled_pts"], target["pts_feature"]), dim=2)
        rcnn_cls, rcnn_reg = self.forward_pts(target["pts_input"])
        ret = {"rcnn_cls": rcnn_cls, "rcnn_reg": rcnn_reg}
        ret.update(target)
        return ret

    def forward(self, input_data):
        """eval branch of RCNNNet.forward with cfg.RCNN.ROI_SAMPLE_JIT: input dict keys rpn_xyz (B,N,3), rpn_features (B,N,C),
        seg_mask (B,N), pts_depth (B,N), roi_boxes3d (B,M,7) [, rpn_intensity] -> {'rcnn_cls', 'rcnn_reg'}"""
        pts_input, empty = self.pool(input_data["rpn_xyz"], input_data["rpn_features"], input_data["seg_mask"],
                                     input_data["pts_depth"], input_data["roi_boxes3d"], input_data.get("rpn_intensity"))
        rcnn_cls, rcnn_reg = self.forward_pts(pts_input)
        return {"rcnn_cls": rcnn_cls, "rcnn_reg": rcnn_reg, "pooled_empty_flag": empty}
