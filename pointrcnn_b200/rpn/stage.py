"""The whole RPN stage of lib/net/rpn.py:11-94 on the H100 path, without the reference tree or its global EasyDict:

    Pointnet2MSG backbone -> rpn_cls_layer / rpn_reg_layer -> ProposalLayer (eval: rois + roi scores)

Same sub-module and parameter names as lib.net.rpn.RPN (`backbone_net`, `rpn_cls_layer.0.conv` ..., `rpn_reg_layer`,
`proposal_layer`), so a reference RPN checkpoint loads as it is.  Used by bench.py's end-to-end leg and the chain tests;
with the reference tree present, `dropin.activate()` + the unchanged lib/net/rpn.py build the same thing.
"""
import types

import numpy as np
import torch
import torch.nn as nn

from ..backbone import Pointnet2MSG
from ..pointnet2 import pytorch_utils as pt_utils
from .heads import invalidate_heads, rpn_heads
from .proposal_layer import ProposalLayer

# tools/cfgs/default.yaml:19
CLS_MEAN_SIZE = np.array([[1.52563191462, 1.62856739989, 3.88311640418]], dtype=np.float32)


class _Cfg(dict):
    __getattr__ = dict.__getitem__


def default_cfg(nms_type="normal", distance_based=True):
    """the slice of tools/cfgs/default.yaml the proposal layer reads (:19, :29-37, :156-165)"""
    ns = types.SimpleNamespace
    c = _Cfg(TEST=ns(RPN_PRE_NMS_TOP_N=9000, RPN_POST_NMS_TOP_N=100, RPN_NMS_THRESH=0.8, RPN_DISTANCE_BASED_PROPOSE=distance_based),
             TRAIN=ns(RPN_PRE_NMS_TOP_N=9000, RPN_POST_NMS_TOP_N=512, RPN_NMS_THRESH=0.85, RPN_DISTANCE_BASED_PROPOSE=True))
    c["CLS_MEAN_SIZE"] = CLS_MEAN_SIZE
    c["RPN"] = ns(LOC_SCOPE=3.0, LOC_BIN_SIZE=0.5, NUM_HEAD_BIN=12, LOC_XZ_FINE=True, NMS_TYPE=nms_type)
    return c


class RPNStage(nn.Module):
    def __init__(self, input_channels=1, mode="TEST", cfg=None, reg_channel=76):
        super().__init__()
        self.backbone_net = Pointnet2MSG(input_channels=input_channels)
        # lib/net/rpn.py:19-47 (cls: [128] + 1, reg: [128] + reg_channel, Dropout(0.5) at index 1)
        self.rpn_cls_layer = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 1, activation=None))
        self.rpn_reg_layer = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5),
                                           pt_utils.Conv1d(128, reg_channel, activation=None))
        self.proposal_layer = ProposalLayer(mode=mode, cfg=cfg if cfg is not None else default_cfg())
        self.backbone_net.FP_modules[0].emit_point_major = True      # the fused heads read the point-major twin

    def _apply(self, fn, *args, **kwargs):
        invalidate_heads(self)         # see _PointnetSAModuleBase._apply; the backbone modules drop their own chains
        return super()._apply(fn, *args, **kwargs)

    def invalidate_fused(self):
        """call after editing weights through `.data` (EMA, weight averaging): drops every packed chain of the stage"""
        invalidate_heads(self)
        for m in self.backbone_net.modules():
            if hasattr(m, "invalidate_fused"):
                m.invalidate_fused()

    def forward(self, pts_input, with_features=False):
        """pts_input (B,N,3+C) -> (rois (B,M,7), roi_scores_raw (B,M)) [+ rpn_cls, rpn_reg, backbone_xyz, backbone_features]"""
        xyz, feats = self.backbone_net(pts_input)
        rpn_cls, rpn_reg = rpn_heads(self, feats)                     # (B,N,1), (B,N,reg)
        rois, scores = self.proposal_layer(rpn_cls[:, :, 0], rpn_reg, xyz)
        if with_features:
            return rois, scores, rpn_cls, rpn_reg, xyz, feats
        return rois, scores
