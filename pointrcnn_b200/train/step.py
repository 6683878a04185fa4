"""One RPN training step on the H100 path (BASELINE configs[2]; reference: tools/train_rcnn.py:199-233 +
lib/net/train_functions.py:12-52): forward in training mode (batch-statistics BatchNorm, Dropout), bin-based loss,
backward, gradient all-reduce over the data-parallel ranks, optimizer step.

Forward / backward use the reference-shaped op-by-op path of the mirror modules: this repo's sampling / neighbour / grouping
/ interpolation natives with their scatter backward kernels (gather_points_grad, group_points_grad,
three_interpolate_grad), the shared MLPs through cuDNN / cuBLAS with torch autograd.  (The fused tensor-core chain is an
eval-mode kernel: batch-statistics BatchNorm couples all tiles of a launch.)  What this module adds over the reference's
loop: no `.item()` inside the loss, per-rank processes instead of nn.DataParallel's per-step replicate / scatter / gather,
and the bucketed all-reduce of `parallel_utils.GradBucketReducer` overlapped with backward.
"""
import numpy as np
import torch

from ..parallel_utils import GradBucketReducer
from ..rpn.stage import CLS_MEAN_SIZE, RPNStage
from .losses import rcnn_loss, rpn_loss


class RPNTrainer:
    def __init__(self, input_channels=1, device="cuda", world=1, lr=0.002, weight_decay=0.001, bucket_mb=4.0, seed=0):
        torch.manual_seed(seed)                       # identical initial weights on every rank
        self.device = torch.device(device)
        self.model = RPNStage(input_channels=input_channels, mode="TRAIN").to(self.device).train()
        self.params = [p for p in self.model.parameters() if p.requires_grad]
        self.reducer = GradBucketReducer(self.params, world=world, bucket_mb=bucket_mb)
        fused = self.device.type == "cuda"
        self.opt = torch.optim.Adam(self.params, lr=lr, weight_decay=weight_decay, **({"fused": True} if fused else {}))
        self.mean_size = torch.from_numpy(CLS_MEAN_SIZE[0]).to(self.device)

    def forward_loss(self, pts_input, rpn_cls_label, rpn_reg_label):
        m = self.model
        xyz, feats = m.backbone_net(pts_input)
        rpn_cls = m.rpn_cls_layer(feats).transpose(1, 2).contiguous()       # lib/net/rpn.py:76-77
        rpn_reg = m.rpn_reg_layer(feats).transpose(1, 2).contiguous()
        return rpn_loss(rpn_cls, rpn_reg, rpn_cls_label, rpn_reg_label, self.mean_size)

    def step(self, pts_input, rpn_cls_label, rpn_reg_label, grad_norm_clip=None):
        self.reducer.reset()
        loss, terms = self.forward_loss(pts_input, rpn_cls_label, rpn_reg_label)
        loss.backward()
        self.reducer.finish()
        if grad_norm_clip:
            torch.nn.utils.clip_grad_norm_(self.params, grad_norm_clip)     # train_utils.py: clip_grad_norm_(.., GRAD_NORM_CLIP)
        self.opt.step()
        return loss.detach(), terms


def synthetic_labels(pts_input, seed=0):
    """RPN labels of the right shapes / statistics for synthetic scenes (kitti_rcnn_dataset.py:generate_rpn_training_labels
    shapes): ~3 % foreground points, regression targets = offsets to a nearby box centre + size + heading"""
    B, N = pts_input.shape[0], pts_input.shape[1]
    g = torch.Generator().manual_seed(seed)
    cls = (torch.rand(B, N, generator=g) < 0.03).long()
    cls[torch.rand(B, N, generator=g) < 0.01] = -1
    reg = torch.zeros(B, N, 7)
    reg[..., 0:3] = torch.randn(B, N, 3, generator=g) * torch.tensor([1.0, 0.3, 1.0])
    reg[..., 3:6] = torch.from_numpy(CLS_MEAN_SIZE[0]) * (1 + 0.1 * torch.randn(B, N, 3, generator=g))
    reg[..., 6] = (torch.rand(B, N, generator=g) * 2 - 1) * float(np.pi)
    return cls.to(pts_input.device), reg.to(pts_input.device)


class RCNNTrainer:
    """One RCNN training step with the RPN fixed (the reference's second training phase: tools/train_rcnn.py --train_mode rcnn,
    cfg.RPN.FIXED): the RPN stage runs in eval mode without grad on the fused path and hands (rois, point features, mask,
    depth) to the RCNN stage, whose target layer samples 64 RoIs per scene; forward / backward of the RCNN network on the
    op-by-op path, get_rcnn_loss, bucketed gradient all-reduce, optimizer step."""

    def __init__(self, input_channels=1, device="cuda", world=1, lr=0.002, weight_decay=0.001, bucket_mb=4.0, seed=0, rpn_score_thresh=0.3):
        from ..rcnn.stage import RCNNStage
        torch.manual_seed(seed)
        self.device = torch.device(device)
        self.rpn = RPNStage(input_channels=input_channels, mode="TRAIN").to(self.device).eval()     # TRAIN quotas: 512 RoIs per scene
        for p in self.rpn.parameters():
            p.requires_grad_(False)
        self.model = RCNNStage(num_classes=2, input_channels=128).to(self.device).train()
        self.params = [p for p in self.model.parameters() if p.requires_grad]
        self.reducer = GradBucketReducer(self.params, world=world, bucket_mb=bucket_mb)
        self.opt = torch.optim.Adam(self.params, lr=lr, weight_decay=weight_decay, **({"fused": True} if self.device.type == "cuda" else {}))
        self.mean_size = torch.from_numpy(CLS_MEAN_SIZE[0]).to(self.device)
        self.rpn_score_thresh = rpn_score_thresh

    @torch.no_grad()
    def rpn_outputs(self, pts_input, gt_boxes3d):
        rois, _, rpn_cls, _, xyz, feats = self.rpn(pts_input, with_features=True)       # point_rcnn.py:36-55
        seg_mask = (torch.sigmoid(rpn_cls[:, :, 0]) > self.rpn_score_thresh).float()
        return {"rpn_xyz": xyz, "rpn_features": feats.permute(0, 2, 1).contiguous(), "seg_mask": seg_mask, "roi_boxes3d": rois,
                "pts_depth": torch.norm(xyz, p=2, dim=2), "gt_boxes3d": gt_boxes3d}

    def forward_loss(self, pts_input, gt_boxes3d):
        ret = self.model.forward_train(self.rpn_outputs(pts_input, gt_boxes3d))
        c = self.model.cfg
        return rcnn_loss(ret["rcnn_cls"], ret["rcnn_reg"], ret["cls_label"], ret["reg_valid_mask"], ret["roi_boxes3d"], ret["gt_of_rois"],
                         self.mean_size, loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"],
                         loc_y_by_bin=c["LOC_Y_BY_BIN"], loc_y_scope=c["LOC_Y_SCOPE"], loc_y_bin_size=c["LOC_Y_BIN_SIZE"])

    def forward_loss_offline(self, batch):
        """the ROI_SAMPLE_JIT=False branch of rcnn_net.forward (:155-163) + get_rcnn_loss on a batch of
        datasets.rcnn_offline.RCNNOfflineSampler.prepare_batch: the network reads the pooled rows as they are (no
        torch.cat of pts_input and pts_features), the targets are the batch's labels and canonical GT boxes"""
        rcnn_cls, rcnn_reg = self.model.forward_pts(batch["rows"])
        c = self.model.cfg
        return rcnn_loss(rcnn_cls, rcnn_reg, batch["cls_label"], batch["reg_valid_mask"], batch["roi_boxes3d"], batch["gt_boxes3d_ct"],
                         self.mean_size, loc_scope=c["LOC_SCOPE"], loc_bin_size=c["LOC_BIN_SIZE"], num_head_bin=c["NUM_HEAD_BIN"],
                         loc_y_by_bin=c["LOC_Y_BY_BIN"], loc_y_scope=c["LOC_Y_SCOPE"], loc_y_bin_size=c["LOC_Y_BIN_SIZE"])

    def step_offline(self, batch, grad_norm_clip=None):
        """one offline-recipe training step (tools/train_rcnn.py --train_mode rcnn_offline) on a prepared batch"""
        return self._step(self.forward_loss_offline, (batch,), grad_norm_clip)

    def step(self, pts_input, gt_boxes3d, grad_norm_clip=None):
        return self._step(self.forward_loss, (pts_input, gt_boxes3d), grad_norm_clip)

    def _step(self, forward_loss, args, grad_norm_clip):
        self.reducer.reset()
        loss, terms = forward_loss(*args)
        loss.backward()
        self.reducer.finish()
        if grad_norm_clip:
            torch.nn.utils.clip_grad_norm_(self.params, grad_norm_clip)
        self.opt.step()
        return loss.detach(), terms
