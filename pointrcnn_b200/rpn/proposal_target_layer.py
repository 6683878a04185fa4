"""RCNN target assignment: mirror of lib/rpn/proposal_target_layer.py:10-374 (same class name, forward(input_dict) keys and
output dict) with the IoU work batched onto the fused 3D-IoU kernels (SURVEY.md section 8(f) rank 2).

What the reference does per training step (B scenes, 512 RoIs each, 64 sampled):
  * `sample_rois_for_rcnn`: per scene one `boxes_iou3d_gpu` call (2 BEV conversions + overlap kernel + ~12 torch kernels),
    index-set sampling with numpy / torch CPU random numbers, then `aug_roi_by_noise_torch`: a Python `while` loop PER
    SAMPLED ROI that draws a jittered box and calls `boxes_iou3d_gpu` on ONE pair, reads the value back (`temp_iou <
    pos_thresh` synchronises), up to ROI_FG_AUG_TIMES = 10 times: up to 64 x B x 10 tiny launches + host syncs.
  * RoI pooling, optional augmentation, canonical transform, labels.
Here:
  * ONE `prb_boxes_iou3d` launch computes every (RoI, GT) pair of the batch (same values as the reference's sequence, bit
    for bit -- tests/test_gpu_ops.py);
  * the index-set sampling keeps the reference's code path and its random calls, in the same order, so that with the
    jitter loop disabled (ROI_FG_AUG_TIMES = 0, AUG_DATA off) the layer reproduces the reference exactly for a given
    numpy / torch seed (tests/golden/proposal_target_layer.npz: outputs of the reference's own Python);
  * the jitter loop runs for ALL sampled RoIs of ALL scenes at once: round t draws the candidates of every still-active
    RoI in one shot and scores them with ONE `prb_boxes_iou3d_aligned` launch -- at most ROI_FG_AUG_TIMES launches and
    no per-RoI host sync.  Per RoI the process is the reference's (keep the original with p = 0.2, else jitter; stop at
    the first candidate reaching the foreground threshold or after aug_times draws; last candidate wins); the random
    STREAM differs (one batched draw per round instead of per-RoI draws), so augmented boxes are equal in distribution,
    not bit for bit.
With draw="device" (or draw=None and config switch target_draw = "device") the whole layer runs on the device without a
host read: rcnn/targets.py runs prb_boxes_iou3d, csrc/rcnn_sample.cu's sample stage, prb_roipool3d_ws and the targets
stage in the layer's recipe (targets.layer_recipe).  Random draws are counter-based hashes of
(seed, scene, stage, row, try, slot): the reference's distribution, not its stream.  The seed is the layer's call
counter unless forward(..., seed=) gives one.  After use_device_seed() the seed is a device int32 counter instead, which
each call reads and then advances on the device, so a CUDA graph that captured the call draws anew on every replay.
Extra output keys: sample_status (B) int32 (0 ok, 1 no fg and no bg RoI -- the reference stops in pdb --, 2 no GT -- the
reference raises; such a scene's rows have cls_label -1 and reg_valid_mask 0) and sample_index (B * ROI_PER_IMAGE, 3) int32 [source RoI, GT, jitter tries].
"""
import numpy as np
import torch
import torch.nn as nn

from .. import _cabi as C
from .. import config, kitti_utils
from ..ext import iou3d_cuda
from ..rcnn import targets
from ..rcnn.targets import AUG_METHODS, DEFAULT_CFG, ns as _ns  # noqa: F401  (the names this module has always exported)
from ..roipool3d import roipool3d_utils

# REG_AUG_METHOD 'multiple' (proposal_target_layer.py:278-284): [pos_range, hwl_range, angle_range]
_RANGE_CONFIG = [[0.2, 0.1, np.pi / 12], [0.3, 0.15, np.pi / 12], [0.5, 0.15, np.pi / 9], [0.8, 0.15, np.pi / 6], [1.0, 0.15, np.pi / 3]]
DRAWS = ("torch", "device")


def boxes_iou3d(boxes_a, boxes_b):
    """(M,7) x (N,7) -> (M,N): iou3d_utils.boxes_iou3d_gpu in one launch"""
    return iou3d_cuda.boxes_iou3d(boxes_a.contiguous().float(), boxes_b.contiguous().float())


class ProposalTargetLayer(nn.Module):
    """draw: "torch" (the reference's random calls), "device" (one pass on the device, hashed draws) or None (the
    target_draw switch of pointrcnn_b200.config, read at every call; "torch" unless changed)"""

    def __init__(self, cfg=None, draw=None):
        super().__init__()
        if cfg is None:
            try:
                from lib.config import cfg as ref_cfg      # inside the reference tree: its own global config
                cfg = ref_cfg
            except ImportError:
                cfg = _ns(DEFAULT_CFG)
        if draw is not None and draw not in DRAWS:
            raise ValueError("draw must be one of %s, not %r" % (DRAWS, draw))
        self.cfg = cfg
        self.draw = draw
        self.calls = 0
        self.seed_counter = None

    def use_device_seed(self, device):
        """draw="device" calls without seed= read their seed from a device int32 counter, started at the call count, and
        advance it on the device"""
        self.seed_counter = torch.full((1,), self.calls, dtype=torch.int32, device=device)

    def _pts_feature(self, input_dict):
        """[intensity?, seg_mask, pts_depth / 70 - 0.5?, rpn_features] (:19-32)"""
        cfg = self.cfg
        extra = ([input_dict['rpn_intensity'].unsqueeze(dim=2)] if cfg.RCNN.USE_INTENSITY else []) + [input_dict['seg_mask'].unsqueeze(dim=2)]
        if cfg.RCNN.USE_DEPTH:
            extra.append((input_dict['pts_depth'] / 70.0 - 0.5).unsqueeze(dim=2))
        return torch.cat(extra + [input_dict['rpn_features']], dim=2)

    # ------------------------------------------------------------------ forward (proposal_target_layer.py:14-76)
    def forward(self, input_dict, seed=None):
        draw = self.draw or config.get("target_draw")
        if draw not in DRAWS:
            raise ValueError("target_draw must be one of %s, not %r" % (DRAWS, draw))
        explicit = seed is not None
        seed = self.calls if seed is None else seed
        self.calls += 1
        if draw == "device":
            return self.forward_device(input_dict, seed if explicit or self.seed_counter is None else None)
        cfg = self.cfg
        roi_boxes3d, gt_boxes3d = input_dict['roi_boxes3d'], input_dict['gt_boxes3d']
        batch_rois, batch_gt_of_rois, batch_roi_iou = self.sample_rois_for_rcnn(roi_boxes3d, gt_boxes3d)

        rpn_xyz = input_dict['rpn_xyz']
        pts_feature = self._pts_feature(input_dict)
        pooled_features, pooled_empty_flag = roipool3d_utils.roipool3d_gpu(rpn_xyz, pts_feature, batch_rois, cfg.RCNN.POOL_EXTRA_WIDTH,
                                                                           sampled_pt_num=cfg.RCNN.NUM_POINTS)
        sampled_pts, sampled_features = pooled_features[:, :, :, 0:3], pooled_features[:, :, :, 3:]
        if cfg.AUG_DATA:
            sampled_pts, batch_rois, batch_gt_of_rois = self.data_augmentation(sampled_pts, batch_rois, batch_gt_of_rois)

        # canonical transformation (:45-56), all scenes at once: rows are independent
        B, M = batch_rois.shape[0], batch_rois.shape[1]
        roi_ry = batch_rois[:, :, 6] % (2 * np.pi)
        roi_center = batch_rois[:, :, 0:3]
        sampled_pts = sampled_pts - roi_center.unsqueeze(dim=2)
        batch_gt_of_rois[:, :, 0:3] = batch_gt_of_rois[:, :, 0:3] - roi_center
        batch_gt_of_rois[:, :, 6] = batch_gt_of_rois[:, :, 6] - roi_ry
        sampled_pts = kitti_utils.rotate_pc_along_y_torch(sampled_pts.reshape(B * M, -1, 3), batch_rois[:, :, 6].reshape(-1)).view(B, M, -1, 3)
        batch_gt_of_rois = kitti_utils.rotate_pc_along_y_torch(batch_gt_of_rois.reshape(B * M, 1, 7), roi_ry.reshape(-1)).view(B, M, 7)

        valid_mask = (pooled_empty_flag == 0)
        reg_valid_mask = ((batch_roi_iou > cfg.RCNN.REG_FG_THRESH) & valid_mask).long()
        batch_cls_label = (batch_roi_iou > cfg.RCNN.CLS_FG_THRESH).long()
        invalid_mask = (batch_roi_iou > cfg.RCNN.CLS_BG_THRESH) & (batch_roi_iou < cfg.RCNN.CLS_FG_THRESH)
        batch_cls_label[valid_mask == 0] = -1
        batch_cls_label[invalid_mask > 0] = -1
        return {'sampled_pts': sampled_pts.reshape(-1, cfg.RCNN.NUM_POINTS, 3),
                'pts_feature': sampled_features.reshape(-1, cfg.RCNN.NUM_POINTS, sampled_features.shape[3]),
                'cls_label': batch_cls_label.view(-1), 'reg_valid_mask': reg_valid_mask.view(-1),
                'gt_of_rois': batch_gt_of_rois.view(-1, 7), 'gt_iou': batch_roi_iou.view(-1), 'roi_boxes3d': batch_rois.view(-1, 7)}

    # ------------------------------------------------------------------ the device path
    def forward_device(self, input_dict, seed):
        """forward() in four device launches and no host read: 3D IoU of every (RoI, GT) pair, the sample stage (selection +
        jitter loop), RoI pooling on the enlarged jittered boxes, the targets stage (augmentation, labels, canonical
        transform).  seed None: the device counter's value, which the call then advances.  Same keys and shapes as the torch path, plus sample_status and sample_index."""
        recipe = targets.layer_recipe(self.cfg)
        rois = input_dict['roi_boxes3d'][:, :, 0:7].contiguous().float()
        gts = input_dict['gt_boxes3d'][:, :, 0:7].contiguous().float()
        xyz = input_dict['rpn_xyz'].contiguous().float()
        C.require_cuda(rois, gts, xyz)
        with torch.cuda.device(rois.device):
            feat = self._pts_feature(input_dict).contiguous().float()
            counter = self.seed_counter if seed is None else None
            o = targets.run(recipe, xyz, feat, rois, gts, None, 0 if seed is None else seed, seed_dev=counter)
            if counter is not None:
                counter.add_(1)
        rows = o["pooled"].view(-1, recipe.num_points, o["pooled"].shape[3])
        return {'sampled_pts': rows[:, :, 0:3], 'pts_feature': rows[:, :, 3:], 'cls_label': o["cls"].long(), 'reg_valid_mask': o["reg"].long(),
                'gt_of_rois': o["gt_ct"], 'gt_iou': o["iou"].view(-1), 'roi_boxes3d': o["rois"].view(-1, 7), 'sample_status': o["status"],
                'sample_index': o["sel"].view(-1, 3)}

    # ------------------------------------------------------------------ sampling (:78-183)
    def sample_rois_for_rcnn(self, roi_boxes3d, gt_boxes3d):
        """roi_boxes3d (B,M,7), gt_boxes3d (B,N,7 or 8; zero rows = padding) -> batch_rois (B,R,7), batch_gt_of_rois (B,R,7), batch_roi_iou (B,R)"""
        cfg = self.cfg.RCNN
        B = roi_boxes3d.size(0)
        R = cfg.ROI_PER_IMAGE
        fg_rois_per_image = int(np.round(cfg.FG_RATIO * R))
        fg_thresh = min(cfg.REG_FG_THRESH, cfg.CLS_FG_THRESH)
        # every (RoI, GT) pair of the batch in ONE launch; padded GT rows are computed and ignored
        iou_all = iou3d_cuda.boxes_iou3d(roi_boxes3d.contiguous().float(), gt_boxes3d[:, :, 0:7].contiguous().float())   # (B,M,N)
        n_gt = self._num_gt(gt_boxes3d)

        src_rois, src_gts, src_iou, aug_times = [], [], [], []
        for idx in range(B):
            cur_roi, cur_gt = roi_boxes3d[idx], gt_boxes3d[idx][:n_gt[idx]]
            max_overlaps, gt_assignment = torch.max(iou_all[idx, :, :n_gt[idx]], dim=1)
            fg_inds = torch.nonzero(max_overlaps >= fg_thresh).view(-1)
            easy_bg_inds = torch.nonzero(max_overlaps < cfg.CLS_BG_THRESH_LO).view(-1)
            hard_bg_inds = torch.nonzero((max_overlaps < cfg.CLS_BG_THRESH) & (max_overlaps >= cfg.CLS_BG_THRESH_LO)).view(-1)
            fg_num_rois = fg_inds.numel()
            bg_num_rois = hard_bg_inds.numel() + easy_bg_inds.numel()
            if fg_num_rois > 0 and bg_num_rois > 0:
                fg_n = min(fg_rois_per_image, fg_num_rois)
                rand_num = torch.from_numpy(np.random.permutation(fg_num_rois)).type_as(gt_boxes3d).long()
                fg_inds = fg_inds[rand_num[:fg_n]]
                bg_n = R - fg_n
                bg_inds = self.sample_bg_inds(hard_bg_inds, easy_bg_inds, bg_n)
            elif fg_num_rois > 0 and bg_num_rois == 0:
                rand_num = np.floor(np.random.rand(R) * fg_num_rois)
                rand_num = torch.from_numpy(rand_num).type_as(gt_boxes3d).long()
                fg_inds = fg_inds[rand_num]
                fg_n, bg_n = R, 0
            elif bg_num_rois > 0 and fg_num_rois == 0:
                bg_n = R
                bg_inds = self.sample_bg_inds(hard_bg_inds, easy_bg_inds, bg_n)
                fg_n = 0
            else:
                raise NotImplementedError("no RoI falls into the foreground or background IoU ranges")
            sel, times = [], []
            if fg_n > 0:
                sel.append(fg_inds)
                times.append(torch.full((fg_inds.numel(),), cfg.ROI_FG_AUG_TIMES, dtype=torch.int64))
            if bg_n > 0:
                sel.append(bg_inds)
                times.append(torch.full((bg_inds.numel(),), 1 if cfg.ROI_FG_AUG_TIMES > 0 else 0, dtype=torch.int64))
            sel = torch.cat(sel, dim=0)
            src_rois.append(cur_roi[sel])
            src_gts.append(cur_gt[gt_assignment[sel]][:, 0:7])
            src_iou.append(max_overlaps[sel])
            aug_times.append(torch.cat(times))
        rois, gts, iou = torch.stack(src_rois), torch.stack(src_gts), torch.stack(src_iou)           # (B,R,7), (B,R,7), (B,R)
        times = torch.stack(aug_times).to(rois.device)
        rois, iou = self.aug_roi_by_noise_batched(rois.view(-1, 7), gts.reshape(-1, 7), iou.view(-1), times.view(-1))
        return rois.view(B, R, 7), gts.contiguous(), iou.view(B, R)

    @staticmethod
    def _num_gt(gt_boxes3d):
        """the reference trims trailing all-zero GT rows (`while cur_gt[k].sum() == 0: k -= 1`, :95-98): one host read per batch"""
        nz = (gt_boxes3d.sum(dim=2) != 0)
        pos = torch.arange(1, gt_boxes3d.size(1) + 1, device=gt_boxes3d.device).unsqueeze(0) * nz.long()
        return [int(v) for v in pos.max(dim=1)[0].tolist()]

    def sample_bg_inds(self, hard_bg_inds, easy_bg_inds, bg_rois_per_this_image):
        """:185-212 (same random calls in the same order)"""
        if hard_bg_inds.numel() > 0 and easy_bg_inds.numel() > 0:
            hard_n = int(bg_rois_per_this_image * self.cfg.RCNN.HARD_BG_RATIO)
            easy_n = bg_rois_per_this_image - hard_n
            hard = hard_bg_inds[torch.randint(low=0, high=hard_bg_inds.numel(), size=(hard_n,)).long()]
            easy = easy_bg_inds[torch.randint(low=0, high=easy_bg_inds.numel(), size=(easy_n,)).long()]
            return torch.cat([hard, easy], dim=0)
        if hard_bg_inds.numel() > 0:
            return hard_bg_inds[torch.randint(low=0, high=hard_bg_inds.numel(), size=(bg_rois_per_this_image,)).long()]
        if easy_bg_inds.numel() > 0:
            return easy_bg_inds[torch.randint(low=0, high=easy_bg_inds.numel(), size=(bg_rois_per_this_image,)).long()]
        raise NotImplementedError

    # ------------------------------------------------------------------ jitter loop (:214-240), all RoIs at once
    def aug_roi_by_noise_batched(self, roi_boxes3d, gt_boxes3d, iou3d_src, aug_times):
        """roi (K,7), gt (K,7), iou3d_src (K), aug_times (K) int64 -> augmented rois (K,7), their IoU with the GT (K)"""
        cfg = self.cfg.RCNN
        pos_thresh = min(cfg.REG_FG_THRESH, cfg.CLS_FG_THRESH)
        K = roi_boxes3d.shape[0]
        dev = roi_boxes3d.device
        out_box = roi_boxes3d.clone()
        out_iou = iou3d_src.clone()              # cnt == 0 or the original kept: the source IoU (:236-237)
        temp_iou = torch.zeros(K, device=dev)
        cnt = torch.zeros(K, dtype=torch.int64, device=dev)
        gt = gt_boxes3d.contiguous().float()
        for _ in range(int(aug_times.max().item()) if K else 0):
            active = (temp_iou < pos_thresh) & (cnt < aug_times)
            keep_orig = torch.rand(K, device=dev) < 0.2            # p = 0.2 to keep the original roi box
            cand = torch.where(keep_orig.unsqueeze(1), roi_boxes3d, self.random_aug_box3d(roi_boxes3d))
            iou = iou3d_cuda.boxes_iou3d_aligned(cand.contiguous().float(), gt)
            out_box = torch.where(active.unsqueeze(1), cand, out_box)
            out_iou = torch.where(active, torch.where(keep_orig, iou3d_src, iou), out_iou)
            temp_iou = torch.where(active, iou, temp_iou)
            cnt = cnt + active.long()
        return out_box, out_iou

    def random_aug_box3d(self, box3d):
        """:242-286, vectorised over (K,7) boxes: random shift, scale, orientation"""
        method = self.cfg.RCNN.REG_AUG_METHOD
        K, dev = box3d.shape[0], box3d.device
        if method == 'single':
            pos_shift = torch.rand(K, 3, device=dev) - 0.5
            hwl_scale = (torch.rand(K, 3, device=dev) - 0.5) / (0.5 / 0.15) + 1.0
            angle_rot = (torch.rand(K, 1, device=dev) - 0.5) / (0.5 / (np.pi / 12))
        elif method == 'multiple':
            rc = torch.tensor(_RANGE_CONFIG, dtype=torch.float32, device=dev)[torch.randint(low=0, high=len(_RANGE_CONFIG), size=(K,), device=dev)]
            pos_shift = ((torch.rand(K, 3, device=dev) - 0.5) / 0.5) * rc[:, 0:1]
            hwl_scale = ((torch.rand(K, 3, device=dev) - 0.5) / 0.5) * rc[:, 1:2] + 1.0
            angle_rot = ((torch.rand(K, 1, device=dev) - 0.5) / 0.5) * rc[:, 2:3]
        elif method == 'normal':
            std = torch.tensor([0.3, 0.2, 0.3, 0.25, 0.15, 0.5], device=dev)
            shift = torch.randn(K, 6, device=dev) * std
            ry_shift = ((torch.rand(K, 1, device=dev) - 0.5) / 0.5) * np.pi / 12
            return torch.cat([box3d[:, 0:6] + shift, box3d[:, 6:7] + ry_shift], dim=1)
        else:
            raise NotImplementedError
        return torch.cat([box3d[:, 0:3] + pos_shift, box3d[:, 3:6] * hwl_scale, box3d[:, 6:7] + angle_rot], dim=1)

    # ------------------------------------------------------------------ point / box augmentation (:288-374)
    def data_augmentation(self, pts, rois, gt_of_rois):
        """pts (B,M,512,3), rois (B,M,7), gt_of_rois (B,M,7): random rotation about y, scaling, x flip"""
        B, M = pts.shape[0], pts.shape[1]
        dev = pts.device
        angles = (torch.rand((B, M), device=dev) - 0.5 / 0.5) * (np.pi / self.cfg.AUG_ROT_RANGE)

        def alpha_of(boxes):      # observation angle: ry + beta - sign(beta) * pi / 2
            beta = torch.atan2(boxes[:, :, 2], boxes[:, :, 0])
            return -torch.sign(beta) * np.pi / 2 + beta + boxes[:, :, 6]
        gt_alpha, roi_alpha = alpha_of(gt_of_rois), alpha_of(rois)
        flat = angles.reshape(-1)
        pts = kitti_utils.rotate_pc_along_y_torch(pts.reshape(B * M, -1, 3), flat).view(B, M, -1, 3)
        gt_of_rois = kitti_utils.rotate_pc_along_y_torch(gt_of_rois.reshape(B * M, 1, 7), flat).view(B, M, 7)
        rois = kitti_utils.rotate_pc_along_y_torch(rois.reshape(B * M, 1, 7), flat).view(B, M, 7)
        for boxes, alpha in ((gt_of_rois, gt_alpha), (rois, roi_alpha)):      # heading after the rotation
            beta = torch.atan2(boxes[:, :, 2], boxes[:, :, 0])
            boxes[:, :, 6] = torch.sign(beta) * np.pi / 2 + alpha - beta

        scales = 1 + ((torch.rand((B, M), device=dev) - 0.5) / 0.5) * 0.05
        pts = pts * scales.unsqueeze(dim=2).unsqueeze(dim=3)
        gt_of_rois[:, :, 0:6] = gt_of_rois[:, :, 0:6] * scales.unsqueeze(dim=2)
        rois[:, :, 0:6] = rois[:, :, 0:6] * scales.unsqueeze(dim=2)

        flip_flag = torch.sign(torch.rand((B, M), device=dev) - 0.5)
        pts[:, :, :, 0] = pts[:, :, :, 0] * flip_flag.unsqueeze(dim=2)
        for boxes in (gt_of_rois, rois):
            boxes[:, :, 0] = boxes[:, :, 0] * flip_flag
            src_ry = boxes[:, :, 6]
            boxes[:, :, 6] = (flip_flag == 1).float() * src_ry + (flip_flag == -1).float() * (torch.sign(src_ry) * np.pi - src_ry)
        return pts, rois, gt_of_rois
