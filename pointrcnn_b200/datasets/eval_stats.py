"""Recall, segmentation IoU and classification accuracy of tools/eval_rcnn.py's evaluation loops, accumulated on the device.

The reference computes these statistics one scene at a time (a boxes_iou3d_gpu call per box set, a dozen `.item()` host
round trips per scene).  Here every `add_*` call is a few launches of csrc/eval_stats.cu for a whole batch, the counts stay
in int64 device accumulators and the per-scene fp32 values (segmentation IoU, accuracies) in device buffers, and
`result()` copies everything to the host once:

    stats = EvalStats()
    for batch in ...:                      # eval_one_epoch_rcnn / _joint
        stats.add_rcnn(pred_boxes3d, roi_boxes3d, gt_boxes3d, gt_count, box_count=roi_count, pred_classes=..., gt_iou=...,
                       select=select)
    ret_dict = stats.result()              # the reference's ret_dict keys and values
    for line in stats.log_lines():
        logger.info(line)

Every statistic is per scene, with the first gt_count[s] GT rows of scene s.  At batch size 1 (what eval_one_epoch_rcnn
asserts, and the CLI default) the values equal the reference's: per-scene fp32 values are summed in float64 in scene
order, as the reference's `total += x.item()` does.  INTEGRATION.md lists the two batch-size quirks of the reference that
are not copied.
"""
import ctypes

import numpy as np
import torch

from .. import _cabi as C

THRESH_LIST = (0.1, 0.3, 0.5, 0.7, 0.9)


def _f32(t):
    return t.float().contiguous()


def _i32(t):
    return t.to(torch.int32).contiguous()


class _Buffer:
    """a growing fp32 device buffer; `take(k)` returns the next k slots (written by a kernel), in scene order"""

    def __init__(self, device, what):
        self.data = torch.empty(1024, dtype=torch.float32, device=device)
        self.n = 0
        self.what = what
        self.used = None          # whether the run's batches give this statistic: all of them or none

    def given(self, flag, scenes_before):
        """checks that every batch of a run gives this statistic or none does: an average over some of the scenes would
        be divided by all of them"""
        if self.used is None and scenes_before == 0:
            self.used = flag
        if self.used != flag:
            raise ValueError("EvalStats: %s given for some batches of the run and not for others" % self.what)
        return flag

    def take(self, k):
        if self.n + k > self.data.numel():
            grown = torch.empty(max(2 * self.data.numel(), self.n + k), dtype=torch.float32, device=self.data.device)
            grown[:self.n].copy_(self.data[:self.n])
            self.data = grown
        out = self.data[self.n:self.n + k]
        self.n += k
        return out


def log_lines(mode, ret, counts):
    """the reference's logger strings for the statistics of one loop.  mode: "rpn", "rcnn" or "joint"; ret: the ret_dict;
    counts: dict with rpn_recalled / rcnn_recalled (lists over the thresholds), gt_total, thresh_list"""
    th, gt = counts["thresh_list"], counts["gt_total"]
    recall = lambda fmt, rec, key: [fmt % (t, rec[k], gt, ret[key % t]) for k, t in enumerate(th)]
    if mode == "rpn":
        return (["max number of objects: %d" % ret["max_obj_num"], "rpn iou avg: %f" % ret["rpn_iou"]] +
                recall("total bbox recall(thresh=%.3f): %d / %d = %f", counts["rpn_recalled"], "rpn_recall(thresh=%.2f)"))
    lines = ["final average detections: %.3f" % ret["rcnn_avg_num"]]
    if mode == "joint":
        lines.append("final average rpn_iou refined: %.3f" % ret["rpn_iou"])
    lines += ["final average cls acc: %.3f" % ret["rcnn_cls_acc"], "final average cls acc refined: %.3f" % ret["rcnn_cls_acc_refined"]]
    lines += recall("total roi bbox recall(thresh=%.3f): %d / %d = %f", counts["rpn_recalled"], "rpn_recall(thresh=%.2f)")
    lines += recall("total bbox recall(thresh=%.3f): %d / %d = %f", counts["rcnn_recalled"], "rcnn_recall(thresh=%.2f)")
    return lines


class EvalStats:
    """Device accumulators for one evaluation run.  cls_fg_thresh / cls_bg_thresh: cfg.RCNN.CLS_FG_THRESH / CLS_BG_THRESH;
    refined_thresh: 0.7 for cfg.CLASSES == 'Car', else 0.5 (eval_rcnn.py:359).  The optional statistics (seg_result /
    rpn_cls_label, pred_classes / gt_iou) are given for every batch of a run or for none; mixing raises ValueError."""

    def __init__(self, thresh_list=THRESH_LIST, device=None, cls_fg_thresh=0.6, cls_bg_thresh=0.45, refined_thresh=0.7):
        self.thresh_list = tuple(float(t) for t in thresh_list)
        self.device = torch.device(device if device is not None else "cuda")
        if self.device.type != "cuda":
            raise RuntimeError("pointrcnn_b200: EvalStats accumulates on a CUDA device (there is no CPU path)")
        T = len(self.thresh_list)
        self._thresh = (ctypes.c_float * max(T, 1))(*self.thresh_list)
        self.cls_fg, self.cls_bg, self.refined = float(cls_fg_thresh), float(cls_bg_thresh), float(refined_thresh)
        # [rpn / roi recalled (T) | rcnn recalled (T) | gt_total | detections]
        self._counts = torch.zeros(2 * T + 2, dtype=torch.int64, device=self.device)
        self._seg = _Buffer(self.device, "seg_result / rpn_cls_label")
        self._acc = _Buffer(self.device, "pred_classes / gt_iou")
        self._acc_refined = _Buffer(self.device, "pred_classes / gt_iou")
        self.scenes = 0
        self.mode = None
        self._result = None

    def _set_mode(self, mode):
        if self.mode is not None and self.mode != mode:
            raise ValueError("EvalStats: %s statistics added to a %s run" % (mode, self.mode))
        self.mode = mode
        self._result = None

    def _recall(self, boxes, box_count, gt_boxes3d, gt_count, recalled, gt_total, box_max_iou=None):
        boxes, gt = _f32(boxes), _f32(gt_boxes3d)
        B, M, G = boxes.shape[0], boxes.shape[1], gt.shape[1]
        T = len(self.thresh_list)
        C.require_cuda(boxes, gt, gt_count, box_count)
        C.check(C.lib().prb_eval_box_recall(B, M, C.ptr(boxes), C.ptr(None if box_count is None else _i32(box_count)), G, C.ptr(gt),
                                            C.ptr(_i32(gt_count)), T, self._thresh, C.ptr(recalled), C.ptr(gt_total),
                                            C.ptr(box_max_iou), C.stream()), "eval_box_recall")

    def _seg_iou(self, seg_result, rpn_cls_label):
        pred, label = _i32(seg_result), _i32(rpn_cls_label)
        B = pred.shape[0]
        pred, label = pred.view(B, -1), label.view(B, -1)
        C.require_cuda(pred, label)
        C.check(C.lib().prb_eval_seg_iou(B, pred.shape[1], C.ptr(pred), C.ptr(label), C.ptr(self._seg.take(B)), C.stream()), "eval_seg_iou")

    def add_rpn(self, rois, gt_boxes3d, gt_count, seg_result=None, rpn_cls_label=None):
        """eval_one_epoch_rpn: rois (B,M,7) with every row counted (zero padding has IoU 0), gt_boxes3d (B,G,7), gt_count (B)
        device int; seg_result / rpn_cls_label (B,N) for the segmentation IoU"""
        self._set_mode("rpn")
        seg = self._seg.given(seg_result is not None and rpn_cls_label is not None, self.scenes)
        T = len(self.thresh_list)
        with torch.cuda.device(self.device):
            self._recall(rois, None, gt_boxes3d, gt_count, self._counts[0:T], self._counts[2 * T:2 * T + 1])
            if seg:
                self._seg_iou(seg_result, rpn_cls_label)
        self.scenes += rois.shape[0]

    def add_rcnn(self, pred_boxes3d, roi_boxes3d, gt_boxes3d, gt_count, box_count=None, pred_classes=None, gt_iou=None, select=None,
                 seg_result=None, rpn_cls_label=None):
        """eval_one_epoch_rcnn (no seg_result) and eval_one_epoch_joint (seg_result / rpn_cls_label given).
        pred_boxes3d / roi_boxes3d (B,M,7), the first box_count[s] rows real (None: all); gt_boxes3d (B,G,7), gt_count (B);
        pred_classes (B,M) = (sigmoid(rcnn_cls) > SCORE_THRESH) and gt_iou (B,M) for the classification accuracy;
        select (B,M) bool, detections_device's mask, for rcnn_avg_num"""
        self._set_mode("joint" if seg_result is not None else "rcnn")
        T = len(self.thresh_list)
        acc = self._acc.given(pred_classes is not None and gt_iou is not None, self.scenes)
        seg = self._seg.given(seg_result is not None and rpn_cls_label is not None, self.scenes)
        B, M = pred_boxes3d.shape[0], pred_boxes3d.shape[1]
        with torch.cuda.device(self.device):
            self._recall(pred_boxes3d, box_count, gt_boxes3d, gt_count, self._counts[T:2 * T], self._counts[2 * T:2 * T + 1])
            self._recall(roi_boxes3d, box_count, gt_boxes3d, gt_count, self._counts[0:T], None)
            if acc:
                pc, gi = _i32(pred_classes).view(B, M), _f32(gt_iou).view(B, M)
                C.require_cuda(pc, gi)
                C.check(C.lib().prb_eval_cls_acc(B, M, C.ptr(None if box_count is None else _i32(box_count)), C.ptr(pc), C.ptr(gi),
                                                 self.cls_fg, self.cls_bg, self.refined, C.ptr(self._acc.take(B)),
                                                 C.ptr(self._acc_refined.take(B)), C.stream()), "eval_cls_acc")
            if select is not None:
                self._counts[2 * T + 1:].add_(select.reshape(-1).sum())
            if seg:
                self._seg_iou(seg_result, rpn_cls_label)
        self.scenes += B

    def counts(self):
        """the host copy: dict of int counts and float64 per-scene sums (one device-to-host copy, cached until the next add)"""
        if self._result is None:
            T = len(self.thresh_list)
            bufs = (self._seg, self._acc, self._acc_refined)
            parts = [self._counts.view(torch.int32)] + [b.data[:b.n].view(torch.int32) for b in bufs]
            host = torch.cat(parts).cpu().numpy()
            c = host[:2 * (2 * T + 2)].view(np.int64)
            off, sums = 2 * (2 * T + 2), []
            for b in bufs:
                total = 0.0
                for v in host[off:off + b.n].view(np.float32).tolist():      # the reference's Python-float `+=`, in scene order
                    total += v
                sums.append(total)
                off += b.n
            self._result = dict(thresh_list=self.thresh_list, rpn_recalled=[int(v) for v in c[0:T]],
                                rcnn_recalled=[int(v) for v in c[T:2 * T]], gt_total=int(c[2 * T]), detections=int(c[2 * T + 1]),
                                rpn_iou_sum=sums[0], cls_acc_sum=sums[1], cls_acc_refined_sum=sums[2], scenes=self.scenes)
        return self._result

    def result(self):
        """the reference's ret_dict for this run's loop (empty_cnt and the AP keys are not statistics of this class)"""
        c = self.counts()
        cnt, gt = max(self.scenes, 1.0), max(c["gt_total"], 1.0)
        if self.mode == "rpn":
            # eval_one_epoch_rpn never updates max_num
            ret = {"max_obj_num": 0, "rpn_iou": c["rpn_iou_sum"] / cnt}
            for k, t in enumerate(self.thresh_list):
                ret["rpn_recall(thresh=%.2f)" % t] = c["rpn_recalled"][k] / gt
            return ret
        ret = {"rpn_iou": c["rpn_iou_sum"] / cnt} if self.mode == "joint" else {}
        ret.update(rcnn_cls_acc=c["cls_acc_sum"] / cnt, rcnn_cls_acc_refined=c["cls_acc_refined_sum"] / cnt,
                   rcnn_avg_num=c["detections"] / cnt)
        for k, t in enumerate(self.thresh_list):
            ret["rpn_recall(thresh=%.2f)" % t] = c["rpn_recalled"][k] / gt
        for k, t in enumerate(self.thresh_list):
            ret["rcnn_recall(thresh=%.2f)" % t] = c["rcnn_recalled"][k] / gt
        return ret

    def log_lines(self):
        """the reference's logger lines for these statistics, character for character"""
        return log_lines(self.mode, self.result(), self.counts())
