"""oracle/eval_stats.py -- numpy restatement of the statistics of tools/eval_rcnn.py's three evaluation loops at batch size 1
(eval_one_epoch_rpn :179-201 and :238-250, eval_one_epoch_rcnn :337-367 and :412-432, eval_one_epoch_joint :541-573 and
:638-660), with oracle.boxes_iou3d for the 3D IoU.  TEST INFRASTRUCTURE ONLY.

Per-scene values are fp32, as the reference's torch lines on the CPU compute them (a Python-number divisor is a true
division there), and are summed as Python floats in scene order.  Each function returns (ret_dict, counts) with counts in
the layout of pointrcnn_b200.datasets.eval_stats.log_lines.
"""
import numpy as np

from . import oracle as O

THRESH_LIST = (0.1, 0.3, 0.5, 0.7, 0.9)
F32 = np.float32


def _recall(boxes, gt, rec):
    """adds (gt_max_iou > thresh) per threshold; returns the (M,) max over GT (refined_iou)"""
    iou = O.boxes_iou3d(np.asarray(boxes, F32).reshape(-1, 7), np.asarray(gt, F32).reshape(-1, 7))
    gmax = iou.max(axis=0)
    for k, t in enumerate(THRESH_LIST):
        rec[k] += int((gmax > t).sum())
    return iou.max(axis=1)


def seg_iou(seg, label):
    seg, label = np.asarray(seg).reshape(-1), np.asarray(label).reshape(-1)
    fg = label > 0
    correct = F32(((seg == label) & fg).sum())
    union = F32(F32(fg.sum()) + F32((seg > 0).sum())) - correct
    return F32(correct / max(union, F32(1.0)))


def cls_acc(pred_cls, gt_iou, fg=0.6, bg=0.45, refined=0.7):
    pred_cls, gt_iou = np.asarray(pred_cls).reshape(-1), np.asarray(gt_iou, F32).reshape(-1)
    label = (gt_iou > F32(fg)).astype(np.int64)
    valid = ((gt_iou >= F32(fg)) | (gt_iou <= F32(bg))).astype(F32)
    acc = F32(((pred_cls == label).astype(F32) * valid).sum(dtype=F32) / max(valid.sum(dtype=F32), F32(1.0)))
    lab_r = (gt_iou >= F32(refined)).astype(np.int64)
    acc_r = F32((pred_cls == lab_r).astype(F32).sum(dtype=F32) / F32(max(len(lab_r), 1.0)))
    return acc, acc_r


def _counts(rpn_rec, rcnn_rec, gt_total):
    return dict(thresh_list=THRESH_LIST, rpn_recalled=list(rpn_rec), rcnn_recalled=list(rcnn_rec), gt_total=gt_total)


def rpn_loop(scenes):
    """scenes: dicts rois (M,7), gt (G,7), seg (N,), label (N,)"""
    rec, gt_total, iou_sum = [0] * 5, 0, 0.0
    for s in scenes:
        if len(s["gt"]):
            _recall(s["rois"], s["gt"], rec)
            gt_total += len(s["gt"])
        iou_sum += float(seg_iou(s["seg"], s["label"]))
    ret = {"max_obj_num": 0, "rpn_iou": iou_sum / len(scenes)}
    for k, t in enumerate(THRESH_LIST):
        ret["rpn_recall(thresh=%.2f)" % t] = rec[k] / max(gt_total, 1.0)
    return ret, _counts(rec, [0] * 5, gt_total)


def rcnn_loop(scenes, joint=False):
    """scenes: dicts pred (M,7), rois (M,7), gt (G,7), n_det; rcnn: pred_cls (M,), gt_iou (M,); joint: seg (N,), label (N,)"""
    rec, roi_rec, gt_total = [0] * 5, [0] * 5, 0
    acc_sum = acc_r_sum = iou_sum = 0.0
    n_det = 0
    for s in scenes:
        if len(s["gt"]):
            _recall(s["pred"], s["gt"], rec)
            _recall(s["rois"], s["gt"], roi_rec)
            gt_total += len(s["gt"])
        if joint:
            iou_sum += float(seg_iou(s["seg"], s["label"]))
        else:
            a, ar = cls_acc(s["pred_cls"], s["gt_iou"])
            acc_sum += float(a)
            acc_r_sum += float(ar)
        n_det += int(s["n_det"])
    cnt = max(len(scenes), 1.0)
    ret = {"rpn_iou": iou_sum / cnt} if joint else {}
    ret.update(rcnn_cls_acc=acc_sum / cnt, rcnn_cls_acc_refined=acc_r_sum / cnt, rcnn_avg_num=n_det / cnt)
    for k, t in enumerate(THRESH_LIST):
        ret["rpn_recall(thresh=%.2f)" % t] = roi_rec[k] / max(gt_total, 1.0)
    for k, t in enumerate(THRESH_LIST):
        ret["rcnn_recall(thresh=%.2f)" % t] = rec[k] / max(gt_total, 1.0)
    return ret, _counts(roi_rec, rec, gt_total)


def gt_iou(rois, gt):
    """get_proposal_from_file's gt_iou with the fp32 overlap: max IoU over the GT, zeros without GT"""
    if len(gt) == 0:
        return np.zeros(len(rois), F32)
    return O.boxes_iou3d(np.asarray(rois, F32), np.asarray(gt, F32)).max(axis=1)
