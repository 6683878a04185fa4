"""Losses of the RPN / RCNN training step: mirror of lib/utils/loss_utils.py:7-233 (DiceLoss,
SigmoidFocalClassificationLoss, get_reg_loss) and of get_rpn_loss / get_rcnn_loss in lib/net/train_functions.py:55-209.

Two implementations behind one signature, chosen by `impl` ("torch" / "device"; None follows the `loss_impl` switch of
pointrcnn_b200.config, "torch" unless changed):

- "torch": the same arithmetic as the reference (the same torch ops in the same order per term); what differs is
  bookkeeping: the reference calls `.item()` on every partial loss (15+ host synchronisations per step,
  `loss_utils.py:127-128,...`, `train_functions.py:77-78,115-118`) -- here every term stays a device tensor and the caller
  reads what it logs once.  The foreground rows are still selected with boolean masks, one host synchronisation each.
- "device": csrc/stage_loss.cu through a torch.autograd.Function: two launches forward, one backward, no host
  synchronisation, the same (total, terms) keys for the same options (each term a 0-d device tensor), and the gradients
  torch autograd derives for the mirror.  Values differ from the torch path in the last bits (float64 sums).  Without a
  foreground row the regression terms are exact zeros here, where the torch path leaves their keys out.  CUDA tensors only.

Under torch.autocast both compute in fp32: rpn_loss / rcnn_loss cast their floating inputs to fp32 and run with autocast
disabled (so the mirror's F.binary_cross_entropy stays legal and its terms match the device loss's), and the inputs'
gradients come back in the inputs' dtypes.  Outside autocast nothing is cast.
"""
import ctypes
import functools

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import _cabi as C
from .. import config

IMPLS = ("torch", "device")


class DiceLoss(nn.Module):
    def __init__(self, ignore_target=-1):
        super().__init__()
        self.ignore_target = ignore_target

    def forward(self, input, target):
        """input (N) logits, target (N) in {0,1} (ignore_target rows are masked)"""
        p = torch.sigmoid(input.view(-1))
        t = target.float().view(-1)
        mask = (t != self.ignore_target).float()
        return 1.0 - (torch.min(p, t) * mask).sum() / torch.clamp((torch.max(p, t) * mask).sum(), min=1.0)


def _sigmoid_cross_entropy_with_logits(logits, labels):
    loss = torch.clamp(logits, min=0) - logits * labels.type_as(logits)
    return loss + torch.log1p(torch.exp(-torch.abs(logits)))


class SigmoidFocalClassificationLoss(nn.Module):
    """sigmoid focal cross entropy (loss_utils.py:25-76)"""

    def __init__(self, gamma=2.0, alpha=0.25):
        super().__init__()
        self._alpha, self._gamma = alpha, gamma

    def forward(self, prediction_tensor, target_tensor, weights):
        ce = _sigmoid_cross_entropy_with_logits(labels=target_tensor, logits=prediction_tensor)
        prob = torch.sigmoid(prediction_tensor)
        p_t = (target_tensor * prob) + ((1 - target_tensor) * (1 - prob))
        mod = torch.pow(1.0 - p_t, self._gamma) if self._gamma else 1.0
        alpha_w = (target_tensor * self._alpha + (1 - target_tensor) * (1 - self._alpha)) if self._alpha is not None else 1.0
        return mod * alpha_w * ce * weights


def _bin_loss(pred, lo, nbin, shift, bin_size, with_res, res_lo):
    """cross entropy over the bins of `shift` (+ smooth-L1 on the residual inside the target bin); returns (bin_loss, res_loss, bin_label)"""
    bin_label = (shift / bin_size).floor().long()
    loss_bin = F.cross_entropy(pred[:, lo:lo + nbin], bin_label)
    loss_res = None
    if with_res:
        res_label = (shift - (bin_label.float() * bin_size + bin_size / 2)) / bin_size
        onehot = torch.zeros((bin_label.size(0), nbin), dtype=pred.dtype, device=pred.device).scatter_(1, bin_label.view(-1, 1), 1)
        loss_res = F.smooth_l1_loss((pred[:, res_lo:res_lo + nbin] * onehot).sum(dim=1), res_label)
    return loss_bin, loss_res, bin_label


def get_reg_loss(pred_reg, reg_label, loc_scope, loc_bin_size, num_head_bin, anchor_size, get_xz_fine=True, get_y_by_bin=False,
                 loc_y_scope=0.5, loc_y_bin_size=0.25, get_ry_fine=False):
    """bin-based box regression loss (loss_utils.py:87-233).  pred_reg (N,C), reg_label (N,7) [dx,dy,dz,h,w,l,ry] ->
    loc_loss, angle_loss, size_loss, dict of the partial terms (device tensors)"""
    nloc = int(loc_scope / loc_bin_size) * 2
    ny = int(loc_y_scope / loc_y_bin_size) * 2
    terms = {}
    x_shift = torch.clamp(reg_label[:, 0] + loc_scope, 0, loc_scope * 2 - 1e-3)
    z_shift = torch.clamp(reg_label[:, 2] + loc_scope, 0, loc_scope * 2 - 1e-3)
    lxb, lxr, _ = _bin_loss(pred_reg, 0, nloc, x_shift, loc_bin_size, get_xz_fine, 2 * nloc)
    lzb, lzr, _ = _bin_loss(pred_reg, nloc, nloc, z_shift, loc_bin_size, get_xz_fine, 3 * nloc)
    terms["loss_x_bin"], terms["loss_z_bin"] = lxb, lzb
    loc_loss = lxb + lzb
    off = 2 * nloc
    if get_xz_fine:
        terms["loss_x_res"], terms["loss_z_res"] = lxr, lzr
        loc_loss = loc_loss + lxr + lzr
        off = 4 * nloc
    y_label = reg_label[:, 1]
    if get_y_by_bin:
        y_shift = torch.clamp(y_label + loc_y_scope, 0, loc_y_scope * 2 - 1e-3)
        lyb, lyr, _ = _bin_loss(pred_reg, off, ny, y_shift, loc_y_bin_size, True, off + ny)
        terms["loss_y_bin"], terms["loss_y_res"] = lyb, lyr
        loc_loss = loc_loss + lyb + lyr
        off += 2 * ny
    else:
        ly = F.smooth_l1_loss(pred_reg[:, off:off + 1].sum(dim=1), y_label)
        terms["loss_y_offset"] = ly
        loc_loss = loc_loss + ly
        off += 1
    ry_label = reg_label[:, 6]
    if get_ry_fine:
        per = (np.pi / 2) / num_head_bin
        ry = ry_label % (2 * np.pi)
        opposite = (ry > np.pi * 0.5) & (ry < np.pi * 1.5)
        ry = torch.where(opposite, (ry + np.pi) % (2 * np.pi), ry)
        shift_angle = torch.clamp((ry + np.pi * 0.5) % (2 * np.pi) - np.pi * 0.25, min=1e-3, max=np.pi * 0.5 - 1e-3)
    else:
        per = (2 * np.pi) / num_head_bin
        shift_angle = ((ry_label % (2 * np.pi)) + per / 2) % (2 * np.pi)
    ry_bin = (shift_angle / per).floor().long()
    ry_res = (shift_angle - (ry_bin.float() * per + per / 2)) / (per / 2)
    onehot = torch.zeros((ry_bin.size(0), num_head_bin), dtype=pred_reg.dtype, device=pred_reg.device).scatter_(1, ry_bin.view(-1, 1), 1)
    l_rb = F.cross_entropy(pred_reg[:, off:off + num_head_bin], ry_bin)
    l_rr = F.smooth_l1_loss((pred_reg[:, off + num_head_bin:off + 2 * num_head_bin] * onehot).sum(dim=1), ry_res)
    terms["loss_ry_bin"], terms["loss_ry_res"] = l_rb, l_rr
    angle_loss = l_rb + l_rr
    off += 2 * num_head_bin
    assert pred_reg.shape[1] == off + 3, "%d vs %d" % (pred_reg.shape[1], off + 3)
    size_loss = F.smooth_l1_loss(pred_reg[:, off:off + 3], (reg_label[:, 3:6] - anchor_size) / anchor_size)
    terms.update(loss_loc=loc_loss, loss_angle=angle_loss, loss_size=size_loss)
    return loc_loss, angle_loss, size_loss, terms


def _impl(impl):
    impl = impl or config.get("loss_impl")
    if impl not in IMPLS:
        raise ValueError("loss_impl must be one of %s, not %r" % (IMPLS, impl))
    return impl


def _fp32_under_autocast(loss_fn):
    """run `loss_fn` as it is outside CUDA autocast; inside, with autocast disabled and every floating CUDA tensor argument
    below float64 cast to float32"""

    def up(v):
        return v.float() if torch.is_tensor(v) and v.is_cuda and v.is_floating_point() and v.dtype != torch.float64 else v

    @functools.wraps(loss_fn)
    def run(*args, **kwargs):
        if not torch.is_autocast_enabled("cuda"):
            return loss_fn(*args, **kwargs)
        with torch.autocast("cuda", enabled=False):
            return loss_fn(*[up(a) for a in args], **{k: up(v) for k, v in kwargs.items()})
    return run


@_fp32_under_autocast
def rpn_loss(rpn_cls, rpn_reg, rpn_cls_label, rpn_reg_label, mean_size, loss_cls="SigmoidFocalLoss", focal_alpha=0.25, focal_gamma=2.0,
             fg_weight=15.0, loc_scope=3.0, loc_bin_size=0.5, num_head_bin=12, loc_xz_fine=True, loss_weight=(1.0, 1.0), impl=None):
    """get_rpn_loss (train_functions.py:55-120).  rpn_cls (B,N,1), rpn_reg (B,N,C), rpn_cls_label (B,N) in {-1,0,1},
    rpn_reg_label (B,N,7) -> total loss, dict of device tensors.  The torch path selects the foreground rows with a boolean
    mask like the reference (one data-dependent shape, no .item()); impl: see the module docstring."""
    if _impl(impl) == "device":
        return _rpn_loss_device(rpn_cls, rpn_reg, rpn_cls_label, rpn_reg_label, mean_size, loss_cls, focal_alpha, focal_gamma, fg_weight,
                                loc_scope, loc_bin_size, num_head_bin, loc_xz_fine, loss_weight)
    cls_label = rpn_cls_label.view(-1)
    cls_flat = rpn_cls.view(-1)
    fg_mask = cls_label > 0
    if loss_cls == "DiceLoss":
        loss_c = DiceLoss()(rpn_cls, cls_label)
    elif loss_cls == "SigmoidFocalLoss":
        target = fg_mask.float()
        pos, neg = target, (cls_label == 0).float()
        w = (pos + neg) / torch.clamp(pos.sum(), min=1.0)
        loss_c = SigmoidFocalClassificationLoss(alpha=focal_alpha, gamma=focal_gamma)(cls_flat, target, w).sum()
    elif loss_cls == "BinaryCrossEntropy":
        weight = torch.where(fg_mask, torch.full_like(cls_flat, fg_weight), torch.ones_like(cls_flat))
        bl = F.binary_cross_entropy(torch.sigmoid(cls_flat), fg_mask.float(), weight=weight, reduction="none")
        valid = (cls_label >= 0).float()
        loss_c = (bl * valid).sum() / torch.clamp(valid.sum(), min=1.0)
    else:
        raise NotImplementedError(loss_cls)
    npts = rpn_reg.size(0) * rpn_reg.size(1)
    reg_fg = rpn_reg.view(npts, -1)[fg_mask]
    terms = {}
    if reg_fg.shape[0] != 0:
        loc, ang, size, terms = get_reg_loss(reg_fg, rpn_reg_label.view(npts, 7)[fg_mask], loc_scope=loc_scope, loc_bin_size=loc_bin_size,
                                             num_head_bin=num_head_bin, anchor_size=mean_size, get_xz_fine=loc_xz_fine,
                                             get_y_by_bin=False, get_ry_fine=False)
        loss_r = loc + ang + 3 * size             # "consistent with old codes" (train_functions.py:107)
    else:
        loss_r = loss_c * 0
    total = loss_c * loss_weight[0] + loss_r * loss_weight[1]
    terms.update(rpn_loss_cls=loss_c, rpn_loss_reg=loss_r, rpn_loss=total)
    return total, terms


@_fp32_under_autocast
def rcnn_loss(rcnn_cls, rcnn_reg, cls_label, reg_valid_mask, roi_boxes3d, gt_of_rois, mean_size, loss_cls="BinaryCrossEntropy",
              focal_alpha=0.25, focal_gamma=2.0, size_res_on_roi=False, loc_scope=1.5, loc_bin_size=0.5, num_head_bin=9,
              loc_y_by_bin=False, loc_y_scope=0.5, loc_y_bin_size=0.25, ce_weight=None, impl=None):
    """get_rcnn_loss (train_functions.py:121-209).  rcnn_cls (R,1|K), rcnn_reg (R,C), cls_label (R) in {-1,0,1},
    reg_valid_mask (R), roi_boxes3d (R,7), gt_of_rois (R,7) canonical -> total loss, dict of device tensors (no .item()).
    impl: see the module docstring."""
    if _impl(impl) == "device":
        return _rcnn_loss_device(rcnn_cls, rcnn_reg, cls_label, reg_valid_mask, roi_boxes3d, gt_of_rois, mean_size, loss_cls, focal_alpha,
                                 focal_gamma, size_res_on_roi, loc_scope, loc_bin_size, num_head_bin, loc_y_by_bin, loc_y_scope,
                                 loc_y_bin_size, ce_weight)
    R = rcnn_reg.shape[0]
    label = cls_label.float().view(-1)
    terms = {}
    if loss_cls == "SigmoidFocalLoss":
        flat = rcnn_cls.view(-1)
        pos, neg = (label > 0).float(), (label == 0).float()
        w = (pos + neg) / torch.clamp(pos.sum(), min=1.0)
        per = SigmoidFocalClassificationLoss(alpha=focal_alpha, gamma=focal_gamma)(flat, pos, w)
        terms["rpn_loss_cls_pos"], terms["rpn_loss_cls_neg"] = (per * pos).sum(), (per * neg).sum()     # the reference's key names
        loss_c = per.sum()
    elif loss_cls == "BinaryCrossEntropy":
        flat = rcnn_cls.view(-1)
        # the reference passes the -1 ("ignore") labels straight into F.binary_cross_entropy and masks the rows afterwards; current
        # torch rejects targets outside [0,1], so the ignored rows get a dummy target here (they are masked out all the same)
        bl = F.binary_cross_entropy(torch.sigmoid(flat), label.clamp(min=0.0), reduction="none")
        valid = (label >= 0).float()
        loss_c = (bl * valid).sum() / torch.clamp(valid.sum(), min=1.0)
    elif loss_cls == "CrossEntropy":
        logits = rcnn_cls.view(R, -1)
        valid = (label >= 0).float()
        bl = F.cross_entropy(logits, label.long(), weight=ce_weight, ignore_index=-1, reduction="none")
        loss_c = (bl * valid).sum() / torch.clamp(valid.sum(), min=1.0)      # (the reference's .mean(dim=1) of a 1-D loss is a no-op for K classes)
    else:
        raise NotImplementedError(loss_cls)
    fg = reg_valid_mask.view(-1) > 0
    reg_fg = rcnn_reg.view(R, -1)[fg]
    if reg_fg.shape[0] != 0:
        anchor = roi_boxes3d.view(R, 7)[:, 3:6][fg] if size_res_on_roi else mean_size
        loc, ang, size, reg_terms = get_reg_loss(reg_fg, gt_of_rois.view(R, 7)[fg], loc_scope=loc_scope, loc_bin_size=loc_bin_size,
                                                 num_head_bin=num_head_bin, anchor_size=anchor, get_xz_fine=True, get_y_by_bin=loc_y_by_bin,
                                                 loc_y_scope=loc_y_scope, loc_y_bin_size=loc_y_bin_size, get_ry_fine=True)
        terms.update(reg_terms)
        loss_r = loc + ang + 3 * size              # "consistent with old codes" (train_functions.py:193)
    else:
        loss_r = loss_c * 0
    total = loss_c + loss_r
    terms.update(rcnn_loss_cls=loss_c, rcnn_loss_reg=loss_r, rcnn_loss=total)
    return total, terms


# ---------------------------------------------------------------------------------------------- the device path
# slots of the loss vector (include/pointrcnn_b200.h: PRB_SL_*)
_SLOT = dict(loss_cls=0, loss_reg=1, loss_x_bin=2, loss_z_bin=3, loss_x_res=4, loss_z_res=5, loss_y_bin=6, loss_y_res=7, loss_y_offset=8,
             loss_ry_bin=9, loss_ry_res=10, loss_loc=11, loss_angle=12, loss_size=13, cls_pos=14, cls_neg=15)
_NUM_SLOTS = 20
_CLS_CODE = {"SigmoidFocalLoss": 0, "BinaryCrossEntropy": 1, "DiceLoss": 2, "CrossEntropy": 3}


class _StageLoss(torch.autograd.Function):
    """(cls, reg) -> (total 0-d, loss vector) through prb_stage_loss_forward; backward through prb_stage_loss_backward, which
    takes the upstream gradient of the total and of every slot of the vector (either may be absent) on the device"""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, cls, reg, desc, label, fg_mask, reg_label, mean_size, anchor_boxes, ce_weight):
        L = C.lib()
        rows = reg.shape[0]
        total = torch.empty((), dtype=torch.float32, device=reg.device)
        vec = torch.empty(_NUM_SLOTS, dtype=torch.float32, device=reg.device)
        ws = torch.empty(L.prb_stage_loss_workspace_bytes(rows), dtype=torch.uint8, device=reg.device)
        with torch.cuda.device(reg.device):
            C.check(L.prb_stage_loss_forward(ctypes.byref(desc), rows, reg.shape[1], C.ptr(cls), C.ptr(reg), C.ptr(label), label.element_size(),
                                             C.ptr(fg_mask), 0 if fg_mask is None else fg_mask.element_size(), C.ptr(reg_label),
                                             C.ptr(mean_size), C.ptr(anchor_boxes), C.ptr(ce_weight), C.ptr(total), C.ptr(vec), C.ptr(ws),
                                             ws.numel(), C.stream()), "stage_loss_forward")
        ctx.desc = desc
        ctx.save_for_backward(cls, reg, label, fg_mask, reg_label, mean_size, anchor_boxes, ce_weight, vec)
        ctx.set_materialize_grads(False)
        return total, vec

    @staticmethod
    def backward(ctx, g_total, g_vec):
        cls, reg, label, fg_mask, reg_label, mean_size, anchor_boxes, ce_weight, vec = ctx.saved_tensors
        if g_total is None and g_vec is None:
            return (None,) * 9
        g_total = None if g_total is None else g_total.float().contiguous()
        g_vec = None if g_vec is None else g_vec.float().contiguous()
        d_cls, d_reg = torch.empty_like(cls), torch.empty_like(reg)
        with torch.cuda.device(reg.device):
            C.check(C.lib().prb_stage_loss_backward(ctypes.byref(ctx.desc), reg.shape[0], reg.shape[1], C.ptr(cls), C.ptr(reg), C.ptr(label),
                                                    label.element_size(), C.ptr(fg_mask), 0 if fg_mask is None else fg_mask.element_size(),
                                                    C.ptr(reg_label), C.ptr(mean_size), C.ptr(anchor_boxes), C.ptr(ce_weight), C.ptr(vec),
                                                    C.ptr(g_total), C.ptr(g_vec), C.ptr(d_cls), C.ptr(d_reg), C.stream()),
                    "stage_loss_backward")
        return d_cls, d_reg, None, None, None, None, None, None, None


def _f32(t, what):
    C.require_cuda(t)
    if t.dtype != torch.float32:
        raise TypeError("device loss: %s must be float32, not %s" % (what, t.dtype))
    return t.contiguous()


def _int_rows(t, n, what):
    """int32 / int64 rows as they are; another dtype as the mirror reads it (label.float() compared with 0, or mask > 0)"""
    C.require_cuda(t)
    t = t.reshape(-1)
    if t.numel() != n:
        raise ValueError("device loss: %s has %d rows, the regression input %d" % (what, t.numel(), n))
    if t.dtype not in (torch.int32, torch.int64):
        t = t.long() if what == "labels" else (t > 0).to(torch.int32)
    return t.contiguous()


def _reg_keys(xz_fine, y_by_bin):
    keys = ["loss_x_bin", "loss_z_bin"] + (["loss_x_res", "loss_z_res"] if xz_fine else [])
    keys += ["loss_y_bin", "loss_y_res"] if y_by_bin else ["loss_y_offset"]
    return keys + ["loss_ry_bin", "loss_ry_res", "loss_loc", "loss_angle", "loss_size"]


def _desc(loss_cls, num_class, focal_alpha, focal_gamma, fg_weight, loss_weight, loc_scope, loc_bin_size, num_head_bin, xz_fine, y_by_bin,
          ry_fine, loc_y_scope, loc_y_bin_size):
    if focal_alpha is None:
        raise NotImplementedError("device loss: focal_alpha=None")
    return C.StageLossDesc(cls_loss=_CLS_CODE[loss_cls], num_class=num_class, focal_alpha=focal_alpha, focal_gamma=focal_gamma or 0.0,
                           fg_weight=fg_weight, loss_weight_cls=loss_weight[0], loss_weight_reg=loss_weight[1], loc_scope=loc_scope,
                           loc_bin_size=loc_bin_size, num_head_bin=num_head_bin, xz_fine=int(bool(xz_fine)), y_by_bin=int(bool(y_by_bin)),
                           ry_fine=int(bool(ry_fine)), loc_y_scope=loc_y_scope, loc_y_bin_size=loc_y_bin_size)


def _mean_size(mean_size, device):
    return torch.as_tensor(mean_size, dtype=torch.float32, device=device).reshape(3).contiguous()


def _rpn_loss_device(rpn_cls, rpn_reg, rpn_cls_label, rpn_reg_label, mean_size, loss_cls, focal_alpha, focal_gamma, fg_weight, loc_scope,
                     loc_bin_size, num_head_bin, loc_xz_fine, loss_weight):
    if loss_cls not in ("SigmoidFocalLoss", "DiceLoss", "BinaryCrossEntropy"):
        raise NotImplementedError(loss_cls)
    npts = rpn_reg.size(0) * rpn_reg.size(1)
    reg = _f32(rpn_reg, "rpn_reg").view(npts, -1)
    cls = _f32(rpn_cls, "rpn_cls").view(npts, 1)
    label = _int_rows(rpn_cls_label, npts, "labels")
    reg_label = _f32(rpn_reg_label, "rpn_reg_label").view(npts, 7)
    desc = _desc(loss_cls, 1, focal_alpha, focal_gamma, fg_weight, loss_weight, loc_scope, loc_bin_size, num_head_bin, loc_xz_fine, False,
                 False, 0.5, 0.25)
    total, vec = _StageLoss.apply(cls, reg, desc, label, None, reg_label, _mean_size(mean_size, reg.device), None, None)
    terms = {k: vec[_SLOT[k]] for k in _reg_keys(loc_xz_fine, False)}
    terms.update(rpn_loss_cls=vec[_SLOT["loss_cls"]], rpn_loss_reg=vec[_SLOT["loss_reg"]], rpn_loss=total)
    return total, terms


def _rcnn_loss_device(rcnn_cls, rcnn_reg, cls_label, reg_valid_mask, roi_boxes3d, gt_of_rois, mean_size, loss_cls, focal_alpha, focal_gamma,
                      size_res_on_roi, loc_scope, loc_bin_size, num_head_bin, loc_y_by_bin, loc_y_scope, loc_y_bin_size, ce_weight):
    if loss_cls not in ("SigmoidFocalLoss", "BinaryCrossEntropy", "CrossEntropy"):
        raise NotImplementedError(loss_cls)
    R = rcnn_reg.shape[0]
    reg = _f32(rcnn_reg, "rcnn_reg").view(R, -1)
    cls = _f32(rcnn_cls, "rcnn_cls").view(R, -1)
    if loss_cls != "CrossEntropy" and cls.shape[1] != 1:
        raise ValueError("device loss: %s takes one logit per RoI, not %d" % (loss_cls, cls.shape[1]))
    label = _int_rows(cls_label, R, "labels")
    fg = _int_rows(reg_valid_mask, R, "reg_valid_mask")
    gt = _f32(gt_of_rois, "gt_of_rois").view(R, 7)
    anchor = _f32(roi_boxes3d, "roi_boxes3d").view(R, 7) if size_res_on_roi else None
    w = None if ce_weight is None or loss_cls != "CrossEntropy" else _f32(ce_weight, "ce_weight").view(-1)
    if w is not None and w.numel() != cls.shape[1]:
        raise ValueError("device loss: %d class weights for %d classes" % (w.numel(), cls.shape[1]))
    desc = _desc(loss_cls, cls.shape[1], focal_alpha, focal_gamma, 1.0, (1.0, 1.0), loc_scope, loc_bin_size, num_head_bin, True, loc_y_by_bin,
                 True, loc_y_scope, loc_y_bin_size)
    total, vec = _StageLoss.apply(cls, reg, desc, label, fg, gt, _mean_size(mean_size, reg.device), anchor, w)
    terms = {}
    if loss_cls == "SigmoidFocalLoss":
        terms["rpn_loss_cls_pos"], terms["rpn_loss_cls_neg"] = vec[_SLOT["cls_pos"]], vec[_SLOT["cls_neg"]]     # the reference's key names
    terms.update({k: vec[_SLOT[k]] for k in _reg_keys(True, loc_y_by_bin)})
    terms.update(rcnn_loss_cls=vec[_SLOT["loss_cls"]], rcnn_loss_reg=vec[_SLOT["loss_reg"]], rcnn_loss=total)
    return total, terms
