"""oracle/proposal.py -- CPU restatement (numpy, fp32 step by step) of the RPN proposal path.  TEST INFRASTRUCTURE ONLY.

Follows, operation for operation:
  * decode_bbox_target          lib/utils/bbox_transform.py:24-121 (the RPN call of lib/rpn/proposal_layer.py:23-31:
                                roi_box3d = xyz (N,3), get_y_by_bin=False, get_ry_fine=False)
  * ProposalLayer.forward       lib/rpn/proposal_layer.py:15-56
  * distance_based_proposal     lib/rpn/proposal_layer.py:58-118
  * score_based_proposal        lib/rpn/proposal_layer.py:120-142
  * boxes3d_to_bev_torch        lib/utils/kitti_utils.py:134-147
  * nms_gpu / nms_normal_gpu    lib/utils/iou3d/iou3d_utils.py:56-87 (through oracle.nms)
Pinned by tests/golden/proposal_layer.npz, which holds the outputs of the reference's own Python run on the CPU
(oracle/make_golden_proposal.py).  Every torch op of the reference is one fp32 rounding; numpy float32 arithmetic
reproduces that as long as no two ops are fused, which is how the expressions below are written.
"""
import numpy as np

from . import oracle as O

F = np.float32


def _argmax(a):
    """torch.argmax over dim 1: the first maximum, and the first NaN when a row holds one (np.argmax agrees)"""
    return np.argmax(a, axis=1)


def descending(scores):
    """torch.sort(descending=True)'s order where no two scores tie: NaN first, then the values from the largest"""
    s = np.asarray(scores, dtype=F)
    return np.lexsort((-np.where(np.isnan(s), F(0), s), ~np.isnan(s)))


def decode_bbox_target(xyz, pred_reg, anchor_size, loc_scope, loc_bin_size, num_head_bin, get_xz_fine=True):
    """xyz (N,3), pred_reg (N,C) -> (N,7) [x, y, z, h, w, l, ry]; bbox_transform.py:40-121"""
    xyz = np.asarray(xyz, dtype=F)
    reg = np.asarray(pred_reg, dtype=F)
    anchor = np.asarray(anchor_size, dtype=F)
    nb = int(loc_scope / loc_bin_size) * 2                                   # :41
    x_bin = _argmax(reg[:, 0:nb])                                           # :49
    z_bin = _argmax(reg[:, nb:2 * nb])                                      # :50
    pos_x = x_bin.astype(F) * F(loc_bin_size) + F(loc_bin_size / 2) - F(loc_scope)   # :52
    pos_z = z_bin.astype(F) * F(loc_bin_size) + F(loc_bin_size / 2) - F(loc_scope)   # :53
    start = 2 * nb
    if get_xz_fine:                                                          # :55-67
        x_res = np.take_along_axis(reg[:, 2 * nb:3 * nb], x_bin[:, None], axis=1)[:, 0] * F(loc_bin_size)
        z_res = np.take_along_axis(reg[:, 3 * nb:4 * nb], z_bin[:, None], axis=1)[:, 0] * F(loc_bin_size)
        pos_x = pos_x + x_res
        pos_z = pos_z + z_res
        start = 4 * nb
    pos_y = xyz[:, 1] + reg[:, start]                                        # :84
    start += 1
    ry_bin = _argmax(reg[:, start:start + num_head_bin])                    # :90
    ry_res_norm = np.take_along_axis(reg[:, start + num_head_bin:start + 2 * num_head_bin], ry_bin[:, None], axis=1)[:, 0]
    angle_per_class = (2 * np.pi) / num_head_bin                             # :98
    ry_res = ry_res_norm * F(angle_per_class / 2)                            # :99
    ry = ry_bin.astype(F) * F(angle_per_class) + ry_res                      # :102
    two_pi = F(2 * np.pi)
    with np.errstate(invalid="ignore"):                                      # an infinite or NaN ry gives NaN
        m = np.fmod(ry, two_pi)                                              # torch.remainder = fmod, then sign fix-up
    m = np.where((m != 0) & (m < 0), m + two_pi, m).astype(F)
    ry = m
    ry = np.where(ry > F(np.pi), ry - two_pi, ry).astype(F)                  # :103
    s = start + 2 * num_head_bin
    assert s + 3 == reg.shape[1]                                             # :107
    hwl = reg[:, s:s + 3] * anchor[None] + anchor[None]                      # :110
    out = np.concatenate([pos_x[:, None], pos_y[:, None], pos_z[:, None], hwl, ry[:, None]], axis=1).astype(F)
    out[:, 0] = out[:, 0] + xyz[:, 0]                                        # :119 (roi_box3d has 3 columns: no rotation)
    out[:, 2] = out[:, 2] + xyz[:, 2]
    return out


def boxes3d_to_bev(boxes3d):
    """kitti_utils.py:134-147"""
    b = np.asarray(boxes3d, dtype=F)
    bev = np.empty((b.shape[0], 5), dtype=F)
    half_l, half_w = b[:, 5] / F(2), b[:, 4] / F(2)
    bev[:, 0], bev[:, 1] = b[:, 0] - half_l, b[:, 2] - half_w
    bev[:, 2], bev[:, 3] = b[:, 0] + half_l, b[:, 2] + half_w
    bev[:, 4] = b[:, 6]
    return bev


def _nms(boxes_bev, scores, thresh, nms_type):
    """iou3d_utils.py:56-87: sort by score (descending), NMS at the C++ boundary, map back"""
    order = descending(scores)
    keep = O.nms(np.ascontiguousarray(boxes_bev[order]), float(thresh), normal=(nms_type == "normal"))
    return order[keep]


def distance_based_proposal(scores, proposals, order, pre_tot, post_tot, thresh, nms_type, near_empty="raise"):
    """proposal_layer.py:58-118.  With nothing in (0, 40] the reference stops on `assert i == 2`; near_empty="far_only"
    is the device's rule instead: the near range contributes no rows and the far range its survivors, from row 0"""
    ranges = [0, 40.0, 80.0]
    pre = [0, int(pre_tot * 0.7), pre_tot - int(pre_tot * 0.7)]
    post = [0, int(post_tot * 0.7), post_tot - int(post_tot * 0.7)]
    s_o, p_o = scores[order], proposals[order]
    dist = p_o[:, 2]
    first = (dist > ranges[0]) & (dist <= ranges[1])
    s_list, p_list = [], []
    for i in range(1, 3):
        mask = (dist > ranges[i - 1]) & (dist <= ranges[i])
        if mask.sum() != 0:
            cs, cp = s_o[mask][:pre[i]], p_o[mask][:pre[i]]
        elif i == 1 and near_empty == "far_only":
            continue
        else:
            assert i == 2, "%d" % i
            cs, cp = s_o[first][pre[i - 1]:][:pre[i]], p_o[first][pre[i - 1]:][:pre[i]]
        keep = _nms(boxes3d_to_bev(cp), cs, thresh, nms_type)[:post[i]]
        s_list.append(cs[keep])
        p_list.append(cp[keep])
    return np.concatenate(s_list), np.concatenate(p_list)


def score_based_proposal(scores, proposals, order, pre_tot, post_tot, thresh):
    """proposal_layer.py:120-142 (always the rotated NMS)"""
    cs, cp = scores[order][:pre_tot], proposals[order][:pre_tot]
    keep = _nms(boxes3d_to_bev(cp), cs, thresh, "rotate")[:post_tot]
    return cs[keep], cp[keep]


def proposal_layer(rpn_scores, rpn_reg, xyz, anchor_size, loc_scope=3.0, loc_bin_size=0.5, num_head_bin=12, get_xz_fine=True,
                   pre_nms_top_n=9000, post_nms_top_n=100, nms_thresh=0.8, nms_type="normal", distance_based=True, order=None,
                   near_empty="raise"):
    """proposal_layer.py:15-56 -> (ret_bbox3d (B,post,7), ret_scores (B,post)).  order (B,N): the per-scene score order
    to use instead of `descending` (the device's own torch.sort, so that how tied scores fall is the device's);
    near_empty: see distance_based_proposal"""
    scores = np.asarray(rpn_scores, dtype=F)
    B, N = scores.shape
    prop = decode_bbox_target(np.asarray(xyz, F).reshape(-1, 3), np.asarray(rpn_reg, F).reshape(B * N, -1), anchor_size,
                              loc_scope, loc_bin_size, num_head_bin, get_xz_fine)
    prop[:, 1] = prop[:, 1] + prop[:, 3] / F(2)                                # :32
    prop = prop.reshape(B, N, 7)
    ret_b = np.zeros((B, post_nms_top_n, 7), dtype=F)
    ret_s = np.zeros((B, post_nms_top_n), dtype=F)
    for k in range(B):
        # :36.  torch.sort need not order tied scores as `descending` does: tests with ties pass the device's order
        o = descending(scores[k]) if order is None else np.asarray(order[k])
        if distance_based:
            s, p = distance_based_proposal(scores[k], prop[k], o, pre_nms_top_n, post_nms_top_n, nms_thresh, nms_type, near_empty)
        else:
            s, p = score_based_proposal(scores[k], prop[k], o, pre_nms_top_n, post_nms_top_n, nms_thresh)
        ret_b[k, :p.shape[0]] = p
        ret_s[k, :s.shape[0]] = s
    return ret_b, ret_s
