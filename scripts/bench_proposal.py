"""RPN proposal layer: device path (csrc/proposal.cu) against the reference-shaped Python loop running on this repo's
own NMS natives (the algorithm of lib/rpn/proposal_layer.py: per-scene masks, two NMS calls with a host keep list).
B=16 scenes x 16384 points, TEST and TRAIN quotas of tools/cfgs/default.yaml.  CUDA events, 20 iterations."""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.append(os.path.join(ROOT, "oracle"))
from make_golden_proposal import rpn_outputs  # noqa: E402
from test_proposal import ANCHOR, MODES, _cfg  # noqa: E402
from pointrcnn_b200.iou3d import iou3d_utils  # noqa: E402
from pointrcnn_b200 import kitti_utils  # noqa: E402
from pointrcnn_b200.rpn.proposal_layer import ProposalLayer, decode_rpn_proposals  # noqa: E402


def loop_reference_shape(scores, proposals, pre_tot, post_tot, thresh, nms_type):
    """the reference's per-scene control flow (proposal_layer.py:34-118) on the H100 NMS natives"""
    B = scores.shape[0]
    ret_b = scores.new_zeros(B, post_tot, 7)
    ret_s = scores.new_zeros(B, post_tot)
    _, order = torch.sort(scores, dim=1, descending=True)
    pre = [0, int(pre_tot * 0.7), pre_tot - int(pre_tot * 0.7)]
    post = [0, int(post_tot * 0.7), post_tot - int(post_tot * 0.7)]
    rng = [0, 40.0, 80.0]
    for k in range(B):
        s_o, p_o = scores[k][order[k]], proposals[k][order[k]]
        dist = p_o[:, 2]
        first = (dist > rng[0]) & (dist <= rng[1])
        sl, pl = [], []
        for i in range(1, 3):
            m = (dist > rng[i - 1]) & (dist <= rng[i])
            if m.sum() != 0:
                cs, cp = s_o[m][:pre[i]], p_o[m][:pre[i]]
            else:
                cs, cp = s_o[first][pre[i - 1]:][:pre[i]], p_o[first][pre[i - 1]:][:pre[i]]
            bev = kitti_utils.boxes3d_to_bev_torch(cp)
            keep = (iou3d_utils.nms_normal_gpu if nms_type == "normal" else iou3d_utils.nms_gpu)(bev, cs, thresh)[:post[i]]
            sl.append(cs[keep]); pl.append(cp[keep])
        s_cat, p_cat = torch.cat(sl), torch.cat(pl)
        ret_b[k, :p_cat.shape[0]] = p_cat
        ret_s[k, :s_cat.shape[0]] = s_cat
    return ret_b, ret_s


def timeit(fn, it=20):
    for _ in range(3):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(it):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / it


def main():
    dev = torch.device("cuda", 0)
    out = {}
    scores, reg, xyz = rpn_outputs(16, 16384, 777)
    ts, tr, tx = (torch.from_numpy(a).to(dev) for a in (scores, reg, xyz))
    for mode in ("TEST", "TRAIN"):
        for nms_type in ("normal", "rotate"):
            layer = ProposalLayer(mode=mode, cfg=_cfg(nms_type, True))
            m = MODES[mode]
            got = layer(ts, tr, tx)
            props = decode_rpn_proposals(tx, tr, ANCHOR, 3.0, 0.5, 12, True)
            want = loop_reference_shape(ts, props, m["pre_nms_top_n"], m["post_nms_top_n"], m["nms_thresh"], nms_type)
            same = bool(torch.equal(got[0], want[0]) and torch.equal(got[1], want[1]))
            t_dev = timeit(lambda: layer(ts, tr, tx))
            t_loop = timeit(lambda: loop_reference_shape(ts, decode_rpn_proposals(tx, tr, ANCHOR, 3.0, 0.5, 12, True), m["pre_nms_top_n"],
                                                         m["post_nms_top_n"], m["nms_thresh"], nms_type), it=5)
            t_dec = timeit(lambda: decode_rpn_proposals(tx, tr, ANCHOR, 3.0, 0.5, 12, True))
            out["%s_%s" % (mode, nms_type)] = {"device_ms": t_dev, "decode_ms": t_dec, "python_loop_on_b200_natives_ms": t_loop,
                                               "identical": same, "scenes_per_s_device": 16 / (t_dev * 1e-3)}
            print(mode, nms_type, out["%s_%s" % (mode, nms_type)])
    if len(sys.argv) > 1:
        json.dump(out, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
