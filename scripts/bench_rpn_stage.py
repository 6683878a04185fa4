"""Full RPN stage (backbone -> cls/reg heads -> proposal layer, TEST quotas), B=16 x 16384 points, pipelined:
everything on the H100 path against the same backbone followed by torch heads + the reference-shaped Python proposal
loop on this repo's NMS natives.  Random weights, synthetic scenes (scores are not meaningful, the work is)."""
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.append(os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "scripts"))
import synth  # noqa: E402
from bench_proposal import loop_reference_shape  # noqa: E402
from test_proposal import ANCHOR, MODES, _cfg  # noqa: E402
from pointrcnn_b200.backbone import Pointnet2MSG  # noqa: E402
from pointrcnn_b200.pipeline import BatchPipeline  # noqa: E402
from pointrcnn_b200.pointnet2 import pytorch_utils as pt_utils  # noqa: E402
from pointrcnn_b200.rpn.heads import rpn_heads  # noqa: E402
from pointrcnn_b200.rpn.proposal_layer import ProposalLayer, decode_rpn_proposals  # noqa: E402


class RPNStage(nn.Module):
    def __init__(self):
        super().__init__()
        self.backbone_net = Pointnet2MSG(input_channels=1)
        self.rpn_cls_layer = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 1, activation=None))
        self.rpn_reg_layer = nn.Sequential(pt_utils.Conv1d(128, 128, bn=True), nn.Dropout(0.5), pt_utils.Conv1d(128, 76, activation=None))
        self.proposal_layer = ProposalLayer(mode="TEST", cfg=_cfg("normal", True))

    def forward(self, pts, fused=True):
        xyz, feats = self.backbone_net(pts)
        if fused:
            cls, reg = rpn_heads(self, feats)
            return self.proposal_layer(cls[:, :, 0], reg, xyz)
        cls = self.rpn_cls_layer(feats).transpose(1, 2).contiguous()
        reg = self.rpn_reg_layer(feats).transpose(1, 2).contiguous()
        m = MODES["TEST"]
        props = decode_rpn_proposals(xyz, reg, ANCHOR, 3.0, 0.5, 12, True)
        return loop_reference_shape(cls[:, :, 0].contiguous(), props, m["pre_nms_top_n"], m["post_nms_top_n"], m["nms_thresh"], "normal")


def main():
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    net = RPNStage().to(dev).eval()
    net.backbone_net.FP_modules[0].emit_point_major = True        # the heads read the point-major twin
    pool = [torch.from_numpy(synth.u_kitti(16, 16384, 900 + i, channels=4)).to(dev) for i in range(12)]
    out = {}
    with torch.no_grad():
        for name, fused, steps in (("b200_path", True, 36), ("torch_heads_python_proposals", False, 6)):
            pipe = BatchPipeline(lambda x: net(x, fused)[0], inflight=6, device=dev)
            pipe.run([pool[i % 12] for i in range(6)], keep=False)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            pipe.run([pool[i % 12] for i in range(steps)], keep=False)
            b.record()
            torch.cuda.synchronize()
            ms = a.elapsed_time(b) / steps
            out[name] = {"ms_per_batch": ms, "scenes_per_s": 16 / (ms * 1e-3)}
            print(name, out[name])
        r1, r2 = net(pool[0], True), net(pool[0], False)
        out["rois_identical_given_same_heads"] = None
        print("rois from both paths: shapes", tuple(r1[0].shape), tuple(r2[0].shape), "max |diff| of kept scores", float((r1[1] - r2[1]).abs().max()))
    if len(sys.argv) > 1:
        json.dump(out, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
