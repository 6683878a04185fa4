"""oracle/make_golden_proposal.py -- golden vectors for the RPN proposal path (SURVEY.md section 8(f) rank 1).

Runs the reference's OWN Python (`lib/rpn/proposal_layer.py`, `lib/utils/bbox_transform.py`, `lib/utils/kitti_utils.py`,
unmodified, imported from /root/reference) on the CPU of this container, on seeded synthetic RPN outputs, and stores
its results in tests/golden/proposal_layer.npz.  Only three things outside those files are substituted, because the
reference hard-wires CUDA: `Tensor.cuda()` is the identity, `Tensor.get_device()` names the CPU, and the two NMS entry
points of `lib.utils.iou3d.iou3d_utils` call the CPU oracle's NMS (oracle/pointops_oracle.c, itself pinned to the
reference's CUDA NMS by tests/golden/reference_kernels.npz).  Usage (here, not on the GPU box):
    python oracle/make_golden_proposal.py
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = "/root/reference"
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

CASES = [
    # name, mode, nms type, distance based, B, N, seed
    ("test_normal", "TEST", "normal", True, 2, 16384, 101),
    ("test_rotate", "TEST", "rotate", True, 2, 16384, 102),
    ("train_normal", "TRAIN", "normal", True, 2, 16384, 103),
    ("test_score_based", "TEST", "rotate", False, 1, 16384, 104),
    ("test_far_area_empty", "TEST", "normal", True, 1, 16384, 105),
]


def rpn_outputs(B, N, seed, far_empty=False):
    """synthetic (rpn_scores, rpn_reg, xyz): points in the KITTI scope, confident scores around a few 'objects' so that
    NMS has real clusters to prune, random bin logits and residuals"""
    rng = np.random.default_rng(seed)
    xyz = np.stack([rng.uniform(-40, 40, (B, N)), rng.uniform(-1, 3, (B, N)), rng.uniform(0.5, 38.0 if far_empty else 70.4, (B, N))], axis=-1)
    centres = np.stack([rng.uniform(-30, 30, (B, 12)), rng.uniform(0, 2, (B, 12)), rng.uniform(5, 35.0 if far_empty else 65, (B, 12))], axis=-1)
    d = np.linalg.norm(xyz[:, :, None, :] - centres[:, None, :, :], axis=-1).min(axis=2)
    scores = 4.0 * np.exp(-d / 3.0) + rng.normal(0, 1.0, (B, N))
    reg = rng.normal(0, 1.0, (B, N, 76))
    reg[..., 48] *= 0.3          # y offset
    reg[..., 73:76] *= 0.1       # size residuals
    return scores.astype(np.float32), reg.astype(np.float32), xyz.astype(np.float32)


def install_reference():
    """import the reference's ProposalLayer, cfg and decode_bbox_target with the CPU stand-ins described above"""
    from pointrcnn_b200 import dropin
    from oracle import oracle as O
    dropin._install_compat()
    sys.path.insert(0, REF)
    stub = types.ModuleType("lib.utils.iou3d.iou3d_utils")

    def _nms(boxes, scores, thresh, normal):
        order = scores.sort(0, descending=True)[1]
        keep = O.nms(boxes[order].contiguous().numpy(), float(thresh), normal=normal)
        return order[torch.from_numpy(keep)].contiguous()

    stub.nms_gpu = lambda boxes, scores, thresh: _nms(boxes, scores, thresh, False)
    stub.nms_normal_gpu = lambda boxes, scores, thresh: _nms(boxes, scores, thresh, True)
    import lib.utils  # noqa: F401  (the reference's own package)
    pkg = types.ModuleType("lib.utils.iou3d")
    pkg.__path__ = []
    sys.modules["lib.utils.iou3d"] = pkg
    sys.modules["lib.utils.iou3d.iou3d_utils"] = stub
    pkg.iou3d_utils = stub
    torch.Tensor.cuda = lambda self, *a, **k: self
    torch.Tensor.get_device = lambda self: "cpu"
    from lib.config import cfg, cfg_from_file
    cfg_from_file(os.path.join(REF, "tools/cfgs/default.yaml"))
    from lib.rpn.proposal_layer import ProposalLayer
    from lib.utils.bbox_transform import decode_bbox_target
    return ProposalLayer, cfg, decode_bbox_target


def main():
    ProposalLayer, cfg, decode_bbox_target = install_reference()
    out = {}
    for name, mode, nms_type, dist_based, B, N, seed in CASES:
        cfg.RPN.NMS_TYPE = nms_type
        cfg.TEST.RPN_DISTANCE_BASED_PROPOSE = dist_based
        scores, reg, xyz = rpn_outputs(B, N, seed, far_empty=name.endswith("far_area_empty"))
        layer = ProposalLayer(mode=mode)
        with torch.no_grad():
            boxes, sc = layer(torch.from_numpy(scores), torch.from_numpy(reg), torch.from_numpy(xyz))
        out[name + "_boxes"] = boxes.numpy()
        out[name + "_scores"] = sc.numpy()
        print(name, boxes.shape, "non-empty rows per scene:", [(sc[b] != 0).sum().item() for b in range(B)])
    # decode alone (all points of one case), to pin the arithmetic
    scores, reg, xyz = rpn_outputs(2, 4096, 106)
    dec = decode_bbox_target(torch.from_numpy(xyz).view(-1, 3), torch.from_numpy(reg).view(-1, 76),
                             anchor_size=torch.from_numpy(cfg.CLS_MEAN_SIZE[0]), loc_scope=cfg.RPN.LOC_SCOPE,
                             loc_bin_size=cfg.RPN.LOC_BIN_SIZE, num_head_bin=cfg.RPN.NUM_HEAD_BIN,
                             get_xz_fine=cfg.RPN.LOC_XZ_FINE, get_y_by_bin=False, get_ry_fine=False)
    out["decode_boxes"] = dec.numpy()
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "proposal_layer.npz"), **out)
    print("wrote tests/golden/proposal_layer.npz")


if __name__ == "__main__":
    main()
