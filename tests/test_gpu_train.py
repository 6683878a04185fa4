"""Training path on the H100 natives (BASELINE configs[2], VERDICT r1 row x1): gradients through the op-by-op path -- this
repo's gather / grouping / interpolation forward kernels and their atomic scatter backward kernels, cuDNN MLPs -- against
the same network with every index op expressed in plain torch (advanced indexing, torch autograd), and the RPN training
step (batch-statistics BN, bin-based loss, bucketed gradient reducer, fused Adam)."""
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import synth  # noqa: E402
from pointrcnn_b200.backbone import Pointnet2MSG  # noqa: E402
from pointrcnn_b200.pointnet2 import pointnet2_utils as pu  # noqa: E402

pytestmark = pytest.mark.gpu


def _torch_gather(features, idx):            # (B,C,N), (B,M) -> (B,C,M)
    return torch.gather(features, 2, idx.long().unsqueeze(1).expand(-1, features.size(1), -1))


def _torch_group(features, idx):             # (B,C,N), (B,M,S) -> (B,C,M,S)
    B, C, _ = features.shape
    _, M, S = idx.shape
    return torch.gather(features, 2, idx.long().view(B, 1, M * S).expand(-1, C, -1)).view(B, C, M, S)


def _torch_interp(features, idx, weight):    # (B,C,M), (B,N,3), (B,N,3) -> (B,C,N)
    B, C, _ = features.shape
    N = idx.shape[1]
    g = torch.gather(features, 2, idx.long().view(B, 1, N * 3).expand(-1, C, -1)).view(B, C, N, 3)
    return (g * weight.unsqueeze(1)).sum(dim=3)


def _run(net, pc, pure_torch):
    saved = (pu.gather_operation, pu.grouping_operation, pu.three_interpolate)
    if pure_torch:
        pu.gather_operation, pu.grouping_operation, pu.three_interpolate = _torch_gather, _torch_group, _torch_interp
    try:
        net.zero_grad(set_to_none=True)
        x = pc.clone().requires_grad_(True)
        xyz, feats = net(x)
        loss = (feats * torch.linspace(0.5, 1.5, feats.shape[2], device=feats.device)).pow(2).mean() + feats.abs().mean()
        loss.backward()
        return feats.detach(), x.grad.clone(), [p.grad.clone() for p in net.parameters()]
    finally:
        pu.gather_operation, pu.grouping_operation, pu.three_interpolate = saved


def test_backbone_gradients_match_pure_torch_index_ops(cuda):
    """d loss / d (weights, BN affine, input intensity) through K3 / K6 / K9 (gather / group / interpolate grad kernels)
    == the gradients torch autograd derives when the same index ops are written with torch.gather (<= 1e-3 of the
    gradient's scale; atomicAdd order only perturbs the last bits)"""
    old = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        torch.manual_seed(31)
        cfg = dict(USE_BN=True, NPOINTS=[512, 128, 32], RADIUS=[[0.1, 0.5], [0.5, 1.0], [1.0, 2.0]], NSAMPLE=[[16, 32], [16, 32], [16, 32]],
                   MLPS=[[[16, 16, 32], [32, 32, 64]], [[64, 64, 128], [64, 96, 128]], [[128, 196, 256], [128, 196, 256]]],
                   FP_MLPS=[[64, 64], [128, 128], [256, 256]])
        net = Pointnet2MSG(input_channels=1, cfg=cfg).to(cuda).train()
        pc = torch.from_numpy(synth.u_kitti(2, 4096, 77, channels=4)).to(cuda)
        pc[..., :3] /= 10.0                                   # denser balls: real neighbourhoods at these radii
        f1, gx1, gp1 = _run(net, pc, pure_torch=False)
        f2, gx2, gp2 = _run(net, pc, pure_torch=True)
        # interpolation: the native kernel uses the reference's FMA order, torch.gather + sum another one -> last-bit noise only
        assert (f1 - f2).abs().max().item() <= 1e-4 * f2.abs().max().item(), "forward differs between native and torch index ops"
        assert (gx1[..., 3:] - gx2[..., 3:]).abs().max().item() <= 1e-3 * gx2[..., 3:].abs().max().item()
        # norm-wise over the whole gradient (the judged bound, 1e-3); per parameter a looser bound: weights in front of a
        # train-mode BatchNorm have near-cancelling gradients, so their own scale is small against the atomicAdd-order noise
        ga, gb = torch.cat([g.reshape(-1) for g in gp1]), torch.cat([g.reshape(-1) for g in gp2])
        assert ((ga - gb).norm() / gb.norm()).item() <= 1e-3, "gradient differs: %g" % ((ga - gb).norm() / gb.norm()).item()
        assert (ga - gb).abs().max().item() <= 1e-3 * gb.abs().max().item()
        worst = max(((a - b).abs().max() / b.abs().max().clamp_min(1e-12)).item() for a, b in zip(gp1, gp2))
        assert worst <= 1e-2, "parameter gradients differ: %g" % worst
        assert all(g.abs().sum() > 0 for g in gp2)
    finally:
        torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = old


def test_rpn_training_step_runs_and_learns(cuda):
    """a few optimizer steps on one fixed batch: the loss falls, BN running statistics move, gradients stay inside the
    reducer's buckets, nothing becomes non-finite"""
    from pointrcnn_b200.train.step import RPNTrainer, synthetic_labels
    tr = RPNTrainer(input_channels=1, device=cuda, world=1, lr=0.002, seed=3)
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 123, channels=4)).to(cuda)
    cls, reg = synthetic_labels(pc, seed=1)
    bn = next(m for m in tr.model.modules() if isinstance(m, torch.nn.BatchNorm2d))
    rm0 = bn.running_mean.clone()
    losses = []
    for _ in range(6):
        loss, terms = tr.step(pc, cls, reg, grad_norm_clip=1.0)
        losses.append(float(loss))
    assert all(np.isfinite(losses)) and losses[-1] < losses[0], losses
    assert not torch.equal(bn.running_mean, rm0)
    for p in tr.params:
        b = tr.reducer.buckets[tr.reducer._owner[p]]["flat"]
        assert b.data_ptr() <= p.grad.data_ptr() < b.data_ptr() + b.numel() * 4
    assert {"rpn_loss_cls", "rpn_loss_reg", "loss_x_bin", "loss_ry_res", "loss_size"} <= set(terms)


def test_rcnn_training_step_runs_and_learns(cuda):
    """RCNN phase with the RPN fixed: RPN stage (fused, no grad) -> target layer (64 RoIs per scene) -> RCNN network in training
    mode -> get_rcnn_loss mirror -> backward -> optimizer; GT boxes sit on proposals so that foreground RoIs exist"""
    from pointrcnn_b200.train.step import RCNNTrainer
    tr = RCNNTrainer(input_channels=1, device=cuda, world=1, lr=0.002, seed=5)
    with torch.no_grad():
        tr.rpn.rpn_reg_layer[-1].conv.weight.mul_(0.2)            # usable box sizes on random weights (as in the chain test)
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 321, channels=4)).to(cuda)
    rois = tr.rpn_outputs(pc, None)["roi_boxes3d"]
    gt = torch.zeros((2, 12, 7), device=cuda)
    gt[:, :8] = rois[:, ::40][:, :8]                               # 8 GT boxes per scene = 8 of the proposals; 4 padding rows
    assert (gt[:, :8, 3:6] > 0).all(), "degenerate proposals"
    w0 = tr.model.cls_layer[0].conv.weight.detach().clone()
    losses = []
    for _ in range(5):
        loss, terms = tr.step(pc, gt, grad_norm_clip=1.0)
        losses.append(float(loss))
    assert all(np.isfinite(losses)), losses
    assert not torch.equal(tr.model.cls_layer[0].conv.weight, w0), "the optimizer did not move the RCNN parameters"
    assert all(p.grad is None for p in tr.rpn.parameters()), "the fixed RPN must not receive gradients"
    assert {"rcnn_loss_cls", "rcnn_loss_reg", "rcnn_loss"} <= set(terms)
    ret = tr.model.forward_train(tr.rpn_outputs(pc, gt))
    assert ret["rcnn_cls"].shape[0] == 2 * 64 and ret["pts_input"].shape[1:] == (512, 133)
    assert int((ret["reg_valid_mask"] > 0).sum()) > 0, "no foreground RoI: the regression branch is not exercised"
