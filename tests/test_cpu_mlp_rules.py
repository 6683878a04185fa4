"""The rules that decide whether a fused kernel path can compute a stack of 1x1 convolutions, checked on the host: every
MLP and head stack the project's networks build is accepted, and blocks the kernels would compute differently from torch
(strided, padded or grouped convolutions, another activation, instance norm, pre-activation order) are refused, so they
take the torch path."""
import pytest
import torch.nn as nn

from pointrcnn_b200.backbone import Pointnet2MSG
from pointrcnn_b200.pointnet2 import pointnet2_modules as pm
from pointrcnn_b200.pointnet2 import pytorch_utils as pt_utils
from pointrcnn_b200.rcnn.stage import RCNNStage
from pointrcnn_b200.rpn.heads import FusedRPNHeads
from pointrcnn_b200.rpn.stage import RPNStage


def test_fused_rule_accepts_every_project_mlp():
    net = Pointnet2MSG(input_channels=1).eval()
    mlps = {"sa%d.%d" % (k, i): mlp for k, sa in enumerate(net.SA_modules) for i, mlp in enumerate(sa.mlps)}
    mlps.update({"fp%d" % k: fp.mlp for k, fp in enumerate(net.FP_modules)})
    for bn in (False, True):
        rcnn = RCNNStage(cfg=dict(USE_BN=bn)).eval()
        mlps.update({"rcnn sa%d bn=%d" % (k, bn): sa.mlps[0] for k, sa in enumerate(rcnn.SA_modules)})
        mlps["rcnn xyz_up bn=%d" % bn] = rcnn.xyz_up_layer
        mlps["rcnn merge bn=%d" % bn] = rcnn.merge_down_layer
    for name, mlp in mlps.items():
        assert pm._FusedMLP.supported(mlp), name


def _conv2d_groups_2():
    block = pt_utils.Conv2d(16, 32, bn=True)
    block.conv = nn.Conv2d(16, 32, kernel_size=1, groups=2, bias=False)
    return block


BAD_BLOCKS = {
    "stride_1x2": lambda: pt_utils.Conv2d(16, 32, stride=(1, 2), bn=True),
    "padding_0x1": lambda: pt_utils.Conv2d(16, 32, padding=(0, 1), bn=True),
    "groups_2": _conv2d_groups_2,
    "leaky_relu": lambda: pt_utils.Conv2d(16, 32, bn=True, activation=nn.LeakyReLU()),
    "instance_norm": lambda: pt_utils.Conv2d(16, 32, instance_norm=True),
}


@pytest.mark.parametrize("case", sorted(BAD_BLOCKS))
def test_fused_rule_rejects_a_block_the_kernel_computes_differently(case):
    mlp = pt_utils.SharedMLP([4, 16, 32], bn=True)
    assert pm._FusedMLP.supported(mlp.eval())
    mlp.layer1 = BAD_BLOCKS[case]()
    assert not pm._FusedMLP.supported(mlp.eval())


def test_fused_rule_rejects_layers_that_do_not_chain():
    mlp = pt_utils.SharedMLP([4, 16, 32], bn=True)
    mlp.layer1 = pt_utils.Conv2d(24, 32, bn=True)
    assert not pm._FusedMLP.supported(mlp.eval())


def test_heads_rule_accepts_the_rpn_heads():
    stage = RPNStage().eval()
    assert FusedRPNHeads.supported(stage.rpn_cls_layer, stage.rpn_reg_layer)


BAD_HEADS = {
    "leaky_relu": lambda: pt_utils.Conv1d(128, 128, bn=True, activation=nn.LeakyReLU()),
    "instance_norm": lambda: pt_utils.Conv1d(128, 128, instance_norm=True),
    "preact": lambda: pt_utils.Conv1d(128, 128, bn=True, preact=True),
}


@pytest.mark.parametrize("case", sorted(BAD_HEADS))
def test_heads_rule_rejects_a_stack_the_kernel_computes_differently(case):
    stage = RPNStage().eval()
    stage.rpn_cls_layer[0] = BAD_HEADS[case]()
    assert not FusedRPNHeads.supported(stage.rpn_cls_layer.eval(), stage.rpn_reg_layer)
