"""RPN classification + regression heads on the tensor-core chain kernel (SURVEY.md section 8(f) rank 3).

The reference runs two Conv1d stacks over the backbone features (lib/net/rpn.py:19-47, :76-77):
    rpn_cls_layer = Conv1d(C,128,bn) - Dropout - Conv1d(128,1, activation=None)
    rpn_reg_layer = Conv1d(C,128,bn) - Dropout - Conv1d(128,reg_channel, activation=None)
and transposes both results to point-major.  In eval mode (Dropout = identity, BN = running statistics) the two stacks
are ONE two-layer MLP over point-major rows: layer 0 stacks the two hidden layers (C -> 256, BN folded into the
weights, ReLU), layer 1 is block diagonal (256 -> 1 + reg_channel, linear: `prb_mlp_desc.flags & 1`).  The rows are
the point-major twin the last FP level already wrote, the output rows are already (B,N,·): no transposes, one launch.
"""
import torch
import torch.nn as nn

from .. import mlp_chain
from ..pointnet2 import pointnet2_modules as pm


def _layers(seq):
    """[(conv, bn or None, relu)] of a reference head stack, Dropout skipped (the identity in eval mode); None unless every
    other child is a plain conv block (pointnet2_modules.read_block)"""
    out = [pm.read_block(layer) for layer in seq.children() if not isinstance(layer, nn.Dropout)]
    return None if any(b is None for b in out) else out


class FusedRPNHeads:
    """cache of the packed two-layer chain of (rpn_cls_layer, rpn_reg_layer); rebuilt when a parameter or buffer is
    replaced or its version changes (pointnet2_modules.tensor_stamp)"""

    def __init__(self):
        self.device = None
        self.stamp = None
        self.chain = None
        self.n_cls = None

    @staticmethod
    def supported(cls_seq, reg_seq):
        a, b = _layers(cls_seq), _layers(reg_seq)
        if a is None or b is None:
            return False
        ok = len(a) == 2 and len(b) == 2 and a[0][2] and b[0][2] and not a[1][2] and not b[1][2]
        ok = ok and a[0][0].in_channels == b[0][0].in_channels and a[0][0].out_channels + b[0][0].out_channels <= 512
        return ok and all(bn is None or not bn.training for _, bn, _ in a + b)

    @staticmethod
    def _build(cls_seq, reg_seq, device):
        """-> (chain, number of classification channels)"""
        (c0, cb0, _), (c1, _, _) = _layers(cls_seq)
        (r0, rb0, _), (r1, _, _) = _layers(reg_seq)
        Wc0, _, sc0 = mlp_chain.fold(c0, cb0, zero_bias=True)
        Wr0, _, sr0 = mlp_chain.fold(r0, rb0, zero_bias=True)
        Wc1, _, sc1 = mlp_chain.fold(c1, None)
        Wr1, _, sr1 = mlp_chain.fold(r1, None)
        hc, hr = Wc0.shape[0], Wr0.shape[0]
        W0 = torch.cat([Wc0, Wr0], 0)
        W1 = torch.zeros(Wc1.shape[0] + Wr1.shape[0], hc + hr)
        W1[:Wc1.shape[0], :hc] = Wc1
        W1[Wc1.shape[0]:, hc:] = Wr1
        chain = mlp_chain.Chain(mlp_chain.ROWS, 0, [W0, W1], [torch.cat([sc0, sr0]), torch.cat([sc1, sr1])], linear_last=True,
                                device=device)
        return chain, Wc1.shape[0]

    def __call__(self, cls_seq, reg_seq, features):
        """features (B,C,N) -> rpn_cls (B,N,n_cls), rpn_reg (B,N,reg_channel), as lib/net/rpn.py:76-77"""
        tensors = [p for seq in (cls_seq, reg_seq) for p in list(seq.parameters()) + list(seq.buffers())]
        stamp = pm.tensor_stamp(tensors)
        if str(features.device) != self.device or not pm.stamp_matches(self.stamp, stamp):
            self.chain, self.n_cls = self._build(cls_seq, reg_seq, features.device)
            self.device, self.stamp = str(features.device), stamp
        B, Cc, N = features.shape
        rows = pm._point_major(features)            # (B,N,C): the twin written by the last FP launch, or one transpose
        out = self.chain.rows(rows.view(B * N, Cc)).view(B, N, -1)
        return out[:, :, :self.n_cls].contiguous(), out[:, :, self.n_cls:self.chain.c_out[-1]].contiguous()


def rpn_heads(rpn_module, backbone_features):
    """eval-mode replacement of `rpn_cls_layer(f).transpose(1,2).contiguous()`, `rpn_reg_layer(f).transpose(...)`
    for a reference lib.net.rpn.RPN instance (or anything with the same two attributes).  The packed chain is cached on
    `rpn_module`; invalidate_heads() drops it."""
    cache = rpn_module.__dict__.setdefault("_prb_heads", FusedRPNHeads())
    fused_ok = (not torch.is_grad_enabled()) and not rpn_module.training and pm._fused_enabled() and \
        FusedRPNHeads.supported(rpn_module.rpn_cls_layer, rpn_module.rpn_reg_layer)
    if not fused_ok:
        return (rpn_module.rpn_cls_layer(backbone_features).transpose(1, 2).contiguous(),
                rpn_module.rpn_reg_layer(backbone_features).transpose(1, 2).contiguous())
    return cache(rpn_module.rpn_cls_layer, rpn_module.rpn_reg_layer, backbone_features)


def invalidate_heads(rpn_module):
    """drop the packed heads chain rpn_heads() cached on `rpn_module`: after weights were edited through `.data`, which
    bumps no version counter, and whenever the module's tensors are converted (RPNStage._apply)"""
    rpn_module.__dict__.pop("_prb_heads", None)
