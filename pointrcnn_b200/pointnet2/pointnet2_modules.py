"""Mirror of pointnet2_lib/pointnet2/pointnet2_modules.py (reference :10-160): PointnetSAModuleMSG,
PointnetSAModule, PointnetFPModule -- same constructor arguments, sub-module names (`groupers`, `mlps`,
`mlp`) and forward signatures, so checkpoints and lib/net/*.py work unchanged.

Two execution paths per module, chosen per call:
  fused    (no autograd graph needed, BatchNorm in eval mode or absent, max-pool, power-of-two nsample):
           FPS(+new_xyz) -> [one ball-query scan for both radii] -> per scale ONE tensor-core kernel that
           gathers the neighbourhood, runs the whole SharedMLP and max-pools (csrc/mlp_tc.cu).  FP modules:
           three_nn(+weights) -> ONE kernel that interpolates, concatenates the skip features and runs the MLP.
  train    (SA modules, opt-in with config.sa_train="device", autograd graph needed, batch-statistics BN or none, every
           layer at most sa_train.FAST_MAX_WIDTH wide):
           the fused path's sampling and ball query, then sa_train.py's autograd Function (csrc/sa_train.cu).
           FP modules (opt-in with config.fp_train="device", levels fp_train.FAST_LEVELS selects): the fused path's
           3-NN, then fp_train.py's autograd Function (csrc/sa_train.cu).
  unfused  (training / anything else): the reference's op-by-op sequence on the H100 natives with
           torch.nn convolutions, full autograd support.
`config.override(disable_fused=True)` forces the unfused path (used by tests to cross-check the two).
"""
from typing import List

import torch
import torch.nn as nn
import torch.nn.functional as F

from .. import config
from .. import mlp_chain
from . import pointnet2_utils
from . import fp_train
from . import pytorch_utils as pt_utils
from . import sa_train


_BLOCK_LAYOUTS = {("conv",), ("conv", "bn"), ("conv", "activation"), ("conv", "bn", "activation")}


def read_block(block):
    """(conv, bn or None, relu) of a pt_utils Conv1d / Conv2d block that is a plain 1x1 convolution, else None: children
    exactly conv [, bn] [, activation] in that order, the activation an nn.ReLU, and a Conv1d / Conv2d whose every kernel,
    stride and dilation entry is 1, with no padding and one group.  `bn` is the inner BatchNorm module.  This is what every
    device path computes for a block; anything else (instance norm, pre-activation order, strided or grouped convolutions)
    must take the torch path."""
    children = block._modules      # read once: the eval path evaluates this on every call, named_children() costs more
    if tuple(children) not in _BLOCK_LAYOUTS:
        return None
    conv, act = children["conv"], children.get("activation")
    if not isinstance(conv, (nn.Conv1d, nn.Conv2d)):
        return None
    ones = (1,) * len(conv.kernel_size)
    if not conv.kernel_size == conv.stride == conv.dilation == ones or conv.padding != (0,) * len(ones) or conv.groups != 1:
        return None
    if act is not None and not isinstance(act, nn.ReLU):
        return None
    bn = getattr(children["bn"], "bn", None) if "bn" in children else None
    if "bn" in children and bn is None:
        return None
    return conv, bn, act is not None


def read_mlp(mlp):
    """[(conv, bn or None, True)] of a SharedMLP of 1-3 plain blocks (read_block), each with ReLU, whose channels chain (the
    input width of block l is the output width of block l - 1), else None"""
    blocks = [read_block(layer) for layer in mlp.children()]
    if not 1 <= len(blocks) <= 3 or any(b is None or not b[2] for b in blocks):
        return None
    if any(b[0].in_channels != a[0].out_channels for a, b in zip(blocks, blocks[1:])):
        return None
    return blocks


def grouping_ok(module, n_points):
    """the grouping every device path of an SA module computes: max-pool over QueryAndGroup / GroupAll groups with use_xyz
    and a power-of-two sample count in 4..128 (GroupAll: the n_points of the input)"""
    if module.pool_method != "max_pool":
        return False
    for g in module.groupers:
        if isinstance(g, pointnet2_utils.QueryAndGroup):
            ns = g.nsample
        elif isinstance(g, pointnet2_utils.GroupAll):
            ns = n_points
        else:
            return False
        if not g.use_xyz or not 4 <= ns <= 128 or ns & (ns - 1):
            return False
    return True


def tensor_stamp(tensors):
    """[(tensor, version)] of the tensors a packed chain is built from, the tensors themselves held: a cache that compares
    stamps with stamp_matches() sees a replaced tensor (a new nn.Parameter, load_state_dict(assign=True)) even when it
    took the id() and the version of the one it replaced, and an in-place edit through its version counter.  Holding them
    keeps a replaced parameter's storage alive until the cache's next call rebuilds the chain (or its module's _apply /
    invalidate_fused drops it)."""
    return [(t, None if t is None else t._version) for t in tensors]


def stamp_matches(old, new):
    return old is not None and len(old) == len(new) and all(a is b and va == vb for (a, va), (b, vb) in zip(old, new))


class _FusedMLP:
    """The mlp_chain.Chain of one SharedMLP (folded BN, packed weights on the device), rebuilt whenever a parameter / buffer
    is replaced or its version changes (optimizer step, load_state_dict, in-place edits)."""

    def __init__(self):
        self.key = None
        self.stamp = None
        self.chain = None
        self.proj = None

    @staticmethod
    def supported(mlp: nn.Sequential):
        """read_mlp's SharedMLP, at most 512 wide, with no BatchNorm in training mode"""
        blocks = read_mlp(mlp)
        return blocks is not None and all(conv.out_channels <= 512 and (bn is None or not bn.training) for conv, bn, _ in blocks)

    def get(self, mlp: nn.Sequential, kind: int, split: int, device, project_known: bool = False):
        """-> the chain of `mlp`, packed as (kind, split) on `device`.
        project_known (FP chains, kind FP): layer 0 is split by linearity -- interp(known) @ W0k^T == interp(known @ W0k^T) --
        into a per-KNOWN-point projection (a separate, 4x smaller row GEMM: `self.proj`, linear, no shift) and a main chain
        whose layer 0 reads [interp(projected rows) | skip] through the weight [I | W0s]: the gather moves c_out0 instead of
        c_known floats per neighbour and layer 0 contracts over c_out0 + c_skip instead of c_known + c_skip columns."""
        layers = list(mlp.children())
        tensors = []
        for layer in layers:
            tensors += [layer.conv.weight, layer.conv.bias]
            if hasattr(layer, "bn"):
                bn = layer.bn.bn
                tensors += [bn.weight, bn.bias, bn.running_mean, bn.running_var]
        key = (kind, split, str(device), _fold_scale(), project_known)
        stamp = tensor_stamp(tensors)
        if key == self.key and stamp_matches(self.stamp, stamp):
            return self.chain
        fold_scale = key[3]
        folded = [mlp_chain.fold(layer.conv, layer.bn.bn if hasattr(layer, "bn") else None, fold_scale) for layer in layers]
        ws = [W for W, _, _ in folded]
        shifts = [t for _, _, t in folded]
        scales = None if fold_scale else [s for _, s, _ in folded]
        self.proj = None
        if project_known:
            # ws[0] is (c_out0, c_known + c_skip) with the BN scale already folded in: W0k -> projection, W0s stays
            assert scales is None, "project_known needs the BN scale folded into the weights"
            W0 = ws[0]
            c1, c_known = W0.shape[0], split
            self.proj = mlp_chain.Chain(mlp_chain.ROWS, 0, [W0[:, :c_known]], [torch.zeros(c1)], linear_last=True, device=device)
            ws[0] = torch.cat([torch.eye(c1), W0[:, c_known:]], dim=1)
            split = c1
        self.chain = mlp_chain.Chain(kind, split, ws, shifts, scales, device=device)
        self.key, self.stamp = key, stamp
        return self.chain


def _attach_pm(t, pm):
    """remember the point-major twin the kernel wrote next to `t`; valid while `t` is not modified in place"""
    t._prb_pm = (pm, t._version)
    return t


def _point_major(t):
    """(B,C,N) -> (B,N,C): the twin written by the producing kernel if it is still valid, else a transpose kernel"""
    twin = getattr(t, "_prb_pm", None)
    if twin is not None and twin[1] == t._version and twin[0].shape == (t.size(0), t.size(2), t.size(1)) and twin[0].device == t.device:
        return twin[0]
    return pointnet2_utils.transpose_bcn_to_bnc(t.contiguous())


def rows_mlp(fused: "_FusedMLP", mlp: nn.Sequential, a: torch.Tensor, b: torch.Tensor = None, tag="rows_mlp"):
    """SharedMLP over point rows on the tensor-core chain: `a` (rows, c_a) and optionally `b` (rows, c_b) are 2-D views with
    unit column stride and any row pitch (e.g. column slices of the pooled RoI rows); layer 0 reads [a | b] without the
    concatenation ever existing in memory.  Returns (rows, c_out) row-major.  Replaces pt_utils.SharedMLP on (B,C,N,1)
    tensors (lib/net/rcnn_net.py:58-66,171-175)."""
    chain = fused.get(mlp, *mlp_chain.rows_layout(a.size(1), 0 if b is None else b.size(1)), a.device)
    out = chain.rows(a, b, tag)
    return out if out.size(1) == chain.c_out[-1] else out[:, :chain.c_out[-1]]


def _fold_scale():
    """config.fold_scale=False keeps the BN scale as a separate epilogue multiply (y = relu(s * (W x) + t))"""
    return config.get("fold_scale")


def _fused_enabled():
    return not config.get("disable_fused")


def _needs_graph(module, *tensors):
    if not torch.is_grad_enabled():
        return False
    if any(t is not None and t.requires_grad for t in tensors):
        return True
    return any(p.requires_grad for p in module.parameters())


class _PointnetSAModuleBase(nn.Module):
    def __init__(self):
        super().__init__()
        self.npoint = None
        self.groupers = None
        self.mlps = None
        self.pool_method = 'max_pool'
        self._fused = None

    def _apply(self, fn, *args, **kwargs):
        # .to() / .half() / .float() / .cuda() replace parameter storage without bumping tensor versions: drop the packed images
        self._fused = None
        return super()._apply(fn, *args, **kwargs)

    def invalidate_fused(self):
        """call after editing weights through `.data` (EMA, weight averaging): such writes do not bump the version counters the
        packed-weight cache keys on"""
        self._fused = None

    # ------------------------------------------------------------------ fused (tensor-core) path
    def _can_fuse(self, xyz, features, new_xyz):
        if not _fused_enabled() or not xyz.is_cuda:
            return False
        if _needs_graph(self, xyz, features, new_xyz):
            return False
        if xyz.dtype != torch.float32 or (features is not None and features.dtype != torch.float32):
            return False
        return grouping_ok(self, xyz.size(1)) and all(_FusedMLP.supported(mlp) for mlp in self.mlps)

    def fused_geometry(self, xyz, new_xyz=None):
        """sampling + neighbour search of the fused path (depends on coordinates only, so a caller may run it on a side
        stream, ahead of the feature MLPs): returns (ret_xyz, centres (B,npoint,3), [idx per scale], [nsample per scale])"""
        B, N, _ = xyz.shape
        dev = xyz.device
        if self.npoint is None:
            centres = torch.zeros((B, 1, 3), dtype=torch.float32, device=dev)   # GroupAll: no centre subtraction
            ar = torch.arange(N, dtype=torch.int32, device=dev).view(1, 1, N).expand(B, 1, N).contiguous()
            return None, centres, [ar for _ in self.groupers], [N for _ in self.groupers]
        if new_xyz is None:
            _, new_xyz = pointnet2_utils.furthest_point_sample_xyz(xyz, self.npoint)
        centres = new_xyz.contiguous()
        if len(self.groupers) == 2:
            g0, g1 = self.groupers
            idxs = list(pointnet2_utils.ball_query_msg2((g0.radius, g1.radius), (g0.nsample, g1.nsample), xyz, centres))
        else:
            idxs = [pointnet2_utils.ball_query(g.radius, g.nsample, xyz, centres) for g in self.groupers]
        return new_xyz, centres, idxs, [g.nsample for g in self.groupers]

    def fused_mlp(self, xyz, features, centres, idxs, nss):
        """gather + SharedMLP + max-pool of every scale (one tensor-core kernel per scale) -> (B, sum C_out, npoint)"""
        B = xyz.size(0)
        dev = xyz.device
        npoint = centres.size(1)
        c_feat = 0 if features is None else features.size(1)
        feats_pm = _point_major(features) if features is not None else None
        if self._fused is None or len(self._fused) != len(self.mlps):
            self._fused = [_FusedMLP() for _ in self.mlps]
        chains = [f.get(mlp, mlp_chain.SA, c_feat, dev) for f, mlp in zip(self._fused, self.mlps)]
        c_total = sum(chain.c_out[-1] for chain in chains)
        out = torch.empty((B, c_total, npoint), dtype=torch.float32, device=dev)
        out_pm = torch.empty((B, npoint, c_total), dtype=torch.float32, device=dev)   # twin for the next gather
        off = 0
        for chain, idx, ns in zip(chains, idxs, nss):
            chain.sa(xyz, centres, feats_pm, idx, ns, out, out_pm, off)
            off += chain.c_out[-1]
        return _attach_pm(out, out_pm)

    def _forward_fused(self, xyz, features, new_xyz):
        xyz = xyz.contiguous()
        ret_xyz, centres, idxs, nss = self.fused_geometry(xyz, new_xyz)
        return ret_xyz, self.fused_mlp(xyz, features, centres, idxs, nss)

    # ------------------------------------------------------------------ training path (config.sa_train == "device")
    def _forward_train(self, xyz, features, new_xyz):
        """the fused path's sampling and neighbour search, then sa_train's autograd Function over all scales"""
        xyz = xyz.contiguous()
        ret_xyz, centres, idxs, nss = self.fused_geometry(xyz, new_xyz)
        features = sa_train.as_fp32(features)          # bfloat16 under autocast: the device path computes in fp32
        feats_pm = _point_major(features) if features is not None else None
        out, out_pm = sa_train.forward(self, xyz, features, feats_pm, centres, idxs, nss)
        return ret_xyz, _attach_pm(out, out_pm)

    # ------------------------------------------------------------------ reference-shaped path
    def forward(self, xyz: torch.Tensor, features: torch.Tensor = None, new_xyz=None) -> (torch.Tensor, torch.Tensor):
        """
        :param xyz: (B, N, 3) coordinates
        :param features: (B, C, N) descriptors (channel-major) or None
        :param new_xyz: optional externally chosen centres (B, npoint, 3)
        :return: new_xyz (B, npoint, 3), new_features (B, sum_k mlps[k][-1], npoint)
        """
        if self._can_fuse(xyz, features, new_xyz):
            return self._forward_fused(xyz, features, new_xyz)
        if (config.get("sa_train") == "device" and _needs_graph(self, xyz, features, new_xyz)
                and sa_train.supported(self, xyz, features, new_xyz) and sa_train.faster_on_device(self)):
            return self._forward_train(xyz, features, new_xyz)

        new_features_list = []
        if new_xyz is None and self.npoint is not None:
            xyz_flipped = xyz.transpose(1, 2).contiguous()
            new_xyz = pointnet2_utils.gather_operation(
                xyz_flipped, pointnet2_utils.furthest_point_sample(xyz, self.npoint)).transpose(1, 2).contiguous()
        for i in range(len(self.groupers)):
            new_features = self.groupers[i](xyz, new_xyz, features)      # (B, C, npoint, nsample)
            new_features = self.mlps[i](new_features)                    # (B, mlp[-1], npoint, nsample)
            if self.pool_method == 'max_pool':
                new_features = F.max_pool2d(new_features, kernel_size=[1, new_features.size(3)])
            elif self.pool_method == 'avg_pool':
                new_features = F.avg_pool2d(new_features, kernel_size=[1, new_features.size(3)])
            else:
                raise NotImplementedError
            new_features_list.append(new_features.squeeze(-1))           # (B, mlp[-1], npoint)
        return new_xyz, torch.cat(new_features_list, dim=1)


class PointnetSAModuleMSG(_PointnetSAModuleBase):
    """Pointnet set abstraction layer with multiscale grouping"""

    def __init__(self, *, npoint: int, radii: List[float], nsamples: List[int], mlps: List[List[int]], bn: bool = True,
                 use_xyz: bool = True, pool_method='max_pool', instance_norm=False):
        super().__init__()
        assert len(radii) == len(nsamples) == len(mlps)
        self.npoint = npoint
        self.groupers = nn.ModuleList()
        self.mlps = nn.ModuleList()
        for i in range(len(radii)):
            self.groupers.append(pointnet2_utils.QueryAndGroup(radii[i], nsamples[i], use_xyz=use_xyz)
                                 if npoint is not None else pointnet2_utils.GroupAll(use_xyz))
            mlp_spec = mlps[i]
            if use_xyz:
                mlp_spec[0] += 3   # in place, like the reference (pointnet2_modules.py:88-89): callers rely on it
            self.mlps.append(pt_utils.SharedMLP(mlp_spec, bn=bn, instance_norm=instance_norm))
        self.pool_method = pool_method


class PointnetSAModule(PointnetSAModuleMSG):
    """Pointnet set abstraction layer"""

    def __init__(self, *, mlp: List[int], npoint: int = None, radius: float = None, nsample: int = None, bn: bool = True,
                 use_xyz: bool = True, pool_method='max_pool', instance_norm=False):
        super().__init__(mlps=[mlp], npoint=npoint, radii=[radius], nsamples=[nsample], bn=bn, use_xyz=use_xyz,
                         pool_method=pool_method, instance_norm=instance_norm)


class PointnetFPModule(nn.Module):
    r"""Propagates the features of one set to another"""

    def __init__(self, *, mlp: List[int], bn: bool = True):
        super().__init__()
        self.mlp = pt_utils.SharedMLP(mlp, bn=bn)
        self._fused = None
        self.emit_point_major = True   # also write a (B,n,C) twin for the next FP level (skips its transpose kernel)
        self.project_known = True      # split layer 0 by linearity when it narrows the gathered rows (see _FusedMLP.get)

    def _apply(self, fn, *args, **kwargs):
        self._fused = None             # see _PointnetSAModuleBase._apply
        return super()._apply(fn, *args, **kwargs)

    def invalidate_fused(self):
        self._fused = None

    def _can_fuse(self, unknown, known, unknow_feats, known_feats):
        if not _fused_enabled() or known is None or not unknown.is_cuda:
            return False
        if _needs_graph(self, unknown, known, unknow_feats, known_feats):
            return False
        if known_feats.dtype != torch.float32 or (unknow_feats is not None and unknow_feats.dtype != torch.float32):
            return False
        return _FusedMLP.supported(self.mlp)

    def fused_geometry(self, unknown, known):
        """3-NN search + inverse-distance weights (coordinates only) -> (idx (B,n,3) int32, weight (B,n,3))"""
        _, idx, weight = pointnet2_utils.three_nn_weights(unknown.contiguous(), known.contiguous())
        return idx, weight

    def fused_mlp(self, n, idx, weight, unknow_feats, known_feats):
        dev = known_feats.device
        B, c_known, m = known_feats.shape
        known_pm = _point_major(known_feats)
        skip = unknow_feats.contiguous() if unknow_feats is not None else None
        if self._fused is None:
            self._fused = _FusedMLP()
        c1 = list(self.mlp.children())[0].conv.out_channels
        # interpolation commutes with the (linear) first layer: project the m known points once instead of gathering
        # c_known floats for each of the 3 neighbours of every one of the n >= m unknown points
        # only worth it at the finest level: at the coarse ones the extra launch costs more than the narrower gather saves
        project = (self.project_known and config.get("fp_project") and _fold_scale() and c1 < c_known and n >= m
                   and B * n >= config.get("fp_project_min_rows"))
        chain = self._fused.get(self.mlp, mlp_chain.FP, c_known, dev, project_known=project)
        if project:
            proj = self._fused.proj.rows(known_pm.view(B * m, c_known), tag="fp_mlp", detail="%d proj [%d]+[%d]" % (B * m, c_known, c1))
            known_pm = proj[:, :c1].contiguous().view(B, m, c1)
        c_last = chain.c_out[-1]
        out = torch.empty((B, c_last, n), dtype=torch.float32, device=dev)
        out_pm = torch.empty((B, n, c_last), dtype=torch.float32, device=dev) if self.emit_point_major else None
        chain.fp(known_pm, idx, weight, skip, out, out_pm)
        return _attach_pm(out, out_pm) if out_pm is not None else out

    def _forward_fused(self, unknown, known, unknow_feats, known_feats):
        idx, weight = self.fused_geometry(unknown, known)
        return self.fused_mlp(unknown.size(1), idx, weight, unknow_feats, known_feats)

    def _forward_train(self, unknown, known, unknow_feats, known_feats):
        """the fused path's 3-NN, then fp_train's autograd Function"""
        idx, weight = self.fused_geometry(unknown, known)
        known_feats = sa_train.as_fp32(known_feats)    # bfloat16 under autocast: the device path computes in fp32
        skip = sa_train.as_fp32(unknow_feats.contiguous()) if unknow_feats is not None else None
        out, out_pm = fp_train.forward(self, idx, weight, _point_major(known_feats), known_feats, skip, self.emit_point_major)
        return _attach_pm(out, out_pm) if out_pm is not None else out

    def forward(self, unknown: torch.Tensor, known: torch.Tensor, unknow_feats: torch.Tensor,
                known_feats: torch.Tensor) -> torch.Tensor:
        """
        :param unknown: (B, n, 3) positions to propagate to
        :param known: (B, m, 3) positions to propagate from (None: broadcast known_feats)
        :param unknow_feats: (B, C1, n) skip features or None
        :param known_feats: (B, C2, m)
        :return: (B, mlp[-1], n)
        """
        if self._can_fuse(unknown, known, unknow_feats, known_feats):
            return self._forward_fused(unknown, known, unknow_feats, known_feats)
        if (config.get("fp_train") == "device" and _needs_graph(self, unknown, known, unknow_feats, known_feats)
                and fp_train.supported(self, unknown, known, unknow_feats, known_feats)
                and fp_train.faster_on_device(self, known_feats.size(1), 0 if unknow_feats is None else unknow_feats.size(1))):
            return self._forward_train(unknown, known, unknow_feats, known_feats)

        if known is not None:
            dist, idx = pointnet2_utils.three_nn(unknown, known)
            dist_recip = 1.0 / (dist + 1e-8)
            norm = torch.sum(dist_recip, dim=2, keepdim=True)
            weight = dist_recip / norm
            interpolated_feats = pointnet2_utils.three_interpolate(known_feats, idx, weight)
        else:
            interpolated_feats = known_feats.expand(*known_feats.size()[0:2], unknown.size(1))
        if unknow_feats is not None:
            new_features = torch.cat([interpolated_feats, unknow_feats], dim=1)   # (B, C2 + C1, n)
        else:
            new_features = interpolated_feats
        new_features = self.mlp(new_features.unsqueeze(-1))
        return new_features.squeeze(-1)
