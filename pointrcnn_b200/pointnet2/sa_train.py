"""The device training path of an SA module's grouped SharedMLP + max-pool (csrc/sa_train.cu), taken when the switch
`config.sa_train` is "device" and `supported` holds; everything else keeps the op-by-op torch path.

One autograd Function per module covers all its scales.  Its inputs are the features and every conv weight / bias and BN
weight / bias, so autograd accumulates their .grad as for the torch path; the BN running statistics and
num_batches_tracked are updated in place by the forward, as BatchNorm2d does in training mode.  Saved for backward: the
pre-activations Z of every layer, the per-channel statistics and the sample each pooled output took (`decisions`).
Precision: TF32 tensor-core GEMMs with fp32 accumulation, the BN statistics summed in float64.
"""
import ctypes

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from .. import _cabi as C
from . import pointnet2_utils

MAX_WIDTH = 512
# Dispatch rule: the device path is taken only for modules whose every layer is at most this wide.  Measured on an H100
# SXM (80 GB, 700 W) at the bench shapes (scripts/bench_sa_train.py): forward + backward of RPN SA1 (widths 16..64,
# 2M grouped rows) is faster than the torch path; the wider levels (RPN SA2-SA4, RCNN SA1-SA3, 96..512 channels) are
# slower, so they keep the torch path.
FAST_MAX_WIDTH = 64
STAT_ROWS = 4          # mean, invstd, a, b (y = relu(a * z + b)) per channel, MAX_WIDTH apart


def _mlp_ok(mlp, c_in):
    """1-3 layers of 1x1 Conv2d + [BatchNorm2d in training mode with tracked statistics | conv bias] + ReLU, at most
    MAX_WIDTH wide, all with or all without BN (one eps / momentum: the descriptor holds one)"""
    layers = list(mlp.children())
    if not 1 <= len(layers) <= 3:
        return False
    kinds = set()
    for layer in layers:
        names = [k for k, _ in layer.named_children()]
        if names not in (["conv", "bn", "activation"], ["conv", "activation"]) or not isinstance(layer.activation, nn.ReLU):
            return False
        conv = layer.conv
        if (not isinstance(conv, nn.Conv2d) or tuple(conv.kernel_size) != (1, 1) or tuple(conv.stride) != (1, 1)
                or tuple(conv.padding) != (0, 0) or tuple(conv.dilation) != (1, 1) or conv.groups != 1
                or conv.in_channels != c_in or conv.out_channels > MAX_WIDTH):
            return False
        if "bn" in names:
            bn = layer.bn.bn
            if (not isinstance(bn, nn.BatchNorm2d) or not bn.training or not bn.track_running_stats or bn.momentum is None
                    or not bn.affine or conv.bias is not None):
                return False
            kinds.add((float(bn.eps), float(bn.momentum)))
        else:
            kinds.add(None)
        c_in = conv.out_channels
    return len(kinds) == 1


def _nsample_ok(ns):
    return 4 <= ns <= 128 and ns & (ns - 1) == 0


def layout_ok(module, c_feat, n_points):
    """the module half of the rule: max-pool, QueryAndGroup / GroupAll with use_xyz and a power-of-two sample count in
    4..128 (GroupAll: the n_points of the input), and every SharedMLP as _mlp_ok describes for 3 + c_feat input channels"""
    if module.pool_method != "max_pool":
        return False
    for g, mlp in zip(module.groupers, module.mlps):
        if isinstance(g, pointnet2_utils.QueryAndGroup):
            if not g.use_xyz or not _nsample_ok(g.nsample):
                return False
        elif isinstance(g, pointnet2_utils.GroupAll):
            if not g.use_xyz or not _nsample_ok(n_points):
                return False
        else:
            return False
        if not _mlp_ok(mlp, 3 + c_feat):
            return False
    return True


def faster_on_device(module):
    """the fixed shape rule of the dispatch (see FAST_MAX_WIDTH)"""
    return all(layer.conv.out_channels <= FAST_MAX_WIDTH for mlp in module.mlps for layer in mlp.children())


def supported(module, xyz, features, new_xyz):
    """the whole rule but the switch and the need for an autograd graph (the caller checks those): fp32 CUDA inputs and
    contiguous fp32 CUDA parameters, coordinates without grad, and layout_ok"""
    if not xyz.is_cuda or xyz.dtype != torch.float32 or xyz.requires_grad:
        return False
    if new_xyz is not None and new_xyz.requires_grad:
        return False
    if features is not None and (not features.is_cuda or features.dtype != torch.float32):
        return False
    # the kernels read the parameters and write their gradients as dense (c_out, c_in) rows
    if any(not t.is_cuda or t.dtype != torch.float32 or not t.is_contiguous()
           for m in module.mlps for t in list(m.parameters()) + list(m.buffers()) if t.is_floating_point()):
        return False
    return layout_ok(module, 0 if features is None else features.size(1), xyz.size(1))


class _Scale:
    """the layer structure of one scale, and its descriptor for the current parameter storage"""

    def __init__(self, mlp):
        self.layers = list(mlp.children())
        self.bn = hasattr(self.layers[0], "bn")
        self.c_out = [layer.conv.out_channels for layer in self.layers]

    def params(self):
        """weight, bias, gamma, beta per layer (None where absent): the Function's differentiable inputs"""
        out = []
        for layer in self.layers:
            bn = layer.bn.bn if self.bn else None
            out += [layer.conv.weight, layer.conv.bias, bn.weight if bn is not None else None, bn.bias if bn is not None else None]
        return out

    def desc(self, c_in, params):
        d = C.SATrainDesc()
        d.num_layers = len(self.layers)
        d.c_in = c_in
        d.bn = int(self.bn)
        for l, layer in enumerate(self.layers):
            d.c_out[l] = self.c_out[l]
            w, b, g, be = params[4 * l:4 * l + 4]
            d.weight[l] = w.data_ptr()
            d.bias[l] = b.data_ptr() if b is not None else None
            if self.bn:
                bn = layer.bn.bn
                d.eps, d.momentum = float(bn.eps), float(bn.momentum)
                d.gamma[l], d.beta[l] = g.data_ptr(), be.data_ptr()
                d.running_mean[l], d.running_var[l] = bn.running_mean.data_ptr(), bn.running_var.data_ptr()
                d.num_batches_tracked[l] = bn.num_batches_tracked.data_ptr()
        return d


class _SATrain(torch.autograd.Function):
    """(features, *params) -> (out (B, sum C_last, npoint), out_pm (B, npoint, sum C_last)) of one SA module"""

    @staticmethod
    def forward(ctx, scales, geom, feats_pm, features, *params):
        xyz, centres, idxs, nss = geom
        L = C.lib()
        B, N, _ = xyz.shape
        npoint = centres.size(1)
        c_feat = 0 if feats_pm is None else feats_pm.size(2)
        dev = xyz.device
        c_total = sum(s.c_out[-1] for s in scales)
        out = torch.empty((B, c_total, npoint), dtype=torch.float32, device=dev)
        out_pm = torch.empty((B, npoint, c_total), dtype=torch.float32, device=dev)
        saved, descs, off = [], [], 0
        with torch.cuda.device(dev):
            for k, (s, idx, ns) in enumerate(zip(scales, idxs, nss)):
                rows = B * npoint * ns
                if s.bn and rows == 1:
                    raise ValueError("Expected more than 1 value per channel when training, got input size %s"
                                     % (torch.Size([B, s.c_out[0], npoint, ns]),))
                p = params[k * 12:(k + 1) * 12]
                d = s.desc(3 + c_feat, p)
                z = [torch.empty((rows, c), dtype=torch.float32, device=dev) for c in s.c_out]
                stats = torch.empty((len(s.c_out), STAT_ROWS, MAX_WIDTH), dtype=torch.float32, device=dev)
                chosen = torch.empty((B * npoint, s.c_out[-1]), dtype=torch.uint8, device=dev)
                ws = torch.empty(L.prb_sa_train_workspace_bytes(B, npoint, ns, c_feat, ctypes.byref(d), 0), dtype=torch.uint8, device=dev)
                zp = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in z])
                C.check(L.prb_sa_train_forward(ctypes.byref(d), B, N, npoint, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm),
                                               C.ptr(idx), zp, C.ptr(stats), C.ptr(chosen), C.ptr(out), C.ptr(out_pm), c_total, off,
                                               C.ptr(ws), ws.numel(), C.stream()), "sa_train_forward")
                saved += z + [stats, chosen]
                descs.append(d)
                off += s.c_out[-1]
        ctx.scales, ctx.nss, ctx.descs, ctx.c_feat, ctx.n_idx = scales, nss, descs, c_feat, len(idxs)
        ctx.save_for_backward(xyz, centres, feats_pm, *idxs, *params, *saved)
        ctx.mark_non_differentiable(out_pm)
        return out, out_pm

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, g_pm):
        t = ctx.saved_tensors
        xyz, centres, feats_pm = t[:3]
        idxs = t[3:3 + ctx.n_idx]
        params = t[3 + ctx.n_idx:3 + ctx.n_idx + 12 * len(ctx.scales)]
        rest = list(t[3 + ctx.n_idx + 12 * len(ctx.scales):])
        grads = [None] * len(params)
        g_feats = None
        if g_out is None:
            return (None, None, None, None) + tuple(grads)
        L = C.lib()
        B, N, _ = xyz.shape
        npoint = centres.size(1)
        c_feat = ctx.c_feat
        dev = xyz.device
        g_out = g_out.contiguous()
        c_total = g_out.size(1)
        if ctx.needs_input_grad[3] and c_feat > 0:
            g_feats = torch.zeros((B, c_feat, N), dtype=torch.float32, device=dev)
        off = 0
        with torch.cuda.device(dev):
            for k, (s, idx, ns, d) in enumerate(zip(ctx.scales, idxs, ctx.nss, ctx.descs)):
                nl = len(s.c_out)
                z, stats, chosen = rest[:nl], rest[nl], rest[nl + 1]
                rest = rest[nl + 2:]
                p = params[k * 12:(k + 1) * 12]
                gw = [torch.empty_like(w) for w in p[0::4][:nl]]
                gb = [torch.empty_like(b) if b is not None else None for b in p[1::4][:nl]]
                gg = [torch.empty_like(g) if g is not None else None for g in p[2::4][:nl]]
                gbe = [torch.empty_like(b) if b is not None else None for b in p[3::4][:nl]]

                def arr(ts):
                    return (ctypes.c_void_p * 3)(*[x.data_ptr() if x is not None else None for x in ts])

                ws = torch.empty(L.prb_sa_train_workspace_bytes(B, npoint, ns, c_feat, ctypes.byref(d), 1), dtype=torch.uint8, device=dev)
                C.check(L.prb_sa_train_backward(ctypes.byref(d), B, N, npoint, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm),
                                                C.ptr(idx), arr(z), C.ptr(stats), C.ptr(chosen), C.ptr(g_out), c_total, off, arr(gw),
                                                arr(gb), arr(gg), arr(gbe), C.ptr(g_feats), C.ptr(ws), ws.numel(), C.stream()),
                        "sa_train_backward")
                for l in range(nl):
                    grads[k * 12 + 4 * l:k * 12 + 4 * l + 4] = [gw[l], gb[l], gg[l], gbe[l]]
                off += s.c_out[-1]
        grads = [g if ctx.needs_input_grad[4 + i] else None for i, g in enumerate(grads)]
        return (None, None, None, g_feats) + tuple(grads)


def forward(module, xyz, features, feats_pm, centres, idxs, nss):
    """the pooled features (B, sum C_last, npoint) of `module` through the device path, and their point-major twin"""
    C.require_cuda(xyz, centres, features, *idxs)
    scales = [_Scale(mlp) for mlp in module.mlps]
    params = []
    for s in scales:
        p = s.params()
        params += p + [None] * (12 - len(p))
    out, out_pm = _SATrain.apply(scales, (xyz, centres, idxs, nss), feats_pm, features, *params)
    # the kernel wrote the running statistics in place: bump their versions as torch's in-place update would, so caches
    # keyed on them (the eval chain's folded weights) see the change
    for s in scales:
        if s.bn:
            for layer in s.layers:
                bn = layer.bn.bn
                torch.autograd.graph.increment_version([bn.running_mean, bn.running_var, bn.num_batches_tracked])
    return out, out_pm


def decisions(out):
    """the device's decisions behind `out` (the first output of the Function): per scale a dict with the pre-activations
    `z` (list of (rows, C_l)), `stats` (layers, 4, 512: mean, invstd, a, b with y = relu(a z + b)) and `chosen`
    ((B * npoint, C_last) uint8 sample index of every pooled output)"""
    fn = out.grad_fn
    t = fn.saved_tensors
    rest = list(t[3 + fn.n_idx + 12 * len(fn.scales):])
    res = []
    for s in fn.scales:
        nl = len(s.c_out)
        res.append(dict(z=rest[:nl], stats=rest[nl], chosen=rest[nl + 1]))
        rest = rest[nl + 2:]
    return res
