"""The device training path of an SA module's grouped SharedMLP + max-pool (csrc/sa_train.cu), taken when the switch
`config.sa_train` is "device" and `supported` holds; everything else keeps the op-by-op torch path.

One autograd Function per module covers all its scales.  Its inputs are the features and every conv weight / bias and BN
weight / bias, so autograd accumulates their .grad as for the torch path; the BN running statistics and
num_batches_tracked are updated in place by the forward, as BatchNorm2d does in training mode.  Saved for backward: the
pre-activations Z of every layer, the per-channel statistics and the sample each pooled output took (`decisions`).
Precision: TF32 tensor-core GEMMs with fp32 accumulation, the BN statistics summed in float64.
Under torch.use_deterministic_algorithms(True) (warn_only too) the backward takes prb_sa_train_backward_det, whose feature
gradient is summed per point in a fixed order instead of scattered with float atomics; every other result is the same.
Under torch.autocast the Function still computes in fp32: bfloat16 features are converted to fp32 before the point-major
copy (fp32), the Function's forward casts its floating inputs to fp32 and runs with autocast off, and each input's
gradient comes back in that input's dtype.  The outputs are fp32.
"""
import ctypes

import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from .. import _cabi as C
from . import pointnet2_modules as pm     # imports this module in turn: read its attributes at call time only

MAX_WIDTH = 512
# Dispatch rule: the device path is taken only for modules whose every layer is at most this wide.  Measured on an H100
# SXM (80 GB, 700 W) at the bench shapes (scripts/bench_sa_train.py): forward + backward of RPN SA1 (widths 16..64,
# 2M grouped rows) is faster than the torch path; the wider levels (RPN SA2-SA4, RCNN SA1-SA3, 96..512 channels) are
# slower, so they keep the torch path.
FAST_MAX_WIDTH = 64
STAT_ROWS = 4          # mean, invstd, a, b (y = relu(a * z + b)) per channel, MAX_WIDTH apart


def _mlp_ok(mlp, c_in):
    """a SharedMLP as pointnet2_modules.read_mlp reads it, of Conv2d blocks, reading c_in channels, at most MAX_WIDTH wide,
    each with [BatchNorm2d in training mode with tracked statistics | conv bias], all with or all without BN (one eps /
    momentum: the descriptor holds one)"""
    blocks = pm.read_mlp(mlp)
    if blocks is None or blocks[0][0].in_channels != c_in:
        return False
    kinds = set()
    for conv, bn, _ in blocks:
        if not isinstance(conv, nn.Conv2d) or conv.out_channels > MAX_WIDTH:
            return False
        if bn is not None and (not isinstance(bn, nn.BatchNorm2d) or not bn.training or not bn.track_running_stats
                               or bn.momentum is None or not bn.affine or conv.bias is not None):
            return False
        kinds.add(None if bn is None else (float(bn.eps), float(bn.momentum)))
    return len(kinds) == 1


def layout_ok(module, c_feat, n_points):
    """the module half of the rule: pointnet2_modules.grouping_ok, and every SharedMLP as _mlp_ok describes for 3 + c_feat
    input channels"""
    return pm.grouping_ok(module, n_points) and all(_mlp_ok(mlp, 3 + c_feat) for mlp in module.mlps)


def faster_on_device(module):
    """the fixed shape rule of the dispatch (see FAST_MAX_WIDTH)"""
    return all(layer.conv.out_channels <= FAST_MAX_WIDTH for mlp in module.mlps for layer in mlp.children())


def _params_ok(module):
    """every floating parameter and buffer of `module` is contiguous fp32 CUDA: the kernels read the parameters and write
    their gradients as dense (c_out, c_in) rows"""
    return all(t.is_cuda and t.dtype == torch.float32 and t.is_contiguous()
               for t in list(module.parameters()) + list(module.buffers()) if t.is_floating_point())


FEATURE_DTYPES = (torch.float32, torch.bfloat16)     # bfloat16: the features of autocast training, converted at entry


def as_fp32(t):
    """`t` itself when None or float32, else its float32 copy (autograd returns the gradient in t's dtype)"""
    return t if t is None or t.dtype == torch.float32 else t.float()


def supported(module, xyz, features, new_xyz):
    """the whole rule but the switch and the need for an autograd graph (the caller checks those): fp32 CUDA coordinates
    without grad, fp32 or bfloat16 CUDA features, contiguous fp32 CUDA parameters, and layout_ok"""
    if not xyz.is_cuda or xyz.dtype != torch.float32 or xyz.requires_grad:
        return False
    if new_xyz is not None and new_xyz.requires_grad:
        return False
    if features is not None and (not features.is_cuda or features.dtype not in FEATURE_DTYPES):
        return False
    if not _params_ok(module.mlps):
        return False
    return layout_ok(module, 0 if features is None else features.size(1), xyz.size(1))


class _Scale:
    """the layer structure of one scale, and its descriptor for the current parameter storage"""

    def __init__(self, mlp):
        self.layers = list(mlp.children())
        self.bn = hasattr(self.layers[0], "bn")
        self.c_out = [layer.conv.out_channels for layer in self.layers]

    def params(self):
        """weight, bias, gamma, beta per layer (None where absent), in the 12 slots of three layers: the Function's
        differentiable inputs"""
        out = []
        for layer in self.layers:
            bn = layer.bn.bn if self.bn else None
            out += [layer.conv.weight, layer.conv.bias, bn.weight if bn is not None else None, bn.bias if bn is not None else None]
        return out + [None] * (12 - len(out))

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


def _check_batch(scale, size):
    """BatchNorm2d's refusal of a training batch with one value per channel; size: (B, C, H, W) of layer 0's output"""
    if scale.bn and size[0] * size[2] * size[3] == 1:
        raise ValueError("Expected more than 1 value per channel when training, got input size %s" % (torch.Size(size),))


def _ptrs(ts):
    """the C ABI's per-layer pointer array of up to three tensors (None where absent)"""
    return (ctypes.c_void_p * 3)(*[t.data_ptr() if t is not None else None for t in ts])


def _grad_buffers(params, nl):
    """[weight, bias, gamma, beta] gradient buffers of one scale's nl layers, each a list of uninitialised tensors shaped as
    the parameter slots of `params` (None where a slot is empty)"""
    return [[torch.empty_like(t) if t is not None else None for t in params[j::4][:nl]] for j in range(4)]


def _slot_grads(bufs, needs):
    """the gradients of one scale's 12 parameter slots from its _grad_buffers, None where `needs` (the scale's entries of
    ctx.needs_input_grad) is False"""
    nl = len(bufs[0])
    grads = [bufs[j][l] for l in range(nl) for j in range(4)] + [None] * (12 - 4 * nl)
    return [g if need else None for g, need in zip(grads, needs)]


def _bump_running_stats(scale):
    """the kernel wrote the running statistics in place: bump their versions as torch's in-place update would, so caches
    keyed on them (the eval chain's folded weights) see the change"""
    if scale.bn:
        for layer in scale.layers:
            bn = layer.bn.bn
            torch.autograd.graph.increment_version([bn.running_mean, bn.running_var, bn.num_batches_tracked])


class _SATrain(torch.autograd.Function):
    """(features, *params) -> (out (B, sum C_last, npoint), out_pm (B, npoint, sum C_last)) of one SA module"""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
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
                _check_batch(s, [B, s.c_out[0], npoint, ns])
                p = params[k * 12:(k + 1) * 12]
                d = s.desc(3 + c_feat, p)
                z = [torch.empty((rows, c), dtype=torch.float32, device=dev) for c in s.c_out]
                stats = torch.empty((len(s.c_out), STAT_ROWS, MAX_WIDTH), dtype=torch.float32, device=dev)
                chosen = torch.empty((B * npoint, s.c_out[-1]), dtype=torch.uint8, device=dev)
                ws = torch.empty(L.prb_sa_train_workspace_bytes(B, npoint, ns, c_feat, ctypes.byref(d), 0), dtype=torch.uint8, device=dev)
                C.check(L.prb_sa_train_forward(ctypes.byref(d), B, N, npoint, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm),
                                               C.ptr(idx), _ptrs(z), C.ptr(stats), C.ptr(chosen), C.ptr(out), C.ptr(out_pm), c_total, off,
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
        g_feats = None
        if g_out is None:
            return (None,) * (4 + len(params))
        L = C.lib()
        B, N, _ = xyz.shape
        npoint = centres.size(1)
        c_feat = ctx.c_feat
        dev = xyz.device
        g_out = g_out.float().contiguous()
        c_total = g_out.size(1)
        ordered = torch.are_deterministic_algorithms_enabled()
        if ctx.needs_input_grad[3] and c_feat > 0:
            # ordered: each scale WRITES its sum, so scales after the first go through a buffer and are added in scale order
            g_feats = (torch.empty if ordered else torch.zeros)((B, c_feat, N), dtype=torch.float32, device=dev)
        grads, off = [], 0
        with torch.cuda.device(dev):
            for k, (s, idx, ns, d) in enumerate(zip(ctx.scales, idxs, ctx.nss, ctx.descs)):
                nl = len(s.c_out)
                z, stats, chosen = rest[:nl], rest[nl], rest[nl + 1]
                rest = rest[nl + 2:]
                bufs = _grad_buffers(params[k * 12:(k + 1) * 12], nl)
                if ordered:
                    entry, name = L.prb_sa_train_backward_det, "sa_train_backward_det"
                    wsb = L.prb_sa_train_det_workspace_bytes(B, N, npoint, ns, c_feat, ctypes.byref(d))
                    g_k = g_feats if k == 0 or g_feats is None else torch.empty_like(g_feats)
                else:
                    entry, name = L.prb_sa_train_backward, "sa_train_backward"
                    wsb = L.prb_sa_train_workspace_bytes(B, npoint, ns, c_feat, ctypes.byref(d), 1)
                    g_k = g_feats
                ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
                C.check(entry(ctypes.byref(d), B, N, npoint, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm), C.ptr(idx), _ptrs(z),
                              C.ptr(stats), C.ptr(chosen), C.ptr(g_out), c_total, off, *[_ptrs(b) for b in bufs], C.ptr(g_k), C.ptr(ws),
                              ws.numel(), C.stream()), name)
                if g_k is not g_feats:
                    g_feats.add_(g_k)
                grads += _slot_grads(bufs, ctx.needs_input_grad[4 + k * 12:4 + (k + 1) * 12])
                off += s.c_out[-1]
        return (None, None, None, g_feats) + tuple(grads)


def forward(module, xyz, features, feats_pm, centres, idxs, nss):
    """the pooled features (B, sum C_last, npoint) of `module` through the device path, and their point-major twin.
    features / feats_pm: fp32 (as_fp32)"""
    C.require_cuda(xyz, centres, features, *idxs)
    scales = [_Scale(mlp) for mlp in module.mlps]
    params = [p for s in scales for p in s.params()]
    out, out_pm = _SATrain.apply(scales, (xyz, centres, idxs, nss), feats_pm, features, *params)
    for s in scales:
        _bump_running_stats(s)
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
