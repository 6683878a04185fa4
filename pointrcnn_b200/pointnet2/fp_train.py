"""The device training path of a PointnetFPModule's three_interpolate + cat(skip) + SharedMLP (csrc/sa_train.cu,
prb_fp_train_*), taken when the switch `config.fp_train` is "device", `supported` holds and the dispatch rule
(`faster_on_device`) selects the level; everything else keeps the op-by-op torch path.

One autograd Function per module.  Its inputs are the known features, the skip features and every conv weight / bias and
BN weight / bias, so autograd accumulates their .grad as for the torch path; the BN running statistics and
num_batches_tracked are updated in place by the forward, as BatchNorm2d does in training mode.  The interpolation taps
come from three_nn_weights (the fused path's 3-NN).  Saved for backward: the taps, the point-major known features, the
skip features, the pre-activations Z of every layer and the per-channel statistics.
Layer 0 runs projected: the m known points go through the interpolated columns of layer 0 first, then the result is
interpolated (n = 4 m at every RPN level, so this removes three quarters of that part of layer 0).
Precision: TF32 tensor-core GEMMs with fp32 accumulation, the BN statistics summed in float64.  Under torch.autocast
it computes in fp32 all the same (see sa_train.py): bfloat16 known / skip features are converted at entry, the outputs
are fp32 and each input's gradient comes back in that input's dtype.
"""
import ctypes

import torch
from torch.autograd.function import once_differentiable

from .. import _cabi as C
from . import sa_train

MAX_IN = 2048          # widest layer-0 input (interpolated + skip channels)

# Dispatch rule: (c_known, c_skip, widths) of the levels the device path is faster on, forward + backward.  Measured on an
# H100 SXM (80 GB, 700 W) with scripts/bench_fp_train.py at B = 16 (see INTEGRATION.md); every other level keeps the
# torch path.
FAST_LEVELS = {
    (256, 1, (128, 128)),       # RPN FP0: 5.7-5.8 ms device vs 6.8-7.0 ms torch
    (1024, 512, (512, 512)),    # RPN FP3: 1.7-2.6 ms device vs 2.7-4.6 ms torch
}
# RPN FP1 (5.2-5.3 ms device vs 4.1-4.7 ms torch) and FP2 (4.3-4.4 vs 2.9-3.5 ms) lose in their backward GEMMs.


def faster_on_device(module, c_known, c_skip):
    """the fixed shape rule of the dispatch (see FAST_LEVELS)"""
    return (c_known, c_skip, tuple(layer.conv.out_channels for layer in module.mlp.children())) in FAST_LEVELS


def supported(module, unknown, known, unknow_feats, known_feats):
    """the whole rule but the switch, the need for an autograd graph and the shape rule: known points given, fp32 CUDA
    coordinates without grad, fp32 or bfloat16 CUDA features, contiguous fp32 CUDA parameters (sa_train._params_ok), and a
    SharedMLP as sa_train._mlp_ok describes for c_known + c_skip (at most MAX_IN) input channels"""
    if known is None or known_feats is None:
        return False
    for t in (unknown, known):
        if not t.is_cuda or t.dtype != torch.float32 or t.requires_grad:
            return False
    for t in (known_feats, unknow_feats):
        if t is not None and (not t.is_cuda or t.dtype not in sa_train.FEATURE_DTYPES):
            return False
    if not sa_train._params_ok(module.mlp):
        return False
    c_in = known_feats.size(1) + (0 if unknow_feats is None else unknow_feats.size(1))
    return c_in <= MAX_IN and sa_train._mlp_ok(module.mlp, c_in)


class _FPTrain(torch.autograd.Function):
    """(known_feats, skip, *params) -> (out (B, C_last, n), out_pm (B, n, C_last) or None) of one FP module"""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, scale, geom, known_pm, known_feats, skip, *params):
        idx, weight, emit_pm = geom
        L = C.lib()
        B, n, _ = idx.shape
        m, c_known = known_pm.size(1), known_pm.size(2)
        c_skip = 0 if skip is None else skip.size(1)
        dev = known_pm.device
        rows = B * n
        sa_train._check_batch(scale, [B, scale.c_out[0], n, 1])
        d = scale.desc(c_known + c_skip, params)
        c_last = scale.c_out[-1]
        out = torch.empty((B, c_last, n), dtype=torch.float32, device=dev)
        out_pm = torch.empty((B, n, c_last), dtype=torch.float32, device=dev) if emit_pm else None
        z = [torch.empty((rows, c), dtype=torch.float32, device=dev) for c in scale.c_out]
        stats = torch.empty((len(scale.c_out), sa_train.STAT_ROWS, sa_train.MAX_WIDTH), dtype=torch.float32, device=dev)
        with torch.cuda.device(dev):
            ws = torch.empty(L.prb_fp_train_workspace_bytes(B, n, m, c_known, c_skip, ctypes.byref(d), 0), dtype=torch.uint8, device=dev)
            C.check(L.prb_fp_train_forward(ctypes.byref(d), B, n, m, c_known, c_skip, C.ptr(idx), C.ptr(weight), C.ptr(known_pm), C.ptr(skip),
                                           sa_train._ptrs(z), C.ptr(stats), C.ptr(out), C.ptr(out_pm), C.ptr(ws), ws.numel(), C.stream()),
                    "fp_train_forward")
        ctx.scale, ctx.desc = scale, d
        ctx.save_for_backward(idx, weight, known_pm, skip, *params, *z, stats)
        if out_pm is not None:
            ctx.mark_non_differentiable(out_pm)
        return out, out_pm

    @staticmethod
    @once_differentiable
    def backward(ctx, g_out, g_pm):
        t = ctx.saved_tensors
        idx, weight, known_pm, skip = t[:4]
        params = t[4:16]
        nl = len(ctx.scale.c_out)
        z, stats = t[16:16 + nl], t[16 + nl]
        if g_out is None:
            return (None,) * (5 + len(params))
        L = C.lib()
        B, n, _ = idx.shape
        m, c_known = known_pm.size(1), known_pm.size(2)
        c_skip = 0 if skip is None else skip.size(1)
        dev = known_pm.device
        g_out = g_out.float().contiguous()
        g_known = torch.empty((B, c_known, m), dtype=torch.float32, device=dev) if ctx.needs_input_grad[3] else None
        g_skip = torch.empty((B, c_skip, n), dtype=torch.float32, device=dev) if ctx.needs_input_grad[4] and c_skip > 0 else None
        bufs = sa_train._grad_buffers(params, nl)
        d = ctx.desc
        with torch.cuda.device(dev):
            ws = torch.empty(L.prb_fp_train_workspace_bytes(B, n, m, c_known, c_skip, ctypes.byref(d), 1), dtype=torch.uint8, device=dev)
            C.check(L.prb_fp_train_backward(ctypes.byref(d), B, n, m, c_known, c_skip, C.ptr(idx), C.ptr(weight), C.ptr(known_pm), C.ptr(skip),
                                            sa_train._ptrs(z), C.ptr(stats), C.ptr(g_out), *[sa_train._ptrs(b) for b in bufs],
                                            C.ptr(g_known), C.ptr(g_skip), C.ptr(ws), ws.numel(), C.stream()), "fp_train_backward")
        return (None, None, None, g_known, g_skip) + tuple(sa_train._slot_grads(bufs, ctx.needs_input_grad[5:]))


def forward(module, idx, weight, known_pm, known_feats, skip, emit_pm):
    """the features (B, C_last, n) of FP module `module` through the device path, and their point-major twin (None unless
    emit_pm).  idx / weight (B, n, 3): three_nn_weights' taps; known_pm (B, m, c_known): known_feats point-major;
    skip (B, c_skip, n) contiguous or None; the features fp32 (sa_train.as_fp32)"""
    C.require_cuda(idx, weight, known_pm, known_feats, skip)
    scale = sa_train._Scale(module.mlp)
    out, out_pm = _FPTrain.apply(scale, (idx, weight, emit_pm), known_pm.detach(), known_feats, skip, *scale.params())
    sa_train._bump_running_stats(scale)
    return out, out_pm


def decisions(out):
    """the device's saved state behind `out`: `z` (list of (rows, C_l)) and `stats` (layers, 4, 512)"""
    fn = out.grad_fn
    t = fn.saved_tensors
    nl = len(fn.scale.c_out)
    return dict(z=list(t[16:16 + nl]), stats=t[16 + nl])
