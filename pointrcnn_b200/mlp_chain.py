"""One MLP chain of the wgmma chain kernel (csrc/mlp_tc.cu): the eval-mode BatchNorm fold, the packed weight image with
its scale / shift and `prb_mlp_desc`, and the launches of the three entry points that run a chain.

The packer's (kind, split) fixes layer 0's K order, and that order must be the one the entry point gathers its rows in:

    prb_sa_group_mlp_max_ws   rows [rel xyz | feats]   kind SA,   split c_feat
    prb_fp_interp_mlp_ws      rows [interp | skip]     kind FP,   split c_known
    prb_mlp_rows2             rows [a | b], c_b > 0    kind FP,   split c_a
                              rows [a]                 kind ROWS, split 0

`prb_mlp_desc` does not record it: a chain packed for another order runs, and computes layer 0 over permuted columns.
So every launch method checks the chain's (kind, split, c_in) against its arguments and raises before launching.
"""
import contextlib
import ctypes

import numpy as np
import torch

from . import _cabi as C
from . import prof

SA, FP, ROWS = 0, 1, 2      # the packer's kinds


def rows_layout(c_a, c_b):
    """(kind, split) that prb_mlp_rows2 reads layer 0 in, for segments of c_a and c_b columns"""
    return (FP, c_a) if c_b else (ROWS, 0)


def fold(conv, bn, fold_scale=True, zero_bias=False):
    """Eval-mode BatchNorm (`bn`, or None) after a 1x1 convolution as y = scale * (W x) + shift.  Returns float32 CPU
    tensors (W (c_out, c_in), scale (c_out), shift (c_out)); the BN terms are computed on the module's device.
    fold_scale: W comes back multiplied by the scale, and scale is None.
    zero_bias: a conv without a bias adds scale * 0 to the shift, as a zero bias would.  The RPN heads fold this way,
    the SharedMLP chains do not; the two differ only where the shift is -0.0 (the sum makes it +0.0 for a positive
    scale) or the scale is not finite."""
    co = conv.out_channels
    W = conv.weight.detach().reshape(co, -1).float().cpu()
    b = conv.bias.detach().float().cpu() if conv.bias is not None else None
    if bn is None:
        return W, (None if fold_scale else torch.ones(co)), (b if b is not None else torch.zeros(co))
    inv = (bn.weight.detach().float() / torch.sqrt(bn.running_var.detach().float() + bn.eps)).cpu()
    sh = bn.bias.detach().float().cpu() - bn.running_mean.detach().float().cpu() * inv
    if b is not None or zero_bias:
        sh = sh + inv * (b if b is not None else torch.zeros(co))
    if fold_scale:
        return W * inv[:, None], None, sh
    return W, inv, sh


def _f32(x):
    """a float32 vector or matrix (numpy or torch) as a contiguous numpy array"""
    if torch.is_tensor(x):
        x = x.detach().cpu().numpy()
    if x.dtype != np.float32:
        raise TypeError("mlp_chain: expected float32, got %s" % x.dtype)
    return np.ascontiguousarray(x)


def _c_out_array(c_out):
    return (ctypes.c_int * 3)(*(list(c_out) + [0] * (3 - len(c_out))))


def pack_image(kind, split, weights):
    """The host image (float32 numpy) of the chain weights[l] (c_out[l], c_in[l]), packed as (kind, split)"""
    ws = [_f32(w) for w in weights]
    for l in range(1, len(ws)):
        if ws[l].shape[1] != ws[l - 1].shape[0]:
            raise ValueError("mlp_chain: layer %d takes %d inputs, layer %d gives %d" % (l, ws[l].shape[1], l - 1, ws[l - 1].shape[0]))
    L, c_in, co = len(ws), ws[0].shape[1], _c_out_array([w.shape[0] for w in ws])
    lib = C.lib()
    img = np.zeros(lib.prb_mlp_packed_bytes_ex(kind, split, L, c_in, co) // 4, dtype=np.float32)
    wp = (ctypes.c_void_p * L)(*[w.ctypes.data for w in ws])
    C.check(lib.prb_mlp_pack_weights_ex(kind, split, L, c_in, co, wp, img.ctypes.data_as(ctypes.c_void_p)), "mlp_pack")
    return img


def _padded(vs, c_out):
    """per-layer vectors -> one float32 tensor, each layer zero-padded to a multiple of 32 (the descriptor's layout)"""
    if len(vs) != len(c_out) or any(len(v) != co for v, co in zip(vs, c_out)):
        raise ValueError("mlp_chain: per-layer vectors of %s entries for layers of %s channels" % ([len(v) for v in vs], c_out))
    return torch.from_numpy(np.concatenate([np.pad(_f32(v), (0, (-co) % 32)) for v, co in zip(vs, c_out)]))


class Chain:
    """A chain of 1..3 layers y = relu(scale * (W x) + shift) packed as (kind, split) and uploaded to `device`.
    weights: float32 (c_out, c_in) per layer, numpy or torch.  shift: one vector per layer.  scale: None when it is folded
    into the weights (the descriptor's scale is NULL), else one vector per layer.  linear_last: no ReLU on the last layer.
    Owns the device tensors `desc` points at."""

    def __init__(self, kind, split, weights, shift, scale=None, linear_last=False, device="cuda"):
        image = pack_image(kind, split, weights)
        self.kind, self.split = kind, split
        self.c_in, self.c_out = weights[0].shape[1], [w.shape[0] for w in weights]
        self.flags = 1 if linear_last else 0
        self.co = _c_out_array(self.c_out)
        self.packed = torch.from_numpy(image).to(device)
        self.shift = _padded(shift, self.c_out).to(device)
        self.scale = None if scale is None else _padded(scale, self.c_out).to(device)
        d = C.MlpDesc()
        d.num_layers, d.c_in = len(self.c_out), self.c_in
        for i in range(3):
            d.c_out[i] = self.co[i]
        d.packed_w, d.shift, d.flags = self.packed.data_ptr(), self.shift.data_ptr(), self.flags
        d.scale = None if self.scale is None else self.scale.data_ptr()
        self.desc = d

    def _require(self, kind, split, c_in, entry):
        if (self.kind, self.split, self.c_in) != (kind, split, c_in):
            raise ValueError("mlp_chain: %s reads layer 0 as kind %d, split %d, %d channels; the chain is packed as kind %d, "
                             "split %d, %d channels" % (entry, kind, split, c_in, self.kind, self.split, self.c_in))

    def sa(self, xyz, centres, feats_pm, idx, ns, out, out_pm, out_c_off):
        """gather [xyz[idx] - centre | feats_pm[idx]] (B, npoint, ns) -> chain -> max over the ns samples, written into
        channels [out_c_off, out_c_off + c_last) of out (B, C, npoint) and of its point-major twin out_pm (or None)"""
        B, N, _ = xyz.shape
        npoint = centres.size(1)
        c_feat = 0 if feats_pm is None else feats_pm.size(2)
        self._require(SA, c_feat, 3 + c_feat, "prb_sa_group_mlp_max_ws")
        lib = C.lib()
        with torch.cuda.device(xyz.device):
            wsb = lib.prb_sa_workspace_bytes(B, npoint, ns, c_feat, len(self.c_out), self.co)
            ws = torch.empty(wsb, dtype=torch.uint8, device=xyz.device)
            with prof.region("sa_mlp", "%dx%d [%d]+%s" % (B * npoint, ns, 3 + c_feat, self.c_out)):
                C.check(lib.prb_sa_group_mlp_max_ws(B, N, npoint, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm),
                                                    C.ptr(idx), ctypes.byref(self.desc), C.ptr(out), C.ptr(out_pm), out.size(1),
                                                    out_c_off, C.ptr(ws), C.c_size_t(wsb), C.stream()), "sa_group_mlp_max")

    def fp(self, known_pm, idx, weight, skip, out, out_pm):
        """[sum_k weight[:, :, k] * known_pm[idx[:, :, k]] | skip] for the n points of idx (B, n, 3) -> chain -> out
        (B, c_last, n) and its point-major twin out_pm (or None).  known_pm (B, m, c_known), skip (B, c_skip, n) or None."""
        B, m, c_known = known_pm.shape
        n = idx.size(1)
        c_skip = 0 if skip is None else skip.size(1)
        self._require(FP, c_known, c_known + c_skip, "prb_fp_interp_mlp_ws")
        lib = C.lib()
        with torch.cuda.device(known_pm.device):
            wsb = lib.prb_fp_workspace_bytes(B, n, c_known, c_skip, len(self.c_out), self.co)
            ws = torch.empty(wsb, dtype=torch.uint8, device=known_pm.device)
            with prof.region("fp_mlp", "%d [%d+%d]+%s" % (B * n, c_known, c_skip, self.c_out)):
                C.check(lib.prb_fp_interp_mlp_ws(B, n, m, c_known, c_skip, C.ptr(known_pm), C.ptr(idx), C.ptr(weight), C.ptr(skip),
                                                 ctypes.byref(self.desc), C.ptr(out), C.ptr(out_pm), C.ptr(ws), C.c_size_t(wsb),
                                                 C.stream()), "fp_interp_mlp")

    def rows(self, a, b=None, tag=None, detail=None):
        """[a | b] -> chain -> (rows, round_up(c_last, 32)) row-major, the padding channels zero.  a (rows, c_a) and b
        (rows, c_b) or None are 2-D views with unit column stride and any row pitch.  tag: the profiling family (None: not
        profiled); detail: its shape string, by default the segment widths and layers."""
        rows, c_a = a.shape
        c_b = 0 if b is None else b.size(1)
        assert a.stride(1) == 1 and (b is None or (b.stride(1) == 1 and b.size(0) == rows))
        self._require(*rows_layout(c_a, c_b), c_a + c_b, "prb_mlp_rows2")
        lib = C.lib()
        dev = a.device
        pitch = (self.c_out[-1] + 31) // 32 * 32
        out = torch.empty((rows, pitch), dtype=torch.float32, device=dev)
        region = contextlib.nullcontext() if tag is None else prof.region(tag, detail or "%d [%d+%d]+%s" % (rows, c_a, c_b, self.c_out))
        with torch.cuda.device(dev):
            wsb = lib.prb_rows2_workspace_bytes(C.c_long(rows), c_a, c_b, len(self.c_out), self.co)
            ws = torch.empty(wsb, dtype=torch.uint8, device=dev)
            with region:
                C.check(lib.prb_mlp_rows2(C.c_long(rows), c_a, C.ptr(a), a.stride(0), c_b, C.ptr(b), b.stride(0) if c_b else 0,
                                          ctypes.byref(self.desc), C.ptr(out), pitch, C.ptr(ws), C.c_size_t(wsb), C.stream()),
                        "mlp_rows2")
        return out
