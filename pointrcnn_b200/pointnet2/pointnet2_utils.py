"""Mirror of pointnet2_lib/pointnet2/pointnet2_utils.py (reference :10-290): the autograd Functions
furthest_point_sample / gather_operation / three_nn / three_interpolate / grouping_operation / ball_query
and the QueryAndGroup / GroupAll modules, on top of the H100 `pointnet2_cuda` natives.

Same names, argument order, output shapes/dtypes and zero-/1e10-fill obligations as the reference.
Extras (used by the fused module paths, not part of the reference API): furthest_point_sample_xyz,
ball_query_msg2, three_nn_weights.

gather_operation, three_interpolate and grouping_operation also take bfloat16 features (what the SharedMLP convolutions
return under torch.autocast): the output and the feature gradient are bfloat16 too, through the *_bf16 natives (copies;
fp32 interpolation rounded once; gradients summed in fp32 and rounded once).  Indices, weights and coordinates stay
int32 / float32; float32 features take the float32 natives as before, any other dtype raises.
"""
from typing import Tuple

import torch
import torch.nn as nn
from torch.autograd import Function

from .. import _cabi as C
from .. import config
from .. import prof
from ..ext import pointnet2_cuda as pointnet2


def _cuda_empty(shape, dtype, like):
    return torch.empty(shape, dtype=dtype, device=like.device)


def _feature_dtype(features):
    """the output dtype of an index op: bfloat16 for bfloat16 features, else float32 (the natives refuse other dtypes)"""
    return torch.bfloat16 if features.dtype == torch.bfloat16 else torch.float32


def _grad_buffer(shape, grad_out):
    """the feature gradient the scatter natives fill, in the dtype of the op's output (= of grad_out, = of the features):
    bfloat16 uninitialised (the _bf16 natives write every element), else float32 zeros (they add into it)"""
    if grad_out.dtype == torch.bfloat16:
        return torch.empty(shape, dtype=torch.bfloat16, device=grad_out.device)
    return torch.zeros(shape, dtype=torch.float32, device=grad_out.device)


# Neighbour searches go through the hash grid (csrc/grid.cu) when the searched set is large enough to pay for the
# build; results are identical to the brute-force kernels either way.  config.override(disable_grid=True) forces brute force.
GRID_MIN_POINTS_BQ = 2048
GRID_MIN_POINTS_NN = 512


def _use_grid(n_points, threshold):
    return n_points >= threshold and not config.get("disable_grid")


def _ball_query_native(B, N, npoint, radii, nsamples, new_xyz, xyz, idxs):
    import ctypes
    lib = C.lib()
    if _use_grid(N, GRID_MIN_POINTS_BQ) and all(r > 0 for r in radii):
        nr = len(radii)
        wsb = lib.prb_grid_workspace_bytes(B, N, npoint)
        ws = torch.empty(wsb, dtype=torch.uint8, device=xyz.device)
        rad = (ctypes.c_float * nr)(*radii)
        nsm = (ctypes.c_int * nr)(*[int(x) for x in nsamples])
        ptrs = (ctypes.c_void_p * nr)(*[t.data_ptr() for t in idxs])
        C.check(lib.prb_ball_query_grid(B, N, npoint, nr, rad, nsm, C.ptr(new_xyz), C.ptr(xyz), ptrs, C.ptr(ws), C.c_size_t(wsb),
                                        C.stream()), "ball_query_grid")
    elif len(radii) == 2:
        C.check(lib.prb_ball_query_msg2(B, N, npoint, C.c_float(radii[0]), int(nsamples[0]), C.c_float(radii[1]), int(nsamples[1]),
                                        C.ptr(new_xyz), C.ptr(xyz), C.ptr(idxs[0]), C.ptr(idxs[1]), C.stream()), "ball_query_msg2")
    else:
        C.check(lib.prb_ball_query(B, N, npoint, C.c_float(radii[0]), int(nsamples[0]), C.ptr(new_xyz), C.ptr(xyz), C.ptr(idxs[0]),
                                   C.stream()), "ball_query")


def _three_nn_native(B, N, m, unknown, known, dist2, idx, weight):
    lib = C.lib()
    if _use_grid(m, GRID_MIN_POINTS_NN):
        wsb = lib.prb_grid_workspace_bytes(B, m, N)
        ws = torch.empty(wsb, dtype=torch.uint8, device=unknown.device)
        C.check(lib.prb_three_nn_grid(B, N, m, C.ptr(unknown), C.ptr(known), C.ptr(dist2), C.ptr(idx), C.ptr(weight), C.ptr(ws),
                                      C.c_size_t(wsb), C.stream()), "three_nn_grid")
    else:
        C.check(lib.prb_three_nn(B, N, m, C.ptr(unknown), C.ptr(known), C.ptr(dist2), C.ptr(idx), C.ptr(weight), C.stream()), "three_nn")


def _fps_native(B, N, npoint, xyz, temp, idx, new_xyz):
    """FPS through the C ABI, lending the library scratch memory (pruned kernel for big scenes)"""
    lib = C.lib()
    wsb = lib.prb_fps_workspace_bytes(B, N)
    ws = torch.empty(wsb, dtype=torch.uint8, device=xyz.device) if wsb else None
    C.check(lib.prb_furthest_point_sampling_ws(B, N, int(npoint), C.ptr(xyz), C.ptr(temp), C.ptr(idx), C.ptr(new_xyz),
                                               C.ptr(ws), C.c_size_t(wsb), C.stream()), "furthest_point_sampling")


class FurthestPointSampling(Function):
    @staticmethod
    def forward(ctx, xyz: torch.Tensor, npoint: int) -> torch.Tensor:
        """xyz (B,N,3) -> (B,npoint) int32 indices of the iteratively furthest points (starts at point 0)"""
        assert xyz.is_contiguous()
        B, N, _ = xyz.size()
        output = _cuda_empty((B, npoint), torch.int32, xyz)
        temp = torch.full((B, N), 1e10, dtype=torch.float32, device=xyz.device)
        pointnet2.furthest_point_sampling_wrapper(B, N, npoint, xyz, temp, output)
        return output

    @staticmethod
    def backward(xyz, a=None):
        return None, None


furthest_point_sample = FurthestPointSampling.apply


def mark_sampling_order(t: torch.Tensor) -> torch.Tensor:
    """tag coordinates as "listed in furthest-point-sampling order from point 0" (a hint, never trusted: see
    furthest_point_sample_xyz)"""
    t._prb_sampling_order = True
    return t


def in_sampling_order(t: torch.Tensor) -> bool:
    return bool(getattr(t, "_prb_sampling_order", False))


def furthest_point_sample_xyz(xyz: torch.Tensor, npoint: int, ordered: bool = None, return_todo: bool = False):
    """FPS that also emits the sampled coordinates: (idx (B,npoint) int32, new_xyz (B,npoint,3)); no grad.
    The returned new_xyz is tagged as being in sampling order.  `ordered` (default: the tag of `xyz`): the input is
    probably the output of an earlier sampling, so try to PROVE idx = 0..npoint-1 per scene first
    (prb_furthest_point_sampling_ordered_ws; scenes where the proof fails are sampled as usual, results identical).
    return_todo: also return the (B,) int32 per-scene flags (1 = sampled by the kernels, 0 = answered by the proof)."""
    assert xyz.is_contiguous()
    C.require_cuda(xyz)
    B, N, _ = xyz.size()
    if ordered is None:
        # below ~256 points a sampling launch costs less than the three proof launches (RCNN stage: 2048 RoIs x 128 -> 32)
        ordered = in_sampling_order(xyz) and config.get("fps_ordered") and N >= 256
    idx = _cuda_empty((B, npoint), torch.int32, xyz)
    new_xyz = _cuda_empty((B, npoint, 3), torch.float32, xyz)
    temp = torch.full((B, N), 1e10, dtype=torch.float32, device=xyz.device)
    todo = None
    with torch.cuda.device(xyz.device), prof.region("fps"):
        if ordered and 2 <= npoint <= N:
            lib = C.lib()
            wsb = lib.prb_fps_ordered_workspace_bytes(B, N, int(npoint))
            ws = torch.empty(wsb, dtype=torch.uint8, device=xyz.device)
            todo = torch.empty(B, dtype=torch.int32, device=xyz.device) if return_todo else None
            C.check(lib.prb_furthest_point_sampling_ordered_ws(B, N, int(npoint), C.ptr(xyz), C.ptr(temp), C.ptr(idx), C.ptr(new_xyz),
                                                               C.ptr(todo), C.ptr(ws), C.c_size_t(wsb), C.stream()),
                    "furthest_point_sampling_ordered")
        else:
            _fps_native(B, N, npoint, xyz, temp, idx, new_xyz)
            if return_todo:
                todo = torch.ones(B, dtype=torch.int32, device=xyz.device)
    mark_sampling_order(new_xyz)
    return (idx, new_xyz, todo) if return_todo else (idx, new_xyz)


class GatherOperation(Function):
    @staticmethod
    def forward(ctx, features: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
        """features (B,C,N), idx (B,npoint) -> (B,C,npoint)"""
        assert features.is_contiguous()
        assert idx.is_contiguous()
        B, npoint = idx.size()
        _, Cc, N = features.size()
        output = _cuda_empty((B, Cc, npoint), _feature_dtype(features), features)
        pointnet2.gather_points_wrapper(B, Cc, N, npoint, features, idx, output)
        ctx.for_backwards = (idx, Cc, N)
        return output

    @staticmethod
    def backward(ctx, grad_out):
        idx, Cc, N = ctx.for_backwards
        B, npoint = idx.size()
        grad_features = _grad_buffer((B, Cc, N), grad_out)
        pointnet2.gather_points_grad_wrapper(B, Cc, N, npoint, grad_out.contiguous(), idx, grad_features)
        return grad_features, None


gather_operation = GatherOperation.apply


class ThreeNN(Function):
    @staticmethod
    def forward(ctx, unknown: torch.Tensor, known: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
        """unknown (B,N,3), known (B,M,3) -> (dist (B,N,3) l2 distances, idx (B,N,3) int32)"""
        assert unknown.is_contiguous()
        assert known.is_contiguous()
        B, N, _ = unknown.size()
        m = known.size(1)
        dist2 = _cuda_empty((B, N, 3), torch.float32, unknown)
        idx = _cuda_empty((B, N, 3), torch.int32, unknown)
        C.require_cuda(unknown, known)
        with torch.cuda.device(unknown.device), prof.region("three_nn"):
            _three_nn_native(B, N, int(m), unknown, known, dist2, idx, None)
        return torch.sqrt(dist2), idx

    @staticmethod
    def backward(ctx, a=None, b=None):
        return None, None


three_nn = ThreeNN.apply


def three_nn_weights(unknown: torch.Tensor, known: torch.Tensor):
    """three_nn + the inverse-distance weights of pointnet2_modules.py:140-142 in one kernel:
    (dist2 (B,N,3), idx (B,N,3) int32, weight (B,N,3)); no grad"""
    assert unknown.is_contiguous() and known.is_contiguous()
    C.require_cuda(unknown, known)
    B, N, _ = unknown.size()
    m = known.size(1)
    dist2 = _cuda_empty((B, N, 3), torch.float32, unknown)
    idx = _cuda_empty((B, N, 3), torch.int32, unknown)
    weight = _cuda_empty((B, N, 3), torch.float32, unknown)
    with torch.cuda.device(unknown.device), prof.region("three_nn"):
        _three_nn_native(B, N, int(m), unknown, known, dist2, idx, weight)
    return dist2, idx, weight


class ThreeInterpolate(Function):
    @staticmethod
    def forward(ctx, features: torch.Tensor, idx: torch.Tensor, weight: torch.Tensor) -> torch.Tensor:
        """features (B,C,M), idx (B,n,3), weight (B,n,3) -> (B,C,n)"""
        assert features.is_contiguous()
        assert idx.is_contiguous()
        assert weight.is_contiguous()
        B, c, m = features.size()
        n = idx.size(1)
        ctx.three_interpolate_for_backward = (idx, weight, m)
        output = _cuda_empty((B, c, n), _feature_dtype(features), features)
        pointnet2.three_interpolate_wrapper(B, c, m, n, features, idx, weight, output)
        return output

    @staticmethod
    def backward(ctx, grad_out: torch.Tensor):
        idx, weight, m = ctx.three_interpolate_for_backward
        B, c, n = grad_out.size()
        grad_features = _grad_buffer((B, c, m), grad_out)
        pointnet2.three_interpolate_grad_wrapper(B, c, n, m, grad_out.contiguous(), idx, weight, grad_features)
        return grad_features, None, None


three_interpolate = ThreeInterpolate.apply


class GroupingOperation(Function):
    @staticmethod
    def forward(ctx, features: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
        """features (B,C,N), idx (B,npoint,nsample) -> (B,C,npoint,nsample)"""
        assert features.is_contiguous()
        assert idx.is_contiguous()
        B, nfeatures, nsample = idx.size()
        _, Cc, N = features.size()
        output = _cuda_empty((B, Cc, nfeatures, nsample), _feature_dtype(features), features)
        pointnet2.group_points_wrapper(B, Cc, N, nfeatures, nsample, features, idx, output)
        ctx.for_backwards = (idx, N)
        return output

    @staticmethod
    def backward(ctx, grad_out: torch.Tensor):
        idx, N = ctx.for_backwards
        B, Cc, npoint, nsample = grad_out.size()
        grad_features = _grad_buffer((B, Cc, N), grad_out)
        pointnet2.group_points_grad_wrapper(B, Cc, N, npoint, nsample, grad_out.contiguous(), idx, grad_features)
        return grad_features, None


grouping_operation = GroupingOperation.apply


class BallQuery(Function):
    @staticmethod
    def forward(ctx, radius: float, nsample: int, xyz: torch.Tensor, new_xyz: torch.Tensor) -> torch.Tensor:
        """xyz (B,N,3), new_xyz (B,npoint,3) -> idx (B,npoint,nsample) int32 (rows without a hit stay 0)"""
        assert new_xyz.is_contiguous()
        assert xyz.is_contiguous()
        B, N, _ = xyz.size()
        npoint = new_xyz.size(1)
        idx = torch.zeros((B, npoint, nsample), dtype=torch.int32, device=xyz.device)
        C.require_cuda(xyz, new_xyz)
        with torch.cuda.device(xyz.device), prof.region("ball_query"):
            _ball_query_native(B, N, npoint, [float(radius)], [int(nsample)], new_xyz, xyz, [idx])
        return idx

    @staticmethod
    def backward(ctx, a=None):
        return None, None, None, None


ball_query = BallQuery.apply


def ball_query_msg2(radii, nsamples, xyz: torch.Tensor, new_xyz: torch.Tensor):
    """two radii over the same centres in one scan -> (idx0, idx1); each equals ball_query(r_k, ns_k, ...)"""
    assert xyz.is_contiguous() and new_xyz.is_contiguous()
    C.require_cuda(xyz, new_xyz)
    B, N, _ = xyz.size()
    npoint = new_xyz.size(1)
    idx0 = torch.zeros((B, npoint, nsamples[0]), dtype=torch.int32, device=xyz.device)
    idx1 = torch.zeros((B, npoint, nsamples[1]), dtype=torch.int32, device=xyz.device)
    with torch.cuda.device(xyz.device), prof.region("ball_query"):
        _ball_query_native(B, N, npoint, list(radii), list(nsamples), new_xyz, xyz, [idx0, idx1])
    return idx0, idx1


def transpose_bcn_to_bnc(t: torch.Tensor) -> torch.Tensor:
    """(B,C,N) -> contiguous (B,N,C)"""
    assert t.is_contiguous()
    B, Cc, N = t.size()
    out = _cuda_empty((B, N, Cc), torch.float32, t)
    with torch.cuda.device(t.device), prof.region("transpose"):
        C.check(C.lib().prb_transpose_bcn_to_bnc(B, Cc, N, C.ptr(t), C.ptr(out), C.stream()), "transpose")
    return out


class QueryAndGroup(nn.Module):
    def __init__(self, radius: float, nsample: int, use_xyz: bool = True):
        super().__init__()
        self.radius, self.nsample, self.use_xyz = radius, nsample, use_xyz

    def forward(self, xyz: torch.Tensor, new_xyz: torch.Tensor, features: torch.Tensor = None) -> Tuple[torch.Tensor]:
        """xyz (B,N,3), new_xyz (B,npoint,3), features (B,C,N) -> (B, 3+C, npoint, nsample); xyz channels first,
        relative to the ball centre"""
        idx = ball_query(self.radius, self.nsample, xyz, new_xyz)
        xyz_trans = xyz.transpose(1, 2).contiguous()
        grouped_xyz = grouping_operation(xyz_trans, idx)
        grouped_xyz = grouped_xyz - new_xyz.transpose(1, 2).unsqueeze(-1)
        if features is not None:
            grouped_features = grouping_operation(features, idx)
            return torch.cat([grouped_xyz, grouped_features], dim=1) if self.use_xyz else grouped_features
        assert self.use_xyz, "Cannot have not features and not use xyz as a feature!"
        return grouped_xyz


class GroupAll(nn.Module):
    def __init__(self, use_xyz: bool = True):
        super().__init__()
        self.use_xyz = use_xyz

    def forward(self, xyz: torch.Tensor, new_xyz: torch.Tensor, features: torch.Tensor = None):
        """-> (B, 3+C, 1, N); no sampling, no centre subtraction"""
        grouped_xyz = xyz.transpose(1, 2).unsqueeze(2)
        if features is not None:
            grouped_features = features.unsqueeze(2)
            return torch.cat([grouped_xyz, grouped_features], dim=1) if self.use_xyz else grouped_features
        return grouped_xyz
