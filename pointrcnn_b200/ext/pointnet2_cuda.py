"""`pointnet2_cuda` -- same exports as pointnet2_lib/pointnet2/src/pointnet2_api.cpp:10-23.

Every function takes the reference's positional arguments (explicit dims + caller-allocated tensors),
sets the device of the first tensor, launches on torch's current stream and raises RuntimeError on
failure (the reference prints and exit(-1)s).

The three gradient scatters (group_points_grad, gather_points_grad, three_interpolate_grad) add with float
atomics, so their sums come in any order.  Under torch.use_deterministic_algorithms(True) (warn_only too)
they take the ordered *_grad_ws entries instead: the same contract, the sums in a fixed order
(include/pointrcnn_b200.h), scratch from torch's allocator.

Grouping, gather and interpolation also take bfloat16 feature data (points / grad_out and the caller's out / grad_points
all bfloat16; idx int32, weight float32), as the features of a network trained under torch.autocast are: they go to the
*_bf16 entries, whose gradients sum in fp32 and round once (the ordered *_bf16_ws entries under the deterministic flag).
float32 data takes the float32 entries as before; any other dtype raises.
"""
import torch

from .. import _cabi as C


def _guard(t):
    C.require_cuda(t)
    return torch.cuda.device(t.device)


def _f32(*tensors_and_sizes):
    """float32 data tensors with at least the element count the explicit dims imply (the reference's `.data<float>()`
    throws on a dtype mismatch; an undersized tensor would be overrun by the kernel)"""
    for t, need, name in tensors_and_sizes:
        if t.dtype != torch.float32:
            raise RuntimeError("%s must be float32, got %s" % (name, t.dtype))
        if t.numel() < need:
            raise RuntimeError("%s has %d elements, the given dimensions need %d" % (name, t.numel(), need))


def _bf16(*tensors_and_sizes):
    for t, need, name in tensors_and_sizes:
        if t.dtype != torch.bfloat16:
            raise RuntimeError("%s must be bfloat16 like the features, got %s" % (name, t.dtype))
        if t.numel() < need:
            raise RuntimeError("%s has %d elements, the given dimensions need %d" % (name, t.numel(), need))


def _is_bf16(t, name):
    """True for bfloat16 feature data (the *_bf16 entries), False for float32; any other dtype raises"""
    if t.dtype == torch.bfloat16:
        return True
    if t.dtype != torch.float32:
        raise RuntimeError("%s must be float32 or bfloat16, got %s" % (name, t.dtype))
    return False


def _i32(*tensors_and_sizes):
    for t, need, name in tensors_and_sizes:
        if t.dtype != torch.int32:
            raise RuntimeError("%s must be int32, got %s" % (name, t.dtype))
        if t.numel() < need:
            raise RuntimeError("%s has %d elements, the given dimensions need %d" % (name, t.numel(), need))


def _workspace(nbytes, like):
    return torch.empty(nbytes, dtype=torch.uint8, device=like.device) if nbytes else None


def ball_query_wrapper(b, n, m, radius, nsample, new_xyz, xyz, idx):
    C.require_cuda(new_xyz, xyz, idx); C.require_contig(new_xyz, xyz, idx)
    _f32((new_xyz, b * m * 3, "new_xyz"), (xyz, b * n * 3, "xyz")); _i32((idx, b * m * nsample, "idx"))
    with _guard(xyz):
        C.check(C.lib().prb_ball_query(int(b), int(n), int(m), C.c_float(radius), int(nsample), C.ptr(new_xyz),
                                       C.ptr(xyz), C.ptr(idx), C.stream()), "ball_query")
    return 1


def group_points_wrapper(b, c, n, npoints, nsample, points, idx, out):
    C.require_cuda(points, idx, out); C.require_contig(points, idx, out)
    if _is_bf16(points, "points"):
        _bf16((points, b * c * n, "points"), (out, b * c * npoints * nsample, "out")); _i32((idx, b * npoints * nsample, "idx"))
        with _guard(points):
            C.check(C.lib().prb_group_points_bf16(int(b), int(c), int(n), int(npoints), int(nsample), C.ptr(points), C.ptr(idx),
                                                  C.ptr(out), C.stream()), "group_points_bf16")
        return 1
    _f32((points, b * c * n, "points"), (out, b * c * npoints * nsample, "out")); _i32((idx, b * npoints * nsample, "idx"))
    with _guard(points):
        C.check(C.lib().prb_group_points(int(b), int(c), int(n), int(npoints), int(nsample), C.ptr(points), C.ptr(idx),
                                         C.ptr(out), C.stream()), "group_points")
    return 1


def group_points_grad_wrapper(b, c, n, npoints, nsample, grad_out, idx, grad_points):
    C.require_cuda(grad_out, idx, grad_points); C.require_contig(grad_out, idx, grad_points)
    if _is_bf16(grad_out, "grad_out"):
        _bf16((grad_out, b * c * npoints * nsample, "grad_out"), (grad_points, b * c * n, "grad_points"))
        _i32((idx, b * npoints * nsample, "idx"))
        with _guard(grad_out):
            lib = C.lib()
            if torch.are_deterministic_algorithms_enabled():
                entry, name = lib.prb_group_points_grad_bf16_ws, "group_points_grad_bf16_ws"
                wsb = lib.prb_group_points_grad_workspace_bytes(int(b), int(n), int(npoints), int(nsample))
            else:
                entry, name = lib.prb_group_points_grad_bf16, "group_points_grad_bf16"
                wsb = lib.prb_group_points_grad_bf16_workspace_bytes(int(b), int(c), int(n))
            ws = _workspace(wsb, grad_out)
            C.check(entry(int(b), int(c), int(n), int(npoints), int(nsample), C.ptr(grad_out), C.ptr(idx), C.ptr(grad_points), C.ptr(ws),
                          C.c_size_t(wsb), C.stream()), name)
        return 1
    _f32((grad_out, b * c * npoints * nsample, "grad_out"), (grad_points, b * c * n, "grad_points")); _i32((idx, b * npoints * nsample, "idx"))
    with _guard(grad_out):
        lib = C.lib()
        if torch.are_deterministic_algorithms_enabled():
            wsb = lib.prb_group_points_grad_workspace_bytes(int(b), int(n), int(npoints), int(nsample))
            ws = _workspace(wsb, grad_out)
            C.check(lib.prb_group_points_grad_ws(int(b), int(c), int(n), int(npoints), int(nsample), C.ptr(grad_out), C.ptr(idx),
                                                 C.ptr(grad_points), C.ptr(ws), C.c_size_t(wsb), C.stream()), "group_points_grad_ws")
        else:
            C.check(lib.prb_group_points_grad(int(b), int(c), int(n), int(npoints), int(nsample), C.ptr(grad_out),
                                              C.ptr(idx), C.ptr(grad_points), C.stream()), "group_points_grad")
    return 1


def gather_points_wrapper(b, c, n, npoints, points, idx, out):
    C.require_cuda(points, idx, out); C.require_contig(points, idx, out)
    if _is_bf16(points, "points"):
        _bf16((points, b * c * n, "points"), (out, b * c * npoints, "out")); _i32((idx, b * npoints, "idx"))
        with _guard(points):
            C.check(C.lib().prb_gather_points_bf16(int(b), int(c), int(n), int(npoints), C.ptr(points), C.ptr(idx), C.ptr(out),
                                                   C.stream()), "gather_points_bf16")
        return 1
    _f32((points, b * c * n, "points"), (out, b * c * npoints, "out")); _i32((idx, b * npoints, "idx"))
    with _guard(points):
        C.check(C.lib().prb_gather_points(int(b), int(c), int(n), int(npoints), C.ptr(points), C.ptr(idx), C.ptr(out),
                                          C.stream()), "gather_points")
    return 1


def gather_points_grad_wrapper(b, c, n, npoints, grad_out, idx, grad_points):
    C.require_cuda(grad_out, idx, grad_points); C.require_contig(grad_out, idx, grad_points)
    if _is_bf16(grad_out, "grad_out"):
        _bf16((grad_out, b * c * npoints, "grad_out"), (grad_points, b * c * n, "grad_points")); _i32((idx, b * npoints, "idx"))
        with _guard(grad_out):
            lib = C.lib()
            if torch.are_deterministic_algorithms_enabled():
                entry, name = lib.prb_gather_points_grad_bf16_ws, "gather_points_grad_bf16_ws"
                wsb = lib.prb_gather_points_grad_workspace_bytes(int(b), int(n), int(npoints))
            else:
                entry, name = lib.prb_gather_points_grad_bf16, "gather_points_grad_bf16"
                wsb = lib.prb_group_points_grad_bf16_workspace_bytes(int(b), int(c), int(n))
            ws = _workspace(wsb, grad_out)
            C.check(entry(int(b), int(c), int(n), int(npoints), C.ptr(grad_out), C.ptr(idx), C.ptr(grad_points), C.ptr(ws), C.c_size_t(wsb),
                          C.stream()), name)
        return 1
    _f32((grad_out, b * c * npoints, "grad_out"), (grad_points, b * c * n, "grad_points")); _i32((idx, b * npoints, "idx"))
    with _guard(grad_out):
        lib = C.lib()
        if torch.are_deterministic_algorithms_enabled():
            wsb = lib.prb_gather_points_grad_workspace_bytes(int(b), int(n), int(npoints))
            ws = _workspace(wsb, grad_out)
            C.check(lib.prb_gather_points_grad_ws(int(b), int(c), int(n), int(npoints), C.ptr(grad_out), C.ptr(idx), C.ptr(grad_points),
                                                  C.ptr(ws), C.c_size_t(wsb), C.stream()), "gather_points_grad_ws")
        else:
            C.check(lib.prb_gather_points_grad(int(b), int(c), int(n), int(npoints), C.ptr(grad_out), C.ptr(idx),
                                               C.ptr(grad_points), C.stream()), "gather_points_grad")
    return 1


def furthest_point_sampling_wrapper(b, n, m, points, temp, idx):
    C.require_cuda(points, temp, idx); C.require_contig(points, temp, idx)
    _f32((points, b * n * 3, "points"), (temp, b * n, "temp")); _i32((idx, b * m, "idx"))
    with _guard(points):
        lib = C.lib()
        wsb = lib.prb_fps_workspace_bytes(int(b), int(n))
        ws = torch.empty(wsb, dtype=torch.uint8, device=points.device) if wsb else None
        C.check(lib.prb_furthest_point_sampling_ws(int(b), int(n), int(m), C.ptr(points), C.ptr(temp), C.ptr(idx), None,
                                                   C.ptr(ws), C.c_size_t(wsb), C.stream()), "furthest_point_sampling")
    return 1


def three_nn_wrapper(b, n, m, unknown, known, dist2, idx):
    C.require_cuda(unknown, known, dist2, idx); C.require_contig(unknown, known, dist2, idx)
    _f32((unknown, b * n * 3, "unknown"), (known, b * m * 3, "known"), (dist2, b * n * 3, "dist2")); _i32((idx, b * n * 3, "idx"))
    with _guard(unknown):
        C.check(C.lib().prb_three_nn(int(b), int(n), int(m), C.ptr(unknown), C.ptr(known), C.ptr(dist2), C.ptr(idx), None,
                                     C.stream()), "three_nn")


def three_interpolate_wrapper(b, c, m, n, points, idx, weight, out):
    C.require_cuda(points, idx, weight, out); C.require_contig(points, idx, weight, out)
    if _is_bf16(points, "points"):
        _bf16((points, b * c * m, "points"), (out, b * c * n, "out")); _f32((weight, b * n * 3, "weight")); _i32((idx, b * n * 3, "idx"))
        with _guard(points):
            C.check(C.lib().prb_three_interpolate_bf16(int(b), int(c), int(m), int(n), C.ptr(points), C.ptr(idx), C.ptr(weight),
                                                       C.ptr(out), C.stream()), "three_interpolate_bf16")
        return
    _f32((points, b * c * m, "points"), (weight, b * n * 3, "weight"), (out, b * c * n, "out")); _i32((idx, b * n * 3, "idx"))
    with _guard(points):
        C.check(C.lib().prb_three_interpolate(int(b), int(c), int(m), int(n), C.ptr(points), C.ptr(idx), C.ptr(weight),
                                              C.ptr(out), C.stream()), "three_interpolate")


def three_interpolate_grad_wrapper(b, c, n, m, grad_out, idx, weight, grad_points):
    C.require_cuda(grad_out, idx, weight, grad_points); C.require_contig(grad_out, idx, weight, grad_points)
    if _is_bf16(grad_out, "grad_out"):
        _bf16((grad_out, b * c * n, "grad_out"), (grad_points, b * c * m, "grad_points")); _f32((weight, b * n * 3, "weight"))
        _i32((idx, b * n * 3, "idx"))
        with _guard(grad_out):
            lib = C.lib()
            if torch.are_deterministic_algorithms_enabled():
                entry, name = lib.prb_three_interpolate_grad_bf16_ws, "three_interpolate_grad_bf16_ws"
                wsb = lib.prb_three_interpolate_grad_workspace_bytes(int(b), int(n), int(m))
            else:
                entry, name = lib.prb_three_interpolate_grad_bf16, "three_interpolate_grad_bf16"
                wsb = lib.prb_three_interpolate_grad_bf16_workspace_bytes(int(b), int(c), int(m))
            ws = _workspace(wsb, grad_out)
            C.check(entry(int(b), int(c), int(n), int(m), C.ptr(grad_out), C.ptr(idx), C.ptr(weight), C.ptr(grad_points), C.ptr(ws),
                          C.c_size_t(wsb), C.stream()), name)
        return
    _f32((grad_out, b * c * n, "grad_out"), (weight, b * n * 3, "weight"), (grad_points, b * c * m, "grad_points")); _i32((idx, b * n * 3, "idx"))
    with _guard(grad_out):
        lib = C.lib()
        if torch.are_deterministic_algorithms_enabled():
            wsb = lib.prb_three_interpolate_grad_workspace_bytes(int(b), int(n), int(m))
            ws = _workspace(wsb, grad_out)
            C.check(lib.prb_three_interpolate_grad_ws(int(b), int(c), int(n), int(m), C.ptr(grad_out), C.ptr(idx), C.ptr(weight),
                                                      C.ptr(grad_points), C.ptr(ws), C.c_size_t(wsb), C.stream()), "three_interpolate_grad_ws")
        else:
            C.check(lib.prb_three_interpolate_grad(int(b), int(c), int(n), int(m), C.ptr(grad_out), C.ptr(idx),
                                                   C.ptr(weight), C.ptr(grad_points), C.stream()), "three_interpolate_grad")
