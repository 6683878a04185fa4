"""ctypes binding of libpointrcnn_b200.so (the C ABI declared in include/pointrcnn_b200.h).

There is deliberately no fallback: if the library is missing or a call fails, a RuntimeError is raised.
"""
import contextlib
import ctypes
import os

import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpointrcnn_b200.so")
_lib = None

c_int, c_long, c_float, c_void_p, c_size_t = ctypes.c_int, ctypes.c_long, ctypes.c_float, ctypes.c_void_p, ctypes.c_size_t


class MlpDesc(ctypes.Structure):
    """struct prb_mlp_desc"""
    _fields_ = [("num_layers", c_int), ("c_in", c_int), ("c_out", c_int * 3),
                ("packed_w", c_void_p), ("scale", c_void_p), ("shift", c_void_p), ("flags", c_int)]


class StageLossDesc(ctypes.Structure):
    """struct prb_stage_loss_desc"""
    _fields_ = [("cls_loss", c_int), ("num_class", c_int), ("focal_alpha", ctypes.c_double), ("focal_gamma", ctypes.c_double),
                ("fg_weight", ctypes.c_double), ("loss_weight_cls", ctypes.c_double), ("loss_weight_reg", ctypes.c_double),
                ("loc_scope", ctypes.c_double), ("loc_bin_size", ctypes.c_double), ("num_head_bin", c_int), ("xz_fine", c_int),
                ("y_by_bin", c_int), ("ry_fine", c_int), ("loc_y_scope", ctypes.c_double), ("loc_y_bin_size", ctypes.c_double)]


class SATrainDesc(ctypes.Structure):
    """struct prb_sa_train_desc"""
    _fields_ = [("num_layers", c_int), ("c_in", c_int), ("c_out", c_int * 3), ("bn", c_int), ("eps", ctypes.c_double),
                ("momentum", ctypes.c_double)] + [(k, c_void_p * 3) for k in ("weight", "bias", "gamma", "beta", "running_mean",
                                                                             "running_var", "num_batches_tracked")]


class Options(ctypes.Structure):
    """struct prb_options (per-thread tuning block)"""
    _fields_ = [(k, c_int) for k in ("mlp_occ", "mlp_sms", "mlp_resident", "nn_sort_queries")]


@contextlib.contextmanager
def options(**kw):
    """with options(mlp_resident=0): ...  -- overrides fields of THIS thread's prb_options for the block.
    Thread-local inside the library (prb_set_thread_options): safe under nn.DataParallel worker threads."""
    L = lib()
    old, new = Options(), Options()
    L.prb_get_thread_options(ctypes.byref(old))
    L.prb_get_thread_options(ctypes.byref(new))
    for k, v in kw.items():
        if not hasattr(new, k):
            raise TypeError("prb_options has no field %r" % k)
        setattr(new, k, v)
    L.prb_set_thread_options(ctypes.byref(new))
    try:
        yield new
    finally:
        L.prb_set_thread_options(ctypes.byref(old))


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                "pointrcnn_b200: %s is missing -- build it with `python -m pointrcnn_b200.build` "
                "(or __graft_entry__.build()); there is no CPU/PyTorch fallback." % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        L.prb_last_error.restype = ctypes.c_char_p
        L.prb_launch_count.restype = ctypes.c_ulonglong
        for name in ("prb_nms_workspace_bytes", "prb_mlp_packed_bytes", "prb_mlp_packed_bytes_ex",
                     "prb_sa_workspace_bytes", "prb_fp_workspace_bytes", "prb_rows_workspace_bytes", "prb_rows2_workspace_bytes", "prb_grid_workspace_bytes",
                     "prb_fps_workspace_bytes", "prb_fps_ordered_workspace_bytes", "prb_kitti_format_detections", "prb_rpn_proposals_workspace_bytes", "prb_roipool3d_workspace_bytes",
                     "prb_kitti_eval_workspace_bytes", "prb_kitti_eval_sets_workspace_bytes", "prb_stage_loss_workspace_bytes", "prb_sa_train_workspace_bytes",
                     "prb_fp_train_workspace_bytes", "prb_sa_train_det_workspace_bytes", "prb_group_points_grad_workspace_bytes",
                     "prb_gather_points_grad_workspace_bytes", "prb_three_interpolate_grad_workspace_bytes",
                     "prb_group_points_grad_bf16_workspace_bytes", "prb_three_interpolate_grad_bf16_workspace_bytes"):
            getattr(L, name).restype = c_size_t
        P, I, F, U = c_void_p, c_int, c_float, ctypes.c_uint
        L.prb_rcnn_sample_rois.argtypes = [I, I, I, P, P, P, P, P, I, I, F, F, F, F, ctypes.c_double, I, I, I, I, I, F, U, P, P, P, P, P, P,
                                           P]
        L.prb_rcnn_roi_targets.argtypes = [I, I, I, I, P, P, P, P, P, I, I, I, I, F, F, F, I, F, F, F, U, P, P, P, P]
        L.prb_rcnn_sample_rois_dseed.argtypes = [P if t is U else t for t in L.prb_rcnn_sample_rois.argtypes]
        L.prb_rcnn_roi_targets_dseed.argtypes = [P if t is U else t for t in L.prb_rcnn_roi_targets.argtypes]
        L.prb_adam_true_wd_step.argtypes = [I, P, P, ctypes.c_double, ctypes.c_double, P]
        L.prb_eval_box_recall.argtypes = [I, I, P, P, I, P, P, I, ctypes.POINTER(F), P, P, P, P]
        L.prb_eval_cls_acc.argtypes = [I, I, P, P, P, F, F, F, P, P, P]
        L.prb_stage_loss_workspace_bytes.argtypes = [I]
        L.prb_stage_loss_forward.argtypes = [P, I, I, P, P, P, I, P, I, P, P, P, P, P, P, P, c_size_t, P]
        L.prb_stage_loss_backward.argtypes = [P, I, I, P, P, P, I, P, I, P, P, P, P, P, P, P, P, P, P]
        L.prb_sa_train_workspace_bytes.argtypes = [I, I, I, I, P, I]
        L.prb_sa_train_forward.argtypes = [P, I, I, I, I, I, P, P, P, P, P, P, P, P, P, I, I, P, c_size_t, P]
        L.prb_sa_train_backward.argtypes = [P, I, I, I, I, I, P, P, P, P, P, P, P, P, I, I, P, P, P, P, P, P, c_size_t, P]
        L.prb_sa_train_det_workspace_bytes.argtypes = [I, I, I, I, I, P]
        L.prb_sa_train_backward_det.argtypes = L.prb_sa_train_backward.argtypes
        L.prb_fp_train_workspace_bytes.argtypes = [I, I, I, I, I, P, I]
        L.prb_fp_train_forward.argtypes = [P, I, I, I, I, I, P, P, P, P, P, P, P, P, P, c_size_t, P]
        L.prb_fp_train_backward.argtypes = [P, I, I, I, I, I, P, P, P, P, P, P, P, P, P, P, P, P, P, P, c_size_t, P]
        L.prb_options_init.restype = None
        L.prb_get_thread_options.restype = None
        if L.prb_abi_version() != 11:
            raise RuntimeError("pointrcnn_b200: ABI version mismatch")
        _lib = L
    return _lib


def check(rc, what):
    if rc != 0:
        raise RuntimeError("pointrcnn_b200.%s failed (%d): %s" % (what, rc, lib().prb_last_error().decode()))


def ptr(t):
    """device (or host) address of a contiguous tensor; None -> NULL"""
    if t is None:
        return None
    return c_void_p(t.data_ptr())


def stream():
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def launch_count():
    return int(lib().prb_launch_count())


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise RuntimeError("pointrcnn_b200: expected a CUDA tensor (there is no CPU path for this op)")


def require_contig(*tensors):
    for t in tensors:
        if t is not None and not t.is_contiguous():
            raise RuntimeError("pointrcnn_b200: tensor must be contiguous")
