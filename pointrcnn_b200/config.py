"""Python-level switches of the mirror modules (which execution path a module takes).  Defaults can be seeded by
environment variables ONCE at import; at run time they are changed with `override(...)`, which is thread-local
(a DataParallel worker thread flipping a switch does not affect the others).

    disable_fused   force the reference-shaped op-by-op path (tests cross-check it against the fused kernels)
    fold_scale      fold the eval-mode BN scale into the packed weights (default) instead of an epilogue multiply
    disable_grid    always use the exhaustive ball-query / 3-NN kernels
    enable_plan     side-stream plan of the backbone forward (measured slower at batch 16, opt-in)
    prof_detail     per-shape lines in prof.collect()
    fp_project      FP modules: project the known points through layer 0 before interpolating (linearity), default on
    fp_project_min_rows   ... for FP levels with at least this many unknown points in the batch (B * n)
    fps_ordered     SA modules whose input coordinates are the output of a previous sampling (nested encoder levels) take
                    the proven-prefix shortcut of prb_furthest_point_sampling_ordered_ws (same indices), default on
    target_draw     which path ProposalTargetLayer(draw=None) takes: "torch" (the reference's random streams, default) or
                    "device" (csrc/rcnn_sample.cu's hashed draws, no host synchronisation)
    loss_impl       which path train.losses.rpn_loss / rcnn_loss(impl=None) take: "torch" (the op-by-op mirror, default) or
                    "device" (csrc/stage_loss.cu: two launches forward, one backward, no host synchronisation)
    sa_train        which path SA modules take when they need an autograd graph: "torch" (the op-by-op mirror, default) or
                    "device" (csrc/sa_train.cu through pointnet2/sa_train.py, where its rule holds)
    fp_train        which path FP modules take when they need an autograd graph: "torch" (the op-by-op mirror, default) or
                    "device" (prb_fp_train_* in csrc/sa_train.cu through pointnet2/fp_train.py, on the levels its rule
                    selects); independent of sa_train
"""
import contextlib
import os
import threading

_DEFAULTS = dict(
    disable_fused=os.environ.get("PRB_DISABLE_FUSED", "0") == "1",
    fold_scale=os.environ.get("PRB_MLP_FOLD", "1") != "0",
    disable_grid=os.environ.get("PRB_DISABLE_GRID", "0") == "1",
    enable_plan=os.environ.get("PRB_ENABLE_PLAN", "0") == "1",
    prof_detail=os.environ.get("PRB_PROF_DETAIL", "0") == "1",
    fp_project=os.environ.get("PRB_FP_PROJECT", "1") != "0",
    fp_project_min_rows=int(os.environ.get("PRB_FP_PROJECT_MIN_ROWS", "131072")),
    fps_ordered=os.environ.get("PRB_FPS_ORDERED", "1") != "0",
    target_draw=os.environ.get("PRB_TARGET_DRAW", "torch"),
    loss_impl=os.environ.get("PRB_LOSS_IMPL", "torch"),
    sa_train=os.environ.get("PRB_SA_TRAIN", "torch"),
    fp_train=os.environ.get("PRB_FP_TRAIN", "torch"),
)
_local = threading.local()


def names():
    """every switch, in a fixed order"""
    return tuple(sorted(_DEFAULTS))


def get(name):
    ov = getattr(_local, "ov", None)
    if ov and name in ov:
        return ov[name]
    return _DEFAULTS[name]


@contextlib.contextmanager
def override(**kw):
    for k in kw:
        if k not in _DEFAULTS:
            raise TypeError("unknown switch %r" % k)
    old = dict(getattr(_local, "ov", None) or {})
    _local.ov = dict(old, **kw)
    try:
        yield
    finally:
        _local.ov = old
