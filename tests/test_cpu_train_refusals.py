"""The SA and FP training entries refuse a missing per-layer buffer before they launch anything: they return -1 with a
message naming the buffer, and no kernel runs on the arguments they were given.

Every other pointer is a non-NULL host placeholder.  An entry that launched before refusing would run kernels on those,
so with a GPU present these cases are skipped; without one, such a launch returns a CUDA error instead of -1."""
import ctypes

import pytest
import torch

from pointrcnn_b200 import _cabi as C

pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="a launch before the refusal would run on placeholder pointers")

_HOST = ctypes.create_string_buffer(64)
PH = ctypes.addressof(_HOST)


def _desc(c_in, widths):
    d = C.SATrainDesc(num_layers=len(widths), c_in=c_in, bn=1, eps=1e-5, momentum=0.1)
    for l, w in enumerate(widths):
        d.c_out[l] = w
        for k in ("weight", "gamma", "beta", "running_mean", "running_var", "num_batches_tracked"):
            getattr(d, k)[l] = PH
    return d


def _layers(*ptrs):
    return (ctypes.c_void_p * 3)(*ptrs)


SA = dict(b=2, n=64, npoint=16, ns=8, c_feat=1, widths=[16, 16, 32])


def test_sa_backward_refuses_a_missing_weight_gradient_before_launching():
    lib, s = C.lib(), SA
    d = _desc(3 + s["c_feat"], s["widths"])
    ws = lib.prb_sa_train_workspace_bytes(s["b"], s["npoint"], s["ns"], s["c_feat"], ctypes.byref(d), 1)
    assert ws > 0
    every = _layers(PH, PH, PH)
    rc = lib.prb_sa_train_backward(ctypes.byref(d), s["b"], s["n"], s["npoint"], s["ns"], s["c_feat"], PH, PH, PH, PH, every, PH, PH, PH,
                                   s["widths"][-1], 0, _layers(None, PH, PH), every, every, every, PH, PH, ws, None)
    assert rc == -1
    assert b"layer 0: no weight gradient" in lib.prb_last_error()


def test_sa_forward_refuses_a_missing_z_buffer_before_launching():
    lib, s = C.lib(), SA
    d = _desc(3 + s["c_feat"], s["widths"])
    ws = lib.prb_sa_train_workspace_bytes(s["b"], s["npoint"], s["ns"], s["c_feat"], ctypes.byref(d), 0)
    rc = lib.prb_sa_train_forward(ctypes.byref(d), s["b"], s["n"], s["npoint"], s["ns"], s["c_feat"], PH, PH, PH, PH, _layers(PH, None, PH),
                                  PH, PH, PH, PH, s["widths"][-1], 0, PH, ws, None)
    assert rc == -1
    assert b"layer 1: no Z buffer" in lib.prb_last_error()


def test_fp_forward_refuses_a_missing_z_buffer_before_launching():
    lib = C.lib()
    b, n, m, c_known, c_skip, widths = 2, 64, 16, 8, 4, [16, 16]
    d = _desc(c_known + c_skip, widths)
    ws = lib.prb_fp_train_workspace_bytes(b, n, m, c_known, c_skip, ctypes.byref(d), 0)
    assert ws > 0
    rc = lib.prb_fp_train_forward(ctypes.byref(d), b, n, m, c_known, c_skip, PH, PH, PH, PH, _layers(PH, None), PH, PH, None, PH, ws, None)
    assert rc == -1
    assert b"layer 1: no Z buffer" in lib.prb_last_error()
