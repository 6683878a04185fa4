"""CPU side of the device stage losses: the C ABI exports the new entries with the header's descriptor layout, bad options
fail with a message instead of launching, and impl="device" refuses CPU tensors instead of falling back to torch."""
import ctypes

import pytest
import torch

from pointrcnn_b200 import _cabi as C
from pointrcnn_b200 import config
from pointrcnn_b200.train import losses as L


def test_stage_loss_symbols_resolve_at_abi_11():
    lib = C.lib()
    for name in ("prb_stage_loss_workspace_bytes", "prb_stage_loss_forward", "prb_stage_loss_backward"):
        assert getattr(lib, name) is not None
    assert lib.prb_stage_loss_workspace_bytes(16 * 16384) > 0
    assert lib.prb_abi_version() == 11


def test_descriptor_layout_matches_the_header():
    """doubles after the two leading ints, NUM_HEAD_BIN and the three flags as ints: 2*4 + 7*8 + 4*4 + 2*8 bytes"""
    assert ctypes.sizeof(C.StageLossDesc) == 96
    assert C.StageLossDesc.num_head_bin.offset == 64 and C.StageLossDesc.loc_y_scope.offset == 80


def _forward(desc, rows, cols, label_bytes=8):
    one = ctypes.c_void_p(16)          # never dereferenced: the checks fail before any launch
    return C.lib().prb_stage_loss_forward(ctypes.byref(desc), rows, cols, one, one, one, label_bytes, None, 0, one, one, None, None, one,
                                          one, one, C.lib().prb_stage_loss_workspace_bytes(rows), None)


def test_bad_options_raise_before_launching():
    rpn = L._desc("SigmoidFocalLoss", 1, 0.25, 2.0, 15.0, (1.0, 1.0), 3.0, 0.5, 12, True, False, False, 0.5, 0.25)
    assert _forward(rpn, 8, 75) != 0 and b"options imply 76" in C.lib().prb_last_error()
    assert _forward(rpn, 8, 76, label_bytes=2) != 0 and b"int32 or int64" in C.lib().prb_last_error()
    ce = L._desc("CrossEntropy", 1, 0.25, 2.0, 1.0, (1.0, 1.0), 1.5, 0.5, 9, True, False, True, 0.5, 0.25)
    assert _forward(ce, 8, 46) != 0 and b"CrossEntropy" in C.lib().prb_last_error()


def test_device_impl_refuses_cpu_tensors():
    cls, reg = torch.randn(1, 10, 1), torch.randn(1, 10, 76)
    lab, rl = torch.ones(1, 10, dtype=torch.long), torch.randn(1, 10, 7)
    with pytest.raises(RuntimeError, match="CUDA"):
        L.rpn_loss(cls, reg, lab, rl, torch.ones(3), impl="device")
    with pytest.raises(RuntimeError, match="CUDA"):
        L.rcnn_loss(torch.randn(10, 1), torch.randn(10, 46), lab.view(-1), lab.view(-1), torch.randn(10, 7), torch.randn(10, 7), torch.ones(3),
                    impl="device")
    with config.override(loss_impl="device"), pytest.raises(RuntimeError, match="CUDA"):
        L.rpn_loss(cls, reg, lab, rl, torch.ones(3))
    with pytest.raises(ValueError):
        L.rpn_loss(cls, reg, lab, rl, torch.ones(3), impl="cuda")
    total, _ = L.rpn_loss(cls, reg, lab, rl, torch.ones(3))            # the default stays the torch mirror
    assert torch.isfinite(total)
