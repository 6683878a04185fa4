"""The ordered gradient entries on the device: bit for bit against the float32 restatement of
test_cpu_deterministic_grads.py at the training shapes and on edge cases, the ordered SA training backward against the
float64 reference and the atomic entry, no host synchronisation, and two seeded training runs under
torch.use_deterministic_algorithms(True) that end with the same bits."""
import ctypes
import hashlib
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import sa_train_reference as R
from test_cpu_deterministic_grads import group_grad_ref, interp_grad_ref
from pointrcnn_b200 import _cabi as C
from pointrcnn_b200.ext import pointnet2_cuda
from pointrcnn_b200.pointnet2 import pointnet2_utils as pu
from pointrcnn_b200.pointnet2 import sa_train

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture
def deterministic():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    yield
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _bits_equal(got, want):
    got, want = np.ascontiguousarray(got, np.float32), np.ascontiguousarray(want, np.float32)
    assert got.shape == want.shape, (got.shape, want.shape)
    bad = got.view(np.int32) != want.view(np.int32)
    assert not bad.any(), "%d of %d words differ, first at %s: %r vs %r" % (bad.sum(), bad.size, np.argwhere(bad)[0].tolist(),
                                                                         got[bad][0], want[bad][0])


def _chunked(ref, g, c_axis, chunk=32, **kw):
    """the restatement channel block by channel block (every channel is independent): bounds the host memory"""
    return np.concatenate([ref(np.take(g, range(c0, min(c0 + chunk, g.shape[c_axis])), axis=c_axis), **kw)
                           for c0 in range(0, g.shape[c_axis], chunk)], axis=1) if g.shape[c_axis] else ref(g, **kw)


def _padded_idx(gen, b, npoint, ns, n):
    """ball-query-like idx: a random number of hits per centre, the rest padded with the first hit"""
    idx = torch.randint(0, n, (b, npoint, ns), generator=gen)
    hits = torch.randint(1, ns + 1, (b, npoint, 1), generator=gen)
    return torch.where(torch.arange(ns) >= hits, idx[:, :, :1], idx).int()


def _group_ws(cuda, g, idx, n, prefill):
    """prb_group_points_grad_ws through the shim (flag on) on a prefilled grad_points"""
    b, c = g.shape[:2]
    npoints, ns = idx.shape[1], idx.shape[2]
    gp = prefill.to(cuda).clone()
    pointnet2_cuda.group_points_grad_wrapper(b, c, n, npoints, ns, g.to(cuda).contiguous(), idx.to(cuda).contiguous(), gp)
    return gp.cpu().numpy()


# ------------------------------------------------------------------------------------------ grouping and gather
GROUP_SHAPES = {
    # name: (B, C, N, npoint, nsample)
    "rpn_sa1_xyz_ns16": (16, 3, 16384, 4096, 16),
    "rpn_sa1_feats_ns32": (16, 1, 16384, 4096, 32),
    "rpn_sa2_ns16": (16, 96, 4096, 1024, 16),
    "rpn_sa2_ns32": (16, 96, 4096, 1024, 32),
    "rpn_sa3_ns16": (16, 256, 1024, 256, 16),
    "rpn_sa3_ns32": (16, 256, 1024, 256, 32),
    "rpn_sa4_ns16": (16, 512, 256, 64, 16),
    "rpn_sa4_ns32": (16, 512, 256, 64, 32),
    "rcnn_sa1_256_rois": (256, 128, 512, 128, 64),
    "rcnn_sa2_256_rois": (256, 128, 128, 32, 64),
}


@pytest.mark.parametrize("name", list(GROUP_SHAPES))
def test_group_grad_ws_bits_at_training_shapes(cuda, deterministic, name):
    B, Cc, N, P, S = GROUP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name))
    idx = _padded_idx(gen, B, P, S, N)
    g = torch.randn(B, Cc, P, S, generator=gen)
    prefill = torch.randn(B, Cc, N, generator=gen)
    got = _group_ws(cuda, g, idx, N, prefill)
    want = _chunked(group_grad_ref, g.numpy(), 1, idx=idx.numpy(), n=N, out=None)
    _bits_equal(got, prefill.numpy() + want)


def test_group_grad_ws_bits_group_all(cuda, deterministic):
    """GroupAll's layout (RCNN SA3: every point once, npoint 1, nsample N)"""
    B, Cc, N = 256, 256, 32
    idx = torch.arange(N, dtype=torch.int32).view(1, 1, N).expand(B, 1, N).contiguous()
    g = torch.randn(B, Cc, 1, N, generator=torch.Generator().manual_seed(1))
    got = _group_ws(cuda, g, idx, N, torch.zeros(B, Cc, N))
    _bits_equal(got, group_grad_ref(g.numpy(), idx.numpy(), N))


@pytest.mark.parametrize("B,Cc,N,npoint", [(16, 3, 16384, 4096), (16, 96, 4096, 1024), (3, 13, 50, 200)])
def test_gather_grad_ws_bits(cuda, deterministic, B, Cc, N, npoint):
    """nsample = 1; the last case names points more than once"""
    gen = torch.Generator().manual_seed(N)
    idx = torch.randint(0, N, (B, npoint), generator=gen).int()
    g = torch.randn(B, Cc, npoint, generator=gen)
    gp = torch.zeros(B, Cc, N, device=cuda)
    pointnet2_cuda.gather_points_grad_wrapper(B, Cc, N, npoint, g.to(cuda), idx.to(cuda), gp)
    _bits_equal(gp.cpu().numpy(), group_grad_ref(g.numpy(), idx.numpy(), N))


# ------------------------------------------------------------------------------------------ interpolation
INTERP_SHAPES = {
    # RPN FP levels, top to bottom: (B, C, n unknown, m known)
    "rpn_fp_sa4_to_sa3": (16, 1024, 256, 64),
    "rpn_fp_sa3_to_sa2": (16, 512, 1024, 256),
    "rpn_fp_sa2_to_sa1": (16, 512, 4096, 1024),
    "rpn_fp_sa1_to_input": (16, 256, 16384, 4096),
}


def _taps(gen, B, n, m):
    """three distinct known points per unknown point and positive weights summing to about 1, as three_nn_weights gives"""
    idx = torch.stack([torch.randperm(m, generator=gen)[:3] for _ in range(min(n, 64))])
    idx = idx[torch.randint(0, idx.shape[0], (B, n), generator=gen)]
    idx = (idx + torch.randint(0, m, (B, n, 1), generator=gen)) % m
    w = torch.rand(B, n, 3, generator=gen) + 0.01
    return idx.int().contiguous(), (w / w.sum(2, keepdim=True)).contiguous()


def _interp_ws(cuda, g, idx, w, m, prefill):
    B, Cc, n = g.shape
    gp = prefill.to(cuda).clone()
    pointnet2_cuda.three_interpolate_grad_wrapper(B, Cc, n, m, g.to(cuda).contiguous(), idx.to(cuda), w.to(cuda), gp)
    return gp.cpu().numpy()


@pytest.mark.parametrize("name", list(INTERP_SHAPES))
def test_three_interpolate_grad_ws_bits_at_training_shapes(cuda, deterministic, name):
    B, Cc, n, m = INTERP_SHAPES[name]
    gen = torch.Generator().manual_seed(len(name))
    idx, w = _taps(gen, B, n, m)
    g = torch.randn(B, Cc, n, generator=gen)
    prefill = torch.randn(B, Cc, m, generator=gen)
    got = _interp_ws(cuda, g, idx, w, m, prefill)
    want = _chunked(interp_grad_ref, g.numpy(), 1, idx=idx.numpy(), weight=w.numpy(), m=m)
    _bits_equal(got, prefill.numpy() + want)


# ------------------------------------------------------------------------------------------ edge cases
def test_lone_points_padded_to_nsample_duplicates(cuda, deterministic):
    """centres whose ball holds one point reference it nsample times; one point is the only neighbour of every centre"""
    B, Cc, N, P, S = 2, 11, 40, 300, 64
    gen = torch.Generator().manual_seed(2)
    idx = _padded_idx(gen, B, P, S, N)
    idx[:, ::3] = idx[:, ::3, :1]            # a third of the centres: one hit, padded
    idx[1] = 7                               # scene 1: point 7 is every centre's only neighbour (19200 references)
    g = torch.randn(B, Cc, P, S, generator=gen)
    got = _group_ws(cuda, g, idx, N, torch.zeros(B, Cc, N))
    _bits_equal(got, group_grad_ref(g.numpy(), idx.numpy(), N))


def test_repeated_taps_and_unreferenced_points(cuda, deterministic):
    """an unknown point whose three taps name one known point; known points nobody names stay as they were"""
    B, Cc, n, m = 3, 21, 500, 700
    gen = torch.Generator().manual_seed(3)
    idx, w = _taps(gen, B, n, m)
    idx[:, :50] = idx[:, :50, :1]
    idx = (idx % 300).int().contiguous()    # known points 300.. are never named
    g = torch.randn(B, Cc, n, generator=gen)
    prefill = torch.randn(B, Cc, m, generator=gen)
    got = _interp_ws(cuda, g, idx, w, m, prefill)
    _bits_equal(got, prefill.numpy() + interp_grad_ref(g.numpy(), idx.numpy(), w.numpy(), m))
    _bits_equal(got[:, :, 300:], prefill.numpy()[:, :, 300:])


@pytest.mark.parametrize("Cc", [1, 7, 9, 17, 130])
def test_channel_counts_off_the_channel_block(cuda, deterministic, Cc):
    B, N, P, S = 2, 333, 100, 16
    gen = torch.Generator().manual_seed(Cc)
    idx = _padded_idx(gen, B, P, S, N)
    g = torch.randn(B, Cc, P, S, generator=gen)
    got = _group_ws(cuda, g, idx, N, torch.zeros(B, Cc, N))
    _bits_equal(got, group_grad_ref(g.numpy(), idx.numpy(), N))
    ti, tw = _taps(gen, B, 257, N)
    gi = torch.randn(B, Cc, 257, generator=gen)
    _bits_equal(_interp_ws(cuda, gi, ti, tw, N, torch.zeros(B, Cc, N)), interp_grad_ref(gi.numpy(), ti.numpy(), tw.numpy(), N))


@pytest.mark.parametrize("b,c,n", [(0, 4, 10), (2, 0, 10), (2, 4, 0)])
def test_empty_sizes_are_a_no_op(cuda, b, c, n):
    """b, c or n of 0: nothing to sum, no scratch needed (NULL, 0 bytes), grad_points untouched"""
    L = C.lib()
    s = C.stream()
    gp = torch.full((max(b * c * max(n, 4), 1),), 3.0, device=cuda)
    g = torch.ones(max(b * c * max(n, 4) * 3, 1), device=cuda)
    idx = torch.zeros(max(b * max(n, 4) * 3, 1), dtype=torch.int32, device=cuda)
    w = torch.ones(max(b * max(n, 4) * 3, 1), device=cuda)
    if c:                                   # the sizes do not depend on c
        assert L.prb_group_points_grad_workspace_bytes(b, n, 4, 2) == 0 and L.prb_three_interpolate_grad_workspace_bytes(b, n, 4) == 0
    C.check(L.prb_group_points_grad_ws(b, c, n, 4, 2, C.ptr(g), C.ptr(idx), C.ptr(gp), None, C.c_size_t(0), s), "group_points_grad_ws")
    C.check(L.prb_gather_points_grad_ws(b, c, n, 4, C.ptr(g), C.ptr(idx), C.ptr(gp), None, C.c_size_t(0), s), "gather_points_grad_ws")
    # interpolation with n unknown points, and with n known points
    C.check(L.prb_three_interpolate_grad_ws(b, c, n, 4, C.ptr(g), C.ptr(idx), C.ptr(w), C.ptr(gp), None, C.c_size_t(0), s), "three_interpolate_grad_ws")
    C.check(L.prb_three_interpolate_grad_ws(b, c, 4, n, C.ptr(g), C.ptr(idx), C.ptr(w), C.ptr(gp), None, C.c_size_t(0), s), "three_interpolate_grad_ws")
    torch.cuda.synchronize()
    assert (gp == 3.0).all()


def test_small_workspace_is_refused(cuda):
    L = C.lib()
    idx = torch.zeros(8, dtype=torch.int32, device=cuda)
    g = torch.ones(16, device=cuda)
    gp = torch.zeros(20, device=cuda)
    need = L.prb_group_points_grad_workspace_bytes(1, 10, 4, 2)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    rc = L.prb_group_points_grad_ws(1, 2, 10, 4, 2, C.ptr(g), C.ptr(idx), C.ptr(gp), C.ptr(ws), C.c_size_t(need - 1), C.stream())
    assert rc != 0 and b"workspace" in L.prb_last_error()


def test_autograd_functions_use_the_ordered_path_and_repeat_bits(cuda, deterministic):
    """GroupingOperation / ThreeInterpolate backward twice under the flag: the same bits, equal to the restatement"""
    gen = torch.Generator().manual_seed(9)
    B, Cc, N, P, S = 4, 40, 2000, 512, 32
    feats = torch.randn(B, Cc, N, generator=gen).to(cuda).requires_grad_(True)
    idx = _padded_idx(gen, B, P, S, N).to(cuda)
    gout = torch.randn(B, Cc, P, S, generator=gen).to(cuda)
    grads = []
    for _ in range(2):
        feats.grad = None
        pu.grouping_operation(feats, idx).backward(gout)
        grads.append(feats.grad.cpu().numpy())
    _bits_equal(grads[0], grads[1])
    _bits_equal(grads[0], group_grad_ref(gout.cpu().numpy(), idx.cpu().numpy(), N))
    ti, tw = _taps(gen, B, N, P)
    known = torch.randn(B, Cc, P, generator=gen).to(cuda).requires_grad_(True)
    gi = torch.randn(B, Cc, N, generator=gen).to(cuda)
    pu.three_interpolate(known, ti.to(cuda), tw.to(cuda)).backward(gi)
    _bits_equal(known.grad.cpu().numpy(), interp_grad_ref(gi.cpu().numpy(), ti.numpy(), tw.numpy(), P))


def test_no_host_synchronisation(cuda, deterministic):
    gen = torch.Generator().manual_seed(4)
    feats = torch.randn(2, 16, 1000, generator=gen).to(cuda).requires_grad_(True)
    idx = _padded_idx(gen, 2, 256, 16, 1000).to(cuda)
    gidx = torch.randint(0, 1000, (2, 256), generator=gen).int().to(cuda)
    ti, tw = _taps(gen, 2, 1000, 256)
    known = torch.randn(2, 16, 256, generator=gen).to(cuda).requires_grad_(True)
    ti, tw = ti.to(cuda), tw.to(cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        y = pu.grouping_operation(feats, idx).sum() + pu.gather_operation(feats, gidx).sum() + pu.three_interpolate(known, ti, tw).sum()
        y.backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()
    assert feats.grad.abs().sum() > 0 and known.grad.abs().sum() > 0


# ------------------------------------------------------------------------------------------ the SA training backward
def _sa_desc(case, cuda):
    layers = case["layers"]
    d = C.SATrainDesc()
    keep = []
    c_feat = 0 if case["feats"] is None else case["feats"].shape[1]
    d.num_layers, d.c_in, d.bn = len(layers), 3 + c_feat, 0
    for l, lay in enumerate(layers):
        w, b = lay["w"].float().to(cuda).contiguous(), lay["b"].float().to(cuda)
        keep += [w, b]
        d.c_out[l], d.weight[l], d.bias[l] = w.shape[0], w.data_ptr(), b.data_ptr()
    return d, keep


def _ptrs(ts):
    return (ctypes.c_void_p * 3)(*[None if t is None else t.data_ptr() for t in ts] + [None] * (3 - len(ts)))


def _sa_run(case, cuda, reps=2):
    """prb_sa_train_forward, then the atomic backward into zeros and the ordered backward `reps` times into NaN-filled
    buffers (it writes every word) -> (atomic grad_feats, [ordered grad_feats], [ordered grad_weight lists], atomic grad_weight)"""
    L = C.lib()
    s = C.stream()
    d, keep = _sa_desc(case, cuda)
    xyz, centres, idx = case["xyz"].to(cuda), case["centres"].to(cuda), case["idx"].to(cuda)
    B, N, _ = xyz.shape
    _, P, ns = idx.shape
    c_feat = case["feats"].shape[1]
    feats_pm = case["feats"].to(cuda).transpose(1, 2).contiguous()
    widths = [d.c_out[l] for l in range(d.num_layers)]
    rows = B * P * ns
    z = [torch.empty((rows, c), device=cuda) for c in widths]
    stats = torch.empty((len(widths), sa_train.STAT_ROWS, sa_train.MAX_WIDTH), device=cuda)
    chosen = torch.empty((B * P, widths[-1]), dtype=torch.uint8, device=cuda)
    out = torch.empty((B, widths[-1], P), device=cuda)
    ws = torch.empty(L.prb_sa_train_workspace_bytes(B, P, ns, c_feat, ctypes.byref(d), 1), dtype=torch.uint8, device=cuda)
    C.check(L.prb_sa_train_forward(ctypes.byref(d), B, N, P, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm), C.ptr(idx), _ptrs(z),
                                   C.ptr(stats), C.ptr(chosen), C.ptr(out), None, widths[-1], 0, C.ptr(ws), ws.numel(), s), "sa_train_forward")
    gout = case["grad_out"].to(cuda).contiguous()

    def backward(entry, ws, gf):
        gw = [torch.empty((c, ci), device=cuda) for c, ci in zip(widths, [3 + c_feat] + widths[:-1])]
        gb = [torch.empty(c, device=cuda) for c in widths]
        C.check(entry(ctypes.byref(d), B, N, P, ns, c_feat, C.ptr(xyz), C.ptr(centres), C.ptr(feats_pm), C.ptr(idx), _ptrs(z), C.ptr(stats),
                      C.ptr(chosen), C.ptr(gout), widths[-1], 0, _ptrs(gw), _ptrs(gb), None, None, C.ptr(gf), C.ptr(ws), ws.numel(), s), "backward")
        return gw, gf

    gw_a, gf_a = backward(L.prb_sa_train_backward, ws, torch.zeros((B, c_feat, N), device=cuda))
    wsd = torch.empty(L.prb_sa_train_det_workspace_bytes(B, N, P, ns, c_feat, ctypes.byref(d)), dtype=torch.uint8, device=cuda)
    det = [backward(L.prb_sa_train_backward_det, wsd, torch.full((B, c_feat, N), float("nan"), device=cuda)) for _ in range(reps)]
    return gf_a, [g for _, g in det], [w for w, _ in det], gw_a


SA_INTEGER_CASES = {
    # name: (B, N, npoint, ns, c_feat, widths)
    "small_c_feat_29": (2, 300, 37, 8, 29, [40, 63, 64]),
    "rpn_sa1_ns32": (16, 16384, 4096, 32, 1, [32, 32, 64]),
    "rcnn_sa1_256_rois": (256, 512, 128, 64, 128, [128, 128, 128]),
}


@pytest.mark.parametrize("name", list(SA_INTEGER_CASES))
def test_sa_train_backward_det_exact_on_integer_cases(cuda, name):
    B, N, P, ns, c_feat, widths = SA_INTEGER_CASES[name]
    case = R.integer_case(B, N, P, ns, c_feat, widths, seed=len(name))
    ref = R.scale(case["xyz"], case["centres"], case["feats"], case["idx"], case["layers"], case["grad_out"], device=cuda)
    R.check_exact(case, ref)
    gf_a, gf_d, gw_d, gw_a = _sa_run(case, cuda)
    want = (ref["feats"].float() + 0.0).cpu().numpy()
    for gf in gf_d:
        _bits_equal(gf.cpu().numpy() + np.float32(0.0), want)
    _bits_equal(gf_a.cpu().numpy() + np.float32(0.0), want)
    for a, b in zip(gw_a, gw_d[0]):
        _bits_equal(b.cpu().numpy(), a.cpu().numpy())


def test_sa_train_backward_det_repeats_bits_on_float_data(cuda):
    """random float inputs: the ordered entry gives the same bits on every call, unlike a scatter with atomics"""
    case = R.integer_case(4, 2000, 512, 32, 7, [32, 48], seed=3)
    g = torch.Generator().manual_seed(8)
    case["feats"] = torch.randn(case["feats"].shape, generator=g)
    case["grad_out"] = torch.randn(case["grad_out"].shape, generator=g)
    for lay in case["layers"]:
        lay["w"] = lay["w"] * torch.rand(lay["w"].shape, generator=g, dtype=lay["w"].dtype)
    _, gf_d, gw_d, _ = _sa_run(case, cuda, reps=3)
    for gf in gf_d[1:]:
        _bits_equal(gf.cpu().numpy(), gf_d[0].cpu().numpy())
    assert torch.isfinite(gf_d[0]).all() and gf_d[0].abs().sum() > 0


def _run_deterministic(fn, *args):
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        return fn(*args)
    finally:
        torch.use_deterministic_algorithms(was, warn_only=warn)


@pytest.mark.parametrize("name", ["rpn_sa2_96", "rcnn_sa1", "sparse_padding", "two_layers"])
def test_sa_module_under_the_flag_within_the_float64_tolerances(cuda, name):
    """the module path of test_gpu_sa_train with the flag on (the ordered backward): every ratio within the same bounds,
    and the feature gradient the same bits on a second backward.  The float64 reference runs with the flag off."""
    import copy
    import test_gpu_sa_train as T
    m, xyz, feats = T._setup(name, cuda)
    m0 = copy.deepcopy(m)
    m1 = copy.deepcopy(m)
    new_xyz, out, gout, dec = _run_deterministic(T._run, m, xyz, feats)
    ratios = T._reference(m0, m, xyz, feats, new_xyz, out, gout, dec)
    ratios["feats"] = T._feature_grad_ratio(m0, m, xyz, feats, new_xyz, gout, dec)
    worst = max(ratios, key=ratios.get)
    assert ratios[worst] <= 1.0, (worst, ratios)
    first = feats.grad.clone()
    feats.grad = None
    _run_deterministic(T._run, m1, xyz, feats, gout)
    _bits_equal(feats.grad.cpu().numpy(), first.cpu().numpy())


def test_sa_train_backward_det_does_not_synchronise(cuda, deterministic):
    import test_gpu_sa_train as T
    m, xyz, feats = T._setup("rpn_sa2_96", cuda)
    from pointrcnn_b200 import config
    with config.override(sa_train="device"):
        _, out = m._forward_train(xyz, feats, None)
    gout = torch.randn(out.shape, device=cuda)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out.backward(gout)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert torch.isfinite(feats.grad).all()


# ------------------------------------------------------------------------------------------ two seeded training runs
def _state_digest(tr):
    h = hashlib.sha256()
    for p in tr.params:
        h.update(p.detach().cpu().numpy().tobytes())
    for b in tr.model.buffers():
        h.update(b.detach().cpu().numpy().tobytes())
    for p in tr.params:
        for k, v in sorted(tr.opt.state.get(p, {}).items()):
            if torch.is_tensor(v):
                h.update(v.detach().cpu().numpy().tobytes())
    return h.hexdigest()


def _worker():
    """two runs of three RPN steps and three RCNN step_jit steps from the same seed and batches, flag on -> JSON digests"""
    import synth
    from oracle import rcnn_offline as RO
    from pointrcnn_b200.datasets.rcnn_offline import RCNNOfflineSampler
    from pointrcnn_b200.train.step import RCNNTrainer, RPNTrainer, synthetic_labels
    torch.use_deterministic_algorithms(True)
    dev = torch.device("cuda:0")
    pc = torch.from_numpy(synth.u_kitti(2, 16384, 123, channels=4)).to(dev)
    cls, reg = synthetic_labels(pc, seed=1)
    scenes = [RO.synth_scene(s, k, n_feat=128) for s, k in ((51, "mixed"), (52, "hard"))]
    batch = RCNNOfflineSampler(device=dev).prepare_jit_batch(scenes)
    res = {"rpn": [], "rcnn": []}
    for _ in range(2):
        tr = RPNTrainer(input_channels=1, device=dev, world=1, seed=3, loss_impl="device", sa_train="device", fp_train="device")
        for _ in range(3):
            tr.step(pc, cls, reg, grad_norm_clip=1.0)
        res["rpn"].append(_state_digest(tr))
        tr = RCNNTrainer(device=dev, seed=5, target_draw="device", loss_impl="device")
        for _ in range(3):
            tr.step_jit(batch, grad_norm_clip=1.0)
        res["rcnn"].append(_state_digest(tr))
    print("DIGESTS " + json.dumps(res))


def test_two_seeded_training_runs_end_with_the_same_bits(cuda):
    env = dict(os.environ, CUBLAS_WORKSPACE_CONFIG=":4096:8",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--worker"], capture_output=True, text=True, env=env, timeout=900)
    assert r.returncode == 0, (r.stdout + r.stderr)[-4000:]
    line = [l for l in r.stdout.splitlines() if l.startswith("DIGESTS ")][-1]
    res = json.loads(line[len("DIGESTS "):])
    assert res["rpn"][0] == res["rpn"][1], "RPNTrainer: two seeded runs differ"
    assert res["rcnn"][0] == res["rcnn"][1], "RCNNTrainer.step_jit: two seeded runs differ"


if __name__ == "__main__" and "--worker" in sys.argv:
    _worker()
