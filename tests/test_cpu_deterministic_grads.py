"""The ordered (deterministic) gradient scatters without a GPU: a float32 numpy restatement of the summation order the
header documents (include/pointrcnn_b200.h, prb_group_points_grad_ws), checked against a float64 scatter, and the Python
dispatch: the shims and the SA training backward take the ordered entries exactly when torch's deterministic mode is on.

test_gpu_deterministic_grads.py compares the device entries with ordered_segment_sum bit for bit."""
import contextlib
import types

import numpy as np
import pytest
import torch

from pointrcnn_b200 import _cabi as C
from pointrcnn_b200.ext import pointnet2_cuda
from pointrcnn_b200.pointnet2 import pointnet2_utils as pu
from pointrcnn_b200.pointnet2 import sa_train


# ------------------------------------------------------------------------------------------ the restatement
def ordered_segment_sum(vals, src, n, out=None):
    """vals (b, L, c) float32: the value of every reference in every channel; src (b, L): the source point each reference
    names (outside [0, n): ignored).  -> (b, c, n) float32: for every source, acc = +0.0 and then acc = fl32(acc + v) over
    its references in increasing reference index; out + acc (one more rounding) when out (b, c, n) is given, else acc."""
    vals = np.asarray(vals, np.float32)
    b, L, c = vals.shape
    src = np.asarray(src, np.int64).reshape(b, L)
    keep = ((src >= 0) & (src < n)).reshape(-1)
    q = np.nonzero(keep)[0]
    key = (src + np.arange(b)[:, None] * n).reshape(-1)[q]
    order = np.argsort(key, kind="stable")          # by source; increasing reference index within a source
    q, key = q[order], key[order]
    counts = np.bincount(key, minlength=b * n)
    starts = np.concatenate([[0], np.cumsum(counts)[:-1]])
    v = vals.reshape(b * L, c)
    acc = np.zeros((b * n, c), np.float32)
    for r in range(int(counts.max()) if counts.size else 0):
        act = np.nonzero(counts > r)[0]
        acc[act] = acc[act] + v[q[starts[act] + r]]     # float32 + float32: one rounding per add
    res = np.ascontiguousarray(acc.reshape(b, n, c).transpose(0, 2, 1))
    return res if out is None else np.asarray(out, np.float32) + res


def group_grad_ref(grad_out, idx, n, out=None):
    """prb_group_points_grad_ws / prb_gather_points_grad_ws: grad_out (b, c, npoints, nsample) or (b, c, npoints), idx of the
    same trailing shape -> (b, c, n)"""
    b, c = grad_out.shape[:2]
    return ordered_segment_sum(np.asarray(grad_out, np.float32).reshape(b, c, -1).transpose(0, 2, 1), np.asarray(idx).reshape(b, -1), n, out)


def interp_grad_ref(grad_out, idx, weight, m, out=None):
    """prb_three_interpolate_grad_ws: grad_out (b, c, n), idx / weight (b, n, 3) -> (b, c, m); each value the fp32 product
    grad_out * weight, rounded before the add"""
    g = np.asarray(grad_out, np.float32)
    w = np.asarray(weight, np.float32)
    b, c, n = g.shape
    vals = g.transpose(0, 2, 1)[:, :, None, :] * w[:, :, :, None]        # (b, n, 3, c), float32 products
    return ordered_segment_sum(vals.reshape(b, 3 * n, c), np.asarray(idx).reshape(b, 3 * n), m, out)


def sa_feats_grad_ref(da_feats, idx, n):
    """prb_sa_train_backward_det's grad_feats from layer 0's feature gradient da_feats (rows, c_feat), rows in idx's flat
    order (b, npoint, nsample) -> (b, c_feat, n), written"""
    b = idx.shape[0]
    return ordered_segment_sum(np.asarray(da_feats, np.float32).reshape(b, -1, da_feats.shape[1]), np.asarray(idx).reshape(b, -1), n)


# ------------------------------------------------------------------------------------------ restatement vs float64
def _scatter64(vals, src, n):
    b, L, c = vals.shape
    out = np.zeros((b, n, c), np.float64)
    for s in range(b):
        ok = (src[s] >= 0) & (src[s] < n)
        np.add.at(out[s], src[s][ok], vals[s][ok].astype(np.float64))
    return out.transpose(0, 2, 1)


def _bound(vals, src, n):
    """|fl(sum) - sum| <= (k - 1) u / (1 - (k - 1) u) * sum |v| over a source's k references (recursive summation)"""
    k = np.stack([np.bincount(s[(s >= 0) & (s < n)], minlength=n) for s in src])[:, None, :]
    u = 2.0 ** -24
    return np.maximum(k - 1, 0) * u / (1 - np.maximum(k - 1, 0) * u) * _scatter64(np.abs(vals), src, n)


def _padded_idx(rng, b, npoint, ns, n):
    """ball-query-like idx: random hits per centre, padded with the first hit (skewed list lengths)"""
    idx = rng.integers(0, n, (b, npoint, ns))
    hits = rng.integers(1, ns + 1, (b, npoint, 1))
    return np.where(np.arange(ns) >= hits, idx[:, :, :1], idx).astype(np.int32)


@pytest.mark.parametrize("b,npoint,ns,n,c", [(2, 64, 16, 100, 5), (3, 40, 32, 30, 9), (1, 1, 64, 64, 3), (2, 50, 1, 200, 4)])
def test_group_restatement_is_a_rounded_scatter(b, npoint, ns, n, c):
    rng = np.random.default_rng(b * 100 + ns)
    idx = _padded_idx(rng, b, npoint, ns, n)
    g = rng.standard_normal((b, c, npoint, ns)).astype(np.float32)
    got = group_grad_ref(g, idx, n)
    vals = g.reshape(b, c, -1).transpose(0, 2, 1)
    src = idx.reshape(b, -1)
    exact = _scatter64(vals, src, n)
    assert (np.abs(got - exact) <= _bound(vals, src, n)).all()
    unused = np.ones((b, n), bool)
    for s in range(b):
        unused[s, src[s]] = False
    assert (got.transpose(0, 2, 1)[unused] == 0).all()


def test_interp_restatement_is_a_rounded_scatter():
    rng = np.random.default_rng(3)
    b, c, n, m = 2, 7, 300, 40
    idx = rng.integers(0, m, (b, n, 3)).astype(np.int32)
    idx[:, :5] = idx[:, :5, :1]                                # repeated taps
    w = rng.random((b, n, 3)).astype(np.float32)
    g = rng.standard_normal((b, c, n)).astype(np.float32)
    got = interp_grad_ref(g, idx, w, m)
    vals = (g.transpose(0, 2, 1)[:, :, None, :] * w[:, :, :, None]).reshape(b, 3 * n, c)
    src = idx.reshape(b, -1)
    exact = _scatter64((g.transpose(0, 2, 1)[:, :, None, :].astype(np.float64) * w[:, :, :, None]).reshape(b, 3 * n, c), src, m)
    # the products are rounded once each (u |g w|) before the recursive sum
    assert (np.abs(got - exact) <= _bound(vals, src, m) + 2.0 ** -24 * _scatter64(np.abs(vals), src, m) * 1.0001).all()


def test_restatement_order_is_increasing_reference_index():
    """four references of one point whose sum depends on the order"""
    vals = np.array([[[1.0], [2.0 ** -24], [2.0 ** -24], [-1.0]]], np.float32)
    got = ordered_segment_sum(vals, np.zeros((1, 4), np.int32), 1)
    # (((0 + 1) + u) + u) - 1 with u = 2^-24: each 1 + u ties to even 1, so the sum is 0; in reverse order
    # (((0 - 1) + u) + u) + 1 every add is exact and the sum is 2^-23
    assert got[0, 0, 0] == np.float32(0.0)
    rev = ordered_segment_sum(vals[:, ::-1], np.zeros((1, 4), np.int32), 1)
    assert rev[0, 0, 0] == np.float32(2.0 ** -23)
    acc = ordered_segment_sum(vals, np.zeros((1, 4), np.int32), 1, out=np.full((1, 1, 1), 5.0, np.float32))
    assert acc[0, 0, 0] == np.float32(5.0)


def test_restatement_ignores_out_of_range_and_handles_empty():
    vals = np.ones((1, 3, 2), np.float32)
    got = ordered_segment_sum(vals, np.array([[0, 5, -1]]), 2)
    assert got.tolist() == [[[1.0, 0.0], [1.0, 0.0]]]
    assert ordered_segment_sum(np.zeros((0, 4, 3), np.float32), np.zeros((0, 4), np.int32), 5).shape == (0, 3, 5)
    assert ordered_segment_sum(np.zeros((2, 0, 3), np.float32), np.zeros((2, 0), np.int32), 5).tolist() == np.zeros((2, 3, 5)).tolist()


# ------------------------------------------------------------------------------------------ the dispatch
@pytest.fixture
def det_mode():
    """sets torch's deterministic mode for a test and restores what it was"""
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()

    def set_mode(mode):
        torch.use_deterministic_algorithms(mode != "off", warn_only=mode == "warn_only")

    yield set_mode
    torch.use_deterministic_algorithms(was, warn_only=warn)


class _FakeLib:
    """records the C ABI entries the Python side calls; every entry succeeds, every size is 64 bytes"""

    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        if not name.startswith("prb_"):
            raise AttributeError(name)
        fn = self.calls.append

        def call(*args):
            fn(name)
            return 64 if name.endswith("_workspace_bytes") else 0
        return call


@pytest.fixture
def fake_lib(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(C, "lib", lambda: lib)
    monkeypatch.setattr(C, "require_cuda", lambda *t: None)
    monkeypatch.setattr(C, "stream", lambda: None)
    monkeypatch.setattr(pointnet2_cuda, "_guard", lambda t: contextlib.nullcontext())
    monkeypatch.setattr(torch.cuda, "device", lambda d: contextlib.nullcontext())
    return lib


MODES = [("off", False), ("on", True), ("warn_only", True)]


@pytest.mark.parametrize("mode,ordered", MODES)
def test_autograd_backwards_take_the_ordered_entries_exactly_under_the_flag(det_mode, fake_lib, mode, ordered):
    det_mode(mode)
    B, Cc, N, P, S = 2, 3, 10, 4, 5
    ctx = types.SimpleNamespace(for_backwards=(torch.zeros((B, P, S), dtype=torch.int32), N))
    pu.GroupingOperation.backward(ctx, torch.zeros((B, Cc, P, S)))
    ctx = types.SimpleNamespace(for_backwards=(torch.zeros((B, P), dtype=torch.int32), Cc, N))
    pu.GatherOperation.backward(ctx, torch.zeros((B, Cc, P)))
    ctx = types.SimpleNamespace(three_interpolate_for_backward=(torch.zeros((B, P, 3), dtype=torch.int32), torch.zeros((B, P, 3)), N))
    pu.ThreeInterpolate.backward(ctx, torch.zeros((B, Cc, P)))
    if ordered:
        want = ["prb_group_points_grad_workspace_bytes", "prb_group_points_grad_ws", "prb_gather_points_grad_workspace_bytes",
                "prb_gather_points_grad_ws", "prb_three_interpolate_grad_workspace_bytes", "prb_three_interpolate_grad_ws"]
    else:
        want = ["prb_group_points_grad", "prb_gather_points_grad", "prb_three_interpolate_grad"]
    assert fake_lib.calls == want


@pytest.mark.parametrize("mode,ordered", MODES)
def test_reference_named_shims_take_the_ordered_entries_exactly_under_the_flag(det_mode, fake_lib, mode, ordered):
    det_mode(mode)
    b, c, n, npoints, ns = 1, 2, 8, 3, 4
    g = torch.zeros(b * c * npoints * ns)
    pointnet2_cuda.group_points_grad_wrapper(b, c, n, npoints, ns, g, torch.zeros(b * npoints * ns, dtype=torch.int32), torch.zeros(b * c * n))
    pointnet2_cuda.gather_points_grad_wrapper(b, c, n, npoints, g, torch.zeros(b * npoints, dtype=torch.int32), torch.zeros(b * c * n))
    pointnet2_cuda.three_interpolate_grad_wrapper(b, c, npoints, n, g, torch.zeros(b * npoints * 3, dtype=torch.int32),
                                                  torch.zeros(b * npoints * 3), torch.zeros(b * c * n))
    names = [k for k in fake_lib.calls if not k.endswith("_workspace_bytes")]
    assert names == [("prb_%s_ws" if ordered else "prb_%s") % k for k in ("group_points_grad", "gather_points_grad", "three_interpolate_grad")]


@pytest.mark.parametrize("mode,ordered", MODES)
def test_sa_train_backward_takes_the_ordered_entry_exactly_under_the_flag(det_mode, fake_lib, mode, ordered):
    """two scales: each calls its backward entry; the ordered one sizes its scratch with the point count"""
    det_mode(mode)
    B, N, P, ns, c_feat = 2, 16, 4, 8, 2
    w = torch.zeros((4, 3 + c_feat, 1, 1), requires_grad=False)
    params = [w, torch.zeros(4), None, None] + [None] * 8
    scale = types.SimpleNamespace(c_out=[4])
    idx = torch.zeros((B, P, ns), dtype=torch.int32)
    z, stats, chosen = torch.zeros((B * P * ns, 4)), torch.zeros((1, 4, 512)), torch.zeros((B * P, 4), dtype=torch.uint8)
    saved = (torch.zeros((B, N, 3)), torch.zeros((B, P, 3)), torch.zeros((B, N, c_feat)), idx, idx) + tuple(params) * 2 + (z, stats, chosen) * 2
    ctx = types.SimpleNamespace(saved_tensors=saved, n_idx=2, scales=[scale, scale], nss=[ns, ns], descs=[C.SATrainDesc(), C.SATrainDesc()],
                                c_feat=c_feat, needs_input_grad=[False, False, False, True] + [True, True] + [False] * 10 + [True, True] + [False] * 10)
    g_out = torch.zeros((B, 8, P))
    res = sa_train._SATrain.backward(ctx, g_out, None)
    assert res[3].shape == (B, c_feat, N)
    if ordered:
        assert fake_lib.calls == ["prb_sa_train_det_workspace_bytes", "prb_sa_train_backward_det"] * 2
    else:
        assert fake_lib.calls == ["prb_sa_train_workspace_bytes", "prb_sa_train_backward"] * 2
