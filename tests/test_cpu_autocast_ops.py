"""The bfloat16 grouping / gather / interpolation natives without a GPU: a numpy restatement of the rules the header states
(include/pointrcnn_b200.h, the *_bf16 entries) -- the forward copies, the fp32 interpolation in the fp32 kernel's order
rounded once, the ordered fp32 gradient sums rounded once, and the bound of the atomic gradients -- checked against
exact arithmetic and against mutants it must tell apart (rounding per term, summing in bfloat16, another order); and the
Python dispatch: float32 data reaches the float32 entries, bfloat16 data the _bf16 ones (ordered under the deterministic
flag), any other dtype raises.

test_gpu_autocast.py compares the device entries with these functions bit for bit."""
import contextlib
from fractions import Fraction

import numpy as np
import pytest
import torch

from test_cpu_deterministic_grads import _FakeLib, _padded_idx, _scatter64, group_grad_ref, interp_grad_ref
from pointrcnn_b200 import _cabi as C
from pointrcnn_b200.ext import pointnet2_cuda


# ------------------------------------------------------------------------------------------ the restatement
def bf16_bits(x):
    """float32 -> bfloat16 bit patterns (uint16), rounded to nearest even; NaN stays NaN"""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.asarray(x, np.float32))
    return np.where(nan, ((b >> 16) | 0x40).astype(np.uint16), r)


def bf16_value(bits):
    """bfloat16 bit patterns -> their exact float32 values"""
    return (np.asarray(bits, np.uint16).astype(np.uint32) << 16).view(np.float32)


def add_rn32(a, b):
    """fl32(a + b) for float64 arrays a, b: the float64 sum rounded to odd (exact sum + TwoSum error), then to float32 --
    one correct rounding of the exact sum"""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    s = a + b
    bb = s - a
    e = (a - (s - bb)) + (b - bb)
    even = (s.view(np.int64) & 1) == 0
    s = np.where((e != 0) & even, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def fma32(a, b, c):
    """fmaf(a, b, c) for float32 a, c and a bfloat16-valued b: a * b is exact in float64 (24 + 8 significant bits)"""
    return add_rn32(np.asarray(a, np.float32).astype(np.float64) * np.asarray(b, np.float32), np.asarray(c, np.float32))


def group_bf16_ref(points, idx):
    """prb_group_points_bf16: points (b, c, n) bit patterns, idx (b, npoints, nsample) -> (b, c, npoints, nsample), a copy"""
    b, c, _ = points.shape
    flat = np.asarray(idx, np.int64).reshape(b, 1, -1)
    return np.take_along_axis(points, np.broadcast_to(flat, (b, c, flat.shape[2])), axis=2).reshape((b, c) + idx.shape[1:])


def gather_bf16_ref(points, idx):
    """prb_gather_points_bf16: idx (b, npoints)"""
    return group_bf16_ref(points, idx)


def interp_f32(points, idx, weight):
    """the fp32 value before the rounding: fmaf(w2, f2, fmaf(w0, f0, w1 * f1)) -> (b, c, n) float32"""
    f = bf16_value(points)
    b, c, _ = f.shape
    n = idx.shape[1]
    g = np.take_along_axis(f, np.broadcast_to(np.asarray(idx, np.int64).reshape(b, 1, 3 * n), (b, c, 3 * n)), axis=2).reshape(b, c, n, 3)
    w = np.asarray(weight, np.float32)[:, None, :, :]
    t = (w[..., 1].astype(np.float64) * g[..., 1]).astype(np.float32)
    return fma32(w[..., 2], g[..., 2], fma32(w[..., 0], g[..., 0], t))


def interp_bf16_ref(points, idx, weight):
    """prb_three_interpolate_bf16: points (b, c, m) bit patterns, idx / weight (b, n, 3) -> (b, c, n) bit patterns"""
    return bf16_bits(interp_f32(points, idx, weight))


def group_grad_bf16_ref(grad_out, idx, n):
    """prb_group_points_grad_bf16_ws / prb_gather_points_grad_bf16_ws: the ordered fp32 sums of the exact values, rounded once"""
    return bf16_bits(group_grad_ref(bf16_value(grad_out), idx, n))


def interp_grad_bf16_ref(grad_out, idx, weight, m):
    """prb_three_interpolate_grad_bf16_ws: the ordered fp32 sums of the fp32 products, rounded once"""
    return bf16_bits(interp_grad_ref(bf16_value(grad_out), idx, weight, m))


def _group_vals(grad_out, idx):
    b, c = grad_out.shape[:2]
    return bf16_value(grad_out).reshape(b, c, -1).transpose(0, 2, 1), np.asarray(idx).reshape(b, -1)


def _interp_vals(grad_out, idx, weight):
    g = bf16_value(grad_out)
    b, c, n = g.shape
    vals = g.transpose(0, 2, 1)[:, :, None, :] * np.asarray(weight, np.float32)[:, :, :, None]
    return vals.reshape(b, 3 * n, c), np.asarray(idx).reshape(b, 3 * n)


def atomic_interval(vals, src, n):
    """the bfloat16 results the atomic entries may give: the fp32 sum of a source's k references lies within
    (k - 1) * 2^-24 * sum |v| (+ the (1 - (k - 1) u) slack of the recursive-summation bound) of the exact sum S, and
    rounding float64 -> float32 -> bfloat16 is monotone, so the result lies in [rn(S - bound), rn(S + bound)].
    vals (b, L, c) float32, src (b, L) -> (lo, hi) bit patterns (b, c, n)"""
    exact = _scatter64(vals, src, n)
    k = np.stack([np.bincount(s[(s >= 0) & (s < n)], minlength=n) for s in src])[:, None, :]
    u = 2.0 ** -24
    km = np.maximum(k - 1, 0)
    bound = km * u / (1 - km * u) * _scatter64(np.abs(vals), src, n)
    return bf16_bits((exact - bound).astype(np.float32)), bf16_bits((exact + bound).astype(np.float32))


def within_bf16_interval(got, lo, hi):
    """got in [lo, hi] as bfloat16 values, elementwise"""
    g, a, b = bf16_value(got), bf16_value(lo), bf16_value(hi)
    return (a <= g) & (g <= b)


# ------------------------------------------------------------------------------------------ the restatement's parts
def test_rounding_matches_torch_bfloat16():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(200000).astype(np.float32) * np.float32(1e3),
                        np.array([0.0, -0.0, 1e-40, -1e-40, 3.4e38, -3.4e38, np.inf, -np.inf], np.float32),
                        # exact ties between two bfloat16 values (odd and even lower halves)
                        (np.arange(1, 2000, dtype=np.uint32) << 16 | 0x8000).view(np.float32)])
    want = torch.from_numpy(x).to(torch.bfloat16).view(torch.int16).numpy().view(np.uint16)
    assert np.array_equal(bf16_bits(x), want)
    assert np.array_equal(bf16_value(want), torch.from_numpy(want.view(np.int16)).view(torch.bfloat16).float().numpy())


def _fl32(q):
    """correct rounding of a Fraction to float32 (to nearest even)"""
    f = np.float32(float(q))                    # may round twice: fix it with the exact neighbours
    cands = [np.nextafter(f, np.float32(-np.inf)), f, np.nextafter(f, np.float32(np.inf))]
    best = min(cands, key=lambda c: (abs(Fraction(float(c)) - q), int(np.array(c, np.float32).view(np.uint32)) & 1))
    return np.float32(best)


def test_fma32_is_one_correct_rounding():
    rng = np.random.default_rng(1)
    a = rng.standard_normal(1200).astype(np.float32)
    b = bf16_value(bf16_bits(rng.standard_normal(1200).astype(np.float32)))
    # c close to -a*b: heavy cancellation, where a double rounding would show
    c = (-(a.astype(np.float64) * b) * (1 + rng.standard_normal(1200) * 2.0 ** -20)).astype(np.float32)
    c[:400] = rng.standard_normal(400).astype(np.float32) * np.float32(1e-6)
    got = fma32(a, b, c)
    want = np.array([_fl32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


# ------------------------------------------------------------------------------------------ the rules, and their mutants
def _interp_case(seed, b=2, c=16, m=300, n=2000):
    rng = np.random.default_rng(seed)
    points = bf16_bits(rng.standard_normal((b, c, m)).astype(np.float32))
    idx = rng.integers(0, m, (b, n, 3)).astype(np.int32)
    w = rng.random((b, n, 3)).astype(np.float32) + np.float32(0.01)
    return points, idx, (w / w.sum(2, keepdims=True)).astype(np.float32)


def test_group_and_gather_forward_are_copies():
    rng = np.random.default_rng(2)
    points = rng.integers(0, 1 << 16, (2, 5, 77)).astype(np.uint16)     # every bit pattern, NaNs included
    idx = _padded_idx(rng, 2, 13, 8, 77)
    out = group_bf16_ref(points, idx)
    assert out.shape == (2, 5, 13, 8)
    for s in range(2):
        for ch in range(5):
            assert np.array_equal(out[s, ch], points[s, ch][idx[s]])
    gidx = rng.integers(0, 77, (2, 9)).astype(np.int32)
    assert np.array_equal(gather_bf16_ref(points, gidx)[1, 3], points[1, 3][gidx[1]])


def test_interpolation_is_the_fp32_kernel_rounded_once():
    """against exact arithmetic: fl32(w2 f2 + fl32(w0 f0 + fl32(w1 f1))), then one rounding to bfloat16"""
    points, idx, w = _interp_case(3, b=1, c=2, m=50, n=150)
    f = bf16_value(points)
    got = interp_bf16_ref(points, idx, w)
    for ch in range(2):
        for j in range(150):
            k = idx[0, j]
            F = [Fraction(float(f[0, ch, kk])) for kk in k]
            W = [Fraction(float(x)) for x in w[0, j]]
            t = _fl32(W[1] * F[1])
            t = _fl32(W[0] * F[0] + Fraction(float(t)))
            t = _fl32(W[2] * F[2] + Fraction(float(t)))
            assert got[0, ch, j] == bf16_bits(np.float32(t)), (ch, j)


def test_interpolation_mutants_are_rejected():
    points, idx, w = _interp_case(4)
    ref, ref32 = interp_bf16_ref(points, idx, w), interp_f32(points, idx, w)
    f = bf16_value(points)
    b, c, _ = f.shape
    n = idx.shape[1]
    g = np.take_along_axis(f, np.broadcast_to(idx.reshape(b, 1, 3 * n).astype(np.int64), (b, c, 3 * n)), axis=2).reshape(b, c, n, 3)
    wv = w[:, None]
    prod = [(wv[..., t].astype(np.float64) * g[..., t]).astype(np.float32) for t in range(3)]
    # rounding every term to bfloat16 before the sum
    r = [bf16_value(bf16_bits(p)) for p in prod]
    assert (bf16_bits(r[0] + r[1] + r[2]) != ref).any()
    # summing in bfloat16
    s = bf16_value(bf16_bits(bf16_value(bf16_bits(prod[1] + prod[0])) + prod[2]))
    assert (bf16_bits(s) != ref).any()
    # another order or contraction: the fp32 value the rounding starts from differs
    assert (fma32(wv[..., 0], g[..., 0], fma32(wv[..., 1], g[..., 1], prod[2])) != ref32).any()
    assert ((prod[0] + prod[1] + prod[2]) != ref32).any()


def _group_grad_case(seed, b=2, c=6, n=60, npoint=400, ns=16):
    rng = np.random.default_rng(seed)
    idx = _padded_idx(rng, b, npoint, ns, n)
    g = bf16_bits(rng.standard_normal((b, c, npoint, ns)).astype(np.float32))
    return g, idx, n


def test_ordered_gradients_sum_in_fp32_then_round_once():
    g, idx, n = _group_grad_case(5)
    got = group_grad_bf16_ref(g, idx, n)
    vals, src = _group_vals(g, idx)
    exact = _scatter64(vals, src, n)
    # the fp32 sum is within the recursive-summation bound of the exact one, and the result is that sum rounded once
    lo, hi = atomic_interval(vals, src, n)
    assert within_bf16_interval(got, lo, hi).all()
    assert np.abs(bf16_value(got) - exact).max() <= 2.0 ** -8 * np.abs(exact).max() + 1e-6
    points, ti, tw = _interp_case(6, m=120, n=500)
    gi = bf16_bits(np.random.default_rng(7).standard_normal((2, 16, 500)).astype(np.float32))
    got = interp_grad_bf16_ref(gi, ti, tw, 120)
    lo, hi = atomic_interval(*_interp_vals(gi, ti, tw), 120)
    assert within_bf16_interval(got, lo, hi).all()


def test_gradient_mutants_are_rejected():
    g, idx, n = _group_grad_case(8, n=20, npoint=600, ns=32)     # long reference lists: every point ~1000 references
    ref = group_grad_bf16_ref(g, idx, n)
    vals, src = _group_vals(g, idx)
    # rounding every value's running sum to bfloat16 (a bfloat16 accumulator)
    b, L, c = vals.shape
    acc = np.zeros((b, c, n), np.float32)
    for q in range(L):
        for s in range(b):
            acc[s, :, src[s, q]] = bf16_value(bf16_bits(acc[s, :, src[s, q]] + vals[s, q]))
    assert (bf16_bits(acc) != ref).any()
    # the references in decreasing order: the fp32 sum the rounding starts from differs
    rev = group_grad_ref(bf16_value(g).reshape(b, c, -1)[:, :, ::-1], idx.reshape(b, -1)[:, ::-1], n)
    assert (rev != group_grad_ref(bf16_value(g), idx, n)).any()
    # an fp32 sum added into a bfloat16 buffer that already holds a rounded partial sum (two roundings)
    half = L // 2
    first = bf16_bits(group_grad_ref(bf16_value(g).reshape(b, c, -1)[:, :, :half], idx.reshape(b, -1)[:, :half], n))
    second = group_grad_ref(bf16_value(g).reshape(b, c, -1)[:, :, half:], idx.reshape(b, -1)[:, half:], n)
    assert (bf16_bits(bf16_value(first) + second) != ref).any()


def test_atomic_interval_rejects_a_bfloat16_accumulator():
    """the stated bound is tight enough to catch summing in bfloat16 at the training list lengths"""
    g, idx, n = _group_grad_case(9, n=20, npoint=600, ns=32)
    vals, src = _group_vals(g, idx)
    lo, hi = atomic_interval(vals, src, n)
    b, L, c = vals.shape
    acc = np.zeros((b, c, n), np.float32)
    for q in range(L):
        for s in range(b):
            acc[s, :, src[s, q]] = bf16_value(bf16_bits(acc[s, :, src[s, q]] + vals[s, q]))
    assert not within_bf16_interval(bf16_bits(acc), lo, hi).all()


# ------------------------------------------------------------------------------------------ the dispatch
@pytest.fixture
def fake_lib(monkeypatch):
    lib = _FakeLib()
    monkeypatch.setattr(C, "lib", lambda: lib)
    monkeypatch.setattr(C, "require_cuda", lambda *t: None)
    monkeypatch.setattr(C, "stream", lambda: None)
    monkeypatch.setattr(pointnet2_cuda, "_guard", lambda t: contextlib.nullcontext())
    return lib


@pytest.fixture
def det_flag():
    was, warn = torch.are_deterministic_algorithms_enabled(), torch.is_deterministic_algorithms_warn_only_enabled()
    yield lambda on: torch.use_deterministic_algorithms(on)
    torch.use_deterministic_algorithms(was, warn_only=warn)


def _forward_calls(dtype):
    b, c, n, P, S = 1, 2, 8, 3, 4
    i3 = torch.zeros(b * P * S, dtype=torch.int32)
    pointnet2_cuda.group_points_wrapper(b, c, n, P, S, torch.zeros(b * c * n, dtype=dtype), i3, torch.zeros(b * c * P * S, dtype=dtype))
    pointnet2_cuda.gather_points_wrapper(b, c, n, P, torch.zeros(b * c * n, dtype=dtype), torch.zeros(b * P, dtype=torch.int32),
                                         torch.zeros(b * c * P, dtype=dtype))
    pointnet2_cuda.three_interpolate_wrapper(b, c, n, P, torch.zeros(b * c * n, dtype=dtype), torch.zeros(b * P * 3, dtype=torch.int32),
                                             torch.zeros(b * P * 3), torch.zeros(b * c * P, dtype=dtype))


def _grad_calls(dtype):
    b, c, n, P, S = 1, 2, 8, 3, 4
    g = torch.zeros(b * c * P * S, dtype=dtype)
    pointnet2_cuda.group_points_grad_wrapper(b, c, n, P, S, g, torch.zeros(b * P * S, dtype=torch.int32), torch.zeros(b * c * n, dtype=dtype))
    pointnet2_cuda.gather_points_grad_wrapper(b, c, n, P, g, torch.zeros(b * P, dtype=torch.int32), torch.zeros(b * c * n, dtype=dtype))
    pointnet2_cuda.three_interpolate_grad_wrapper(b, c, P, n, g, torch.zeros(b * P * 3, dtype=torch.int32), torch.zeros(b * P * 3),
                                                  torch.zeros(b * c * n, dtype=dtype))


def test_float32_data_takes_the_float32_entries(fake_lib, det_flag):
    det_flag(False)
    _forward_calls(torch.float32)
    _grad_calls(torch.float32)
    assert fake_lib.calls == ["prb_group_points", "prb_gather_points", "prb_three_interpolate", "prb_group_points_grad",
                              "prb_gather_points_grad", "prb_three_interpolate_grad"]


@pytest.mark.parametrize("ordered", [False, True])
def test_bfloat16_data_takes_the_bf16_entries(fake_lib, det_flag, ordered):
    det_flag(ordered)
    _forward_calls(torch.bfloat16)
    _grad_calls(torch.bfloat16)
    names = [k for k in fake_lib.calls if not k.endswith("_workspace_bytes")]
    grads = ["prb_group_points_grad_bf16", "prb_gather_points_grad_bf16", "prb_three_interpolate_grad_bf16"]
    assert names == ["prb_group_points_bf16", "prb_gather_points_bf16", "prb_three_interpolate_bf16"] + [k + "_ws" * ordered for k in grads]
    sizes = [k for k in fake_lib.calls if k.endswith("_workspace_bytes")]
    assert sizes == (["prb_group_points_grad_workspace_bytes", "prb_gather_points_grad_workspace_bytes",
                      "prb_three_interpolate_grad_workspace_bytes"] if ordered else
                     ["prb_group_points_grad_bf16_workspace_bytes", "prb_group_points_grad_bf16_workspace_bytes",
                      "prb_three_interpolate_grad_bf16_workspace_bytes"])


def test_other_dtypes_still_raise(fake_lib):
    for dtype in (torch.float16, torch.float64):
        with pytest.raises(RuntimeError, match="float32 or bfloat16"):
            _forward_calls(dtype)
        with pytest.raises(RuntimeError, match="float32 or bfloat16"):
            _grad_calls(dtype)
    assert fake_lib.calls == []


def test_mixed_bfloat16_and_float32_buffers_raise(fake_lib):
    """bfloat16 features need bfloat16 outputs: the reference's own callers, which allocate float32 outputs, get an error"""
    with pytest.raises(RuntimeError, match="bfloat16"):
        pointnet2_cuda.group_points_wrapper(1, 2, 8, 3, 4, torch.zeros(16, dtype=torch.bfloat16), torch.zeros(12, dtype=torch.int32),
                                            torch.zeros(24))
    assert fake_lib.calls == []
