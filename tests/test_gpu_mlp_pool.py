"""The SA max-pool of the chain kernels, bit for bit: resident against streaming, and both against goldens.

Both chain kernels max-pool an SA centre from the accumulator registers (warp shuffles; per-warp maxima behind one barrier
for a centre of 32 or more rows), and the resident kernel runs two 64-row tiles per warpgroup where every layer is at most
64 wide.  These cases cover the centre sizes (4 .. 128 samples), odd tile counts and partial last pairs, and chains whose
last layer yields exact zeros of both signs: max is independent of order except for the sign of zero, so those pin the
pooling order.  Outputs are compared as int32 bit patterns (torch.equal treats -0.0 and +0.0 as equal).
"""
import ctypes
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.mlp_chain import Chain  # noqa: E402

SENTINEL = -7.0   # outputs a kernel does not write keep this value in both runs
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "sa_pool.npz")


def _both(run):
    """run(): list of output tensors; returns (resident outputs, streaming outputs)"""
    outs = []
    for resident in (1, 0):
        with C.options(mlp_resident=resident):
            outs.append([t.clone() for t in run()])
        torch.cuda.synchronize()
    return outs


def _assert_bits(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32)), \
            "outputs differ in %d words" % (x.view(torch.int32) != y.view(torch.int32)).sum().item()


def _sa_run(cuda, b, n, npoint, ns, c_feat, ch, feats_np, rng):
    """seeded SA inputs for chain ch; returns run() -> [out (b, C, npoint), out_pm (b, npoint, C)]"""
    lib = C.lib()
    xyz = torch.from_numpy(rng.uniform(-1, 1, (b, n, 3)).astype(np.float32)).to(cuda)
    new_xyz = torch.from_numpy(rng.uniform(-1, 1, (b, npoint, 3)).astype(np.float32)).to(cuda)
    feats = torch.from_numpy(feats_np(rng, (b, n, c_feat)).astype(np.float32)).to(cuda) if c_feat else None
    idx = torch.from_numpy(rng.integers(0, n, (b, npoint, ns)).astype(np.int32)).to(cuda)
    C_out = ch.c_out[-1]
    out = torch.empty((b, C_out, npoint), device=cuda)
    out_pm = torch.empty((b, npoint, C_out), device=cuda)
    wsb = lib.prb_sa_workspace_bytes(b, npoint, ns, c_feat, len(ch.c_out), ch.co)
    wsp = torch.empty(max(wsb, 1), dtype=torch.uint8, device=cuda)

    def run():
        out.fill_(SENTINEL); out_pm.fill_(SENTINEL)
        C.check(lib.prb_sa_group_mlp_max_ws(b, n, npoint, ns, c_feat, C.ptr(xyz), C.ptr(new_xyz), C.ptr(feats), C.ptr(idx),
                                            ctypes.byref(ch.desc), C.ptr(out), C.ptr(out_pm), C_out, 0, C.ptr(wsp),
                                            C.c_size_t(wsb), C.stream()), "sa_group_mlp_max")
        return [out, out_pm]
    run.chain = ch   # keeps the packed weights alive with the closure
    return run


POOL_CASES = [
    # b, n, npoint, ns, c_feat, c_out
    (2, 600, 101, 4, 1, [16, 16, 32]),        # four samples per centre; 13 tiles, the last pair one partial tile
    (2, 600, 84, 8, 1, [32, 32, 64]),         # eight samples per centre; 21 full tiles, an odd count
    (2, 600, 86, 8, 1, [32, 32, 64]),         # 22 tiles, the second tile of the last pair partial
    (3, 700, 42, 32, 1, [32, 32, 64]),        # 63 full tiles, an odd count
    (2, 500, 29, 128, 1, [32, 32, 64]),       # two tiles per centre on a 64-wide chain: one pair per centre
    (2, 500, 45, 64, 8, [32, 64]),            # one centre per tile, a pair of centres
    (2, 300, 37, 16, 96, [64, 96, 128]),      # one tile per warpgroup, 128 wide
]


@pytest.mark.parametrize("folded", [True, False])
@pytest.mark.parametrize("b,n,npoint,ns,c_feat,c_out", POOL_CASES)
def test_sa_pool_resident_bits(cuda, b, n, npoint, ns, c_feat, c_out, folded):
    rng = np.random.default_rng(b * 1000 + ns + c_feat + npoint)
    dims = [3 + c_feat] + list(c_out)
    ws = [(rng.standard_normal((co, ci)) * np.sqrt(2.0 / ci)).astype(np.float32) for ci, co in zip(dims[:-1], dims[1:])]
    scale = [rng.uniform(0.5, 1.5, co).astype(np.float32) for co in c_out]
    shift = [rng.normal(0, 0.2, co).astype(np.float32) for co in c_out]
    ch = Chain(0, c_feat, ws, shift, None if folded else scale, device=cuda)
    res, stream = _both(_sa_run(cuda, b, n, npoint, ns, c_feat, ch, lambda r, s: r.standard_normal(s), rng))
    assert (res[0] != SENTINEL).all()
    _assert_bits(res, stream)
    _assert_bits([res[1]], [res[0].transpose(1, 2)])


# The tensor cores return +0 for a zero sum, so the signs of zero come from the epilogue: channel c of the last layer has,
# by c % 4, one positive weight on an input that is zero for about half of the samples (a ReLU output, or a clipped
# feature on a one-layer chain) with a negative scale and shift -0 (samples give -0 or a negative value), the same with
# shift +0 (+0 or negative), all-zero weights with a negative scale and shift -0 (-0 everywhere), random weights and shift.
ZERO_CASES = [
    # b, n, npoint, ns, c_feat, c_out
    (2, 600, 36, 8, 1, [32]),                 # 9 tiles: an odd count
    (2, 600, 38, 16, 1, [16, 32]),            # 19 tiles, an inner layer before the zeros
    (2, 500, 13, 128, 1, [32, 64]),           # two tiles per centre: the zeros pass through the carried partial maxima
    (2, 777, 37, 32, 1, [32, 32, 128]),       # a 128-wide last layer
]


def golden_key(case, folded, linear):
    return "%s_%s_%s" % ("_".join(str(v) for v in case[:5]) + "_" + "-".join(str(c) for c in case[5]),
                         "folded" if folded else "scaled", "linear" if linear else "relu")


def sa_signed_zero_run(cuda, case, folded, linear):
    """the ZERO_CASES chain on seeded inputs; returns run() -> [out (b, C, npoint), out_pm (b, npoint, C)]"""
    b, n, npoint, ns, c_feat, c_out = case
    rng = np.random.default_rng(b * 1000 + ns + len(c_out))
    dims = [3 + c_feat] + list(c_out)
    ws = [(rng.standard_normal((co, ci)) * np.sqrt(2.0 / ci)).astype(np.float32) for ci, co in zip(dims[:-1], dims[1:])]
    scale = [rng.uniform(0.5, 1.5, co).astype(np.float32) for co in c_out]
    shift = [rng.normal(0, 0.2, co).astype(np.float32) for co in c_out]
    k = 3 if len(c_out) == 1 else 0            # the clipped feature, or an inner ReLU channel
    ws[-1][0::4] = 0.0
    ws[-1][1::4] = 0.0
    ws[-1][2::4] = 0.0
    ws[-1][0::4, k] = 1.0
    ws[-1][1::4, k] = 1.0
    scale[-1][0::4] *= -1.0
    scale[-1][1::4] *= -1.0
    scale[-1][2::4] *= -1.0
    shift[-1][0::4] = -0.0
    shift[-1][1::4] = 0.0
    shift[-1][2::4] = -0.0
    ch = Chain(0, c_feat, ws, shift, None if folded else scale, linear_last=linear, device=cuda)
    return _sa_run(cuda, b, n, npoint, ns, c_feat, ch, lambda r, s: np.maximum(r.standard_normal(s), 0), rng)


@pytest.mark.parametrize("linear", [False, True])
@pytest.mark.parametrize("folded", [True, False])
@pytest.mark.parametrize("case", ZERO_CASES)
def test_sa_signed_zero_bits(cuda, case, folded, linear):
    """resident against streaming, and both against the outputs of the staged shared-memory pool they replaced"""
    res, stream = _both(sa_signed_zero_run(cuda, case, folded, linear))
    assert (res[0] != SENTINEL).all()
    out = res[0].view(torch.int32).cpu().numpy()
    if linear and not folded:
        assert (out == -2 ** 31).any() and (out == 0).any(), "the case yields zeros of both signs"
    _assert_bits(res, stream)
    _assert_bits([res[1]], [res[0].transpose(1, 2)])
    gold = np.load(GOLDEN)[golden_key(case, folded, linear)]
    assert np.array_equal(out, gold), "SA pool differs from the golden in %d words" % (out != gold).sum()
