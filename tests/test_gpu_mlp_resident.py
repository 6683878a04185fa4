"""The resident-weight chain kernel against the streaming one, bit for bit.

Chains whose layers are at most 128 wide and whose packed weights fit in shared memory run, by default
(`prb_options.mlp_resident = 1`), on a kernel that loads the whole weight image once per CTA and runs one 64-row tile
per warpgroup.  With `mlp_resident = 0` every launch streams its weights.  Both kernels share the gather and epilogue
code and issue the same MMA sequence per K chunk, so every output must be identical.  (Images larger than half of a CTA's
shared memory, such as the FP0 chain and its projection below, stream under both settings.)
"""
import ctypes

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pointrcnn_b200 import _cabi as C  # noqa: E402
from pointrcnn_b200.mlp_chain import Chain  # noqa: E402

SENTINEL = -7.0   # outputs a kernel does not write keep this value in both runs


def _chain(rng, dev, kind, split, c_in, c_out, folded, linear_last=False):
    """random weights packed for the chain; folded: no separate scale (scale = NULL in the descriptor)"""
    dims = [c_in] + list(c_out)
    ws = [(rng.standard_normal((co, ci)) * np.sqrt(2.0 / ci)).astype(np.float32) for ci, co in zip(dims[:-1], dims[1:])]
    scale = [rng.uniform(0.5, 1.5, co).astype(np.float32) for co in c_out]
    shift = [rng.normal(0, 0.2, co).astype(np.float32) for co in c_out]
    return Chain(kind, split, ws, shift, None if folded else scale, linear_last=linear_last, device=dev)


def _both(run):
    """run(): list of output tensors; returns (resident outputs, streaming outputs)"""
    outs = []
    for resident in (1, 0):
        with C.options(mlp_resident=resident):
            outs.append([t.clone() for t in run()])
        torch.cuda.synchronize()
    return outs


def _assert_equal(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x, y), "resident and streaming outputs differ: max |d| = %g" % (x - y).abs().max().item()


SA_CASES = [
    # b, n, npoint, ns, c_feat, c_out
    (16, 4096, 512, 16, 1, [16, 16, 32]),     # SA1-like, every layer 32 wide
    (16, 4096, 512, 32, 1, [32, 32, 64]),     # SA1-like
    (4, 1024, 256, 16, 96, [64, 64, 128]),    # SA2-like
    (4, 1024, 256, 32, 96, [64, 96, 128]),    # SA2-like, a 96-wide inner layer
    (3, 777, 37, 16, 0, [32]),                # xyz only, one 32-wide layer, 37 centres: a partial last tile
    (2, 500, 45, 64, 8, [32, 64]),            # one centre per tile
    (2, 500, 29, 128, 6, [64, 64, 128]),      # two tiles per centre: partial maxima carried between them
]


@pytest.mark.parametrize("folded", [True, False])
@pytest.mark.parametrize("b,n,npoint,ns,c_feat,c_out", SA_CASES)
def test_sa_resident_bits(cuda, b, n, npoint, ns, c_feat, c_out, folded):
    rng = np.random.default_rng(b * 1000 + ns + c_feat)
    lib = C.lib()
    ch = _chain(rng, cuda, 0, c_feat, 3 + c_feat, c_out, folded)
    xyz = torch.from_numpy(rng.uniform(-1, 1, (b, n, 3)).astype(np.float32)).to(cuda)
    new_xyz = torch.from_numpy(rng.uniform(-1, 1, (b, npoint, 3)).astype(np.float32)).to(cuda)
    feats = torch.from_numpy(rng.standard_normal((b, n, c_feat)).astype(np.float32)).to(cuda) if c_feat else None
    idx = torch.from_numpy(rng.integers(0, n, (b, npoint, ns)).astype(np.int32)).to(cuda)
    C_out = c_out[-1]
    out = torch.empty((b, C_out, npoint), device=cuda)
    out_pm = torch.empty((b, npoint, C_out), device=cuda)
    wsb = lib.prb_sa_workspace_bytes(b, npoint, ns, c_feat, len(c_out), ch.co)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=cuda)

    def run():
        out.fill_(SENTINEL); out_pm.fill_(SENTINEL)
        C.check(lib.prb_sa_group_mlp_max_ws(b, n, npoint, ns, c_feat, C.ptr(xyz), C.ptr(new_xyz), C.ptr(feats), C.ptr(idx),
                                            ctypes.byref(ch.desc), C.ptr(out), C.ptr(out_pm), C_out, 0, C.ptr(ws), C.c_size_t(wsb),
                                            C.stream()), "sa_group_mlp_max")
        return [out, out_pm]

    res, stream = _both(run)
    assert (res[0] != SENTINEL).all()
    _assert_equal(res, stream)


FP_CASES = [
    # b, n, m, c_known, c_skip, c_out
    (16, 1000, 250, 128, 1, [128, 128]),      # FP0 after the projection: [interp 128 | skip 1]
    (4, 1000, 250, 64, 0, [64, 32]),          # no skip features
    (4, 999, 300, 70, 5, [96, 128]),          # c_known not a multiple of 4 (scalar gather), odd row count
]


@pytest.mark.parametrize("folded", [True, False])
@pytest.mark.parametrize("b,n,m,c_known,c_skip,c_out", FP_CASES)
def test_fp_resident_bits(cuda, b, n, m, c_known, c_skip, c_out, folded):
    rng = np.random.default_rng(n + c_known + c_skip)
    lib = C.lib()
    ch = _chain(rng, cuda, 1, c_known, c_known + c_skip, c_out, folded)
    known_pm = torch.from_numpy(rng.standard_normal((b, m, c_known)).astype(np.float32)).to(cuda)
    idx = torch.from_numpy(rng.integers(0, m, (b, n, 3)).astype(np.int32)).to(cuda)
    w = rng.uniform(0.1, 1.0, (b, n, 3)).astype(np.float32)
    weight = torch.from_numpy(w / w.sum(-1, keepdims=True)).to(cuda)
    skip = torch.from_numpy(rng.standard_normal((b, c_skip, n)).astype(np.float32)).to(cuda) if c_skip else None
    C_out = c_out[-1]
    out = torch.empty((b, C_out, n), device=cuda)
    out_pm = torch.empty((b, n, C_out), device=cuda)
    wsb = lib.prb_fp_workspace_bytes(b, n, c_known, c_skip, len(c_out), ch.co)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=cuda)

    def run():
        out.fill_(SENTINEL); out_pm.fill_(SENTINEL)
        C.check(lib.prb_fp_interp_mlp_ws(b, n, m, c_known, c_skip, C.ptr(known_pm), C.ptr(idx), C.ptr(weight), C.ptr(skip),
                                         ctypes.byref(ch.desc), C.ptr(out), C.ptr(out_pm), C.ptr(ws), C.c_size_t(wsb), C.stream()),
                "fp_interp_mlp")
        return [out, out_pm]

    res, stream = _both(run)
    assert (res[0] != SENTINEL).all()
    _assert_equal(res, stream)


ROW_CASES = [
    # rows, c_in, c_out, linear last layer
    (65536, 256, [128], True),                # the FP0 projection: 256 -> 128, linear, no shift beyond the bias
    (1000, 40, [48, 64], False),              # K and N not multiples of 32, a partial last tile
    (4097, 99, [64, 96, 128], False),         # three layers at the resident limit
    (130, 32, [32, 32, 32], True),            # 32 wide only, linear last layer
]


@pytest.mark.parametrize("folded", [True, False])
@pytest.mark.parametrize("rows,c_in,c_out,linear", ROW_CASES)
def test_rows_resident_bits(cuda, rows, c_in, c_out, linear, folded):
    rng = np.random.default_rng(rows + c_in)
    lib = C.lib()
    ch = _chain(rng, cuda, 2, 0, c_in, c_out, folded, linear_last=linear)
    x = torch.from_numpy(rng.standard_normal((rows, c_in)).astype(np.float32)).to(cuda)
    pitch = (c_out[-1] + 31) // 32 * 32
    out = torch.empty((rows, pitch), device=cuda)
    wsb = lib.prb_rows_workspace_bytes(C.c_long(rows), c_in, len(c_out), ch.co)
    ws = torch.empty(max(wsb, 1), dtype=torch.uint8, device=cuda)

    def run():
        out.fill_(SENTINEL)
        C.check(lib.prb_mlp_rows(C.c_long(rows), c_in, C.ptr(x), ctypes.byref(ch.desc), C.ptr(out), pitch, C.ptr(ws),
                                 C.c_size_t(wsb), C.stream()), "mlp_rows")
        return [out]

    res, stream = _both(run)
    assert (res[0] != SENTINEL).all()
    if linear:
        assert (res[0] < 0).any()   # the last layer kept its sign
    _assert_equal(res, stream)


def test_backbone_resident_bits(cuda):
    """the RPN backbone at its default widths: every chain launch, resident where it applies, against streaming"""
    from pointrcnn_b200.backbone import Pointnet2MSG
    torch.manual_seed(0)
    net = Pointnet2MSG(input_channels=1).to(cuda).eval()
    for mod in net.modules():
        if isinstance(mod, torch.nn.BatchNorm2d):
            mod.running_mean.uniform_(-0.1, 0.1)
            mod.running_var.uniform_(0.5, 1.5)
    rng = np.random.default_rng(1)
    pc = np.concatenate([rng.uniform(-20, 20, (2, 16384, 3)), rng.uniform(0, 1, (2, 16384, 1))], -1).astype(np.float32)
    x = torch.from_numpy(pc).to(cuda)

    def run():
        with torch.no_grad():
            return [net(x)[1]]

    res, stream = _both(run)
    _assert_equal(res, stream)
